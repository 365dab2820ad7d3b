"""Inception-v4 and Inception-ResNet-v2 (reference: pretorched/models/inceptionv4.py, inceptionresnetv2.py).

The modules are parameter containers created under the reference's names and in its order, so the ``state_dict`` keys, their
order and a seeded random init are the reference's and its checkpoints load unchanged.  The forward runs on the engine
(engine.run_inception_trunk): every block is one ``functions.frozen`` call whose branches write their columns of the
concatenated block output in place -- the 1x1 heads that read the block input as one split GEMM, the convolutions with taps
(valid-padded 3x3, 1x7 / 7x1, 1x3 / 3x1, 5x5) as slab slice convolutions, the pool branches as slice pools -- and whose
residual form (Block35 / 17 / 8) closes with the persistent GEMM: per-column scale, shift, the block input as residual, ReLU.
Each ``BasicConv2d`` is conv (no bias) -> BatchNorm(eps = 0.001) -> ReLU.  Inference only: the trunk is frozen, ``last_linear``
is trainable on engine features; there is no ``fine_tune``.
"""
import torch.nn as nn

from .. import engine, ops
from ..ops import Act
from .resnet3d import _attach_settings
from .utils import Trunk

__all__ = ['InceptionV4', 'inceptionv4', 'InceptionResNetV2', 'inceptionresnetv2']


def _row(url, num_classes):
    return {'url': url, 'input_space': 'RGB', 'input_size': [3, 299, 299], 'input_range': [0, 1], 'mean': [0.5, 0.5, 0.5],
            'std': [0.5, 0.5, 0.5], 'num_classes': num_classes}


# inceptionv4.py:10-31, inceptionresnetv2.py:10-31
_V4_URL = 'http://pretorched-x.csail.mit.edu/models/inceptionv4-0f7d42d3.pth'
_IRV2_URL = 'http://pretorched-x.csail.mit.edu/models/inceptionresnetv2-c2ef1dee.pth'
pretrained_settings = {
    'inceptionv4': {'imagenet': _row(_V4_URL, 1000), 'imagenet+background': _row(_V4_URL, 1001)},
    'inceptionresnetv2': {'imagenet': _row(_IRV2_URL, 1000), 'imagenet+background': _row(_IRV2_URL, 1001)},
}


class BasicConv2d(nn.Module):
    """conv (no bias) -> BatchNorm2d(eps=0.001, momentum=0.1) -> ReLU (inceptionv4.py:34-51)."""

    def __init__(self, in_planes, out_planes, kernel_size, stride, padding=0):
        super().__init__()
        self.conv = nn.Conv2d(in_planes, out_planes, kernel_size=kernel_size, stride=stride, padding=padding, bias=False)
        self.bn = nn.BatchNorm2d(out_planes, eps=0.001, momentum=0.1, affine=True)
        self.relu = nn.ReLU(inplace=True)


def _seq(*units):
    return nn.Sequential(*[BasicConv2d(*u[:4], **({'padding': u[4]} if len(u) > 4 else {})) for u in units])


def _pool_branch(cin, proj):
    return nn.Sequential(nn.AvgPool2d(3, stride=1, padding=1, count_include_pad=False), BasicConv2d(cin, proj, kernel_size=1, stride=1))


# Blocks as data (engine._inception_block_body): BRANCHES[kind] lists the branches in the order of the reference's torch.cat.
#   ('chain', paths)        BasicConv2d units in sequence from the block input, the last one writes the branch's slice
#   ('fork', paths, (a, b)) a chain whose output feeds two units that write adjacent slices (Inception-C, inceptionv4.py:245-255)
#   ('max', path)           MaxPool2d(3, stride=2) of the block input, its slice the block input's channels (``path`` None: a
#                           functional F.max_pool2d(3, 2), as in torchvision's blocks)
#   ('avg', paths, incl)    AvgPool2d(3, 1, 1) of the block input, the padding counted in the divisor when ``incl``
#                           (count_include_pad), then the unit(s) in ``paths``
# RESIDUAL kinds close with ``conv2d`` (1x1 with bias): out = relu(conv2d(cat) * scale + x) (inceptionresnetv2.py:109-117).
# The Inception* rows are torchvision's Inception3 blocks (models/inceptionv3.py), whose pools are functional calls.
BRANCHES = {
    'Mixed_3a': [('max', 'maxpool'), ('chain', ['conv'])],
    'Mixed_4a': [('chain', ['branch0.0', 'branch0.1']), ('chain', ['branch1.0', 'branch1.1', 'branch1.2', 'branch1.3'])],
    'Mixed_5a': [('chain', ['conv']), ('max', 'maxpool')],
    'Inception_A': [('chain', ['branch0']), ('chain', ['branch1.0', 'branch1.1']), ('chain', ['branch2.0', 'branch2.1', 'branch2.2']),
                    ('avg', ['branch3.1'], False)],
    'Reduction_A': [('chain', ['branch0']), ('chain', ['branch1.0', 'branch1.1', 'branch1.2']), ('max', 'branch2')],
    'Inception_B': [('chain', ['branch0']), ('chain', ['branch1.0', 'branch1.1', 'branch1.2']),
                    ('chain', ['branch2.0', 'branch2.1', 'branch2.2', 'branch2.3', 'branch2.4']), ('avg', ['branch3.1'], False)],
    'Reduction_B': [('chain', ['branch0.0', 'branch0.1']), ('chain', ['branch1.0', 'branch1.1', 'branch1.2', 'branch1.3']),
                    ('max', 'branch2')],
    'Inception_C': [('chain', ['branch0']), ('fork', ['branch1_0'], ('branch1_1a', 'branch1_1b')),
                    ('fork', ['branch2_0', 'branch2_1', 'branch2_2'], ('branch2_3a', 'branch2_3b')), ('avg', ['branch3.1'], False)],
    'Mixed_5b': [('chain', ['branch0']), ('chain', ['branch1.0', 'branch1.1']), ('chain', ['branch2.0', 'branch2.1', 'branch2.2']),
                 ('avg', ['branch3.1'], False)],
    'Block35': [('chain', ['branch0']), ('chain', ['branch1.0', 'branch1.1']), ('chain', ['branch2.0', 'branch2.1', 'branch2.2'])],
    'Mixed_6a': [('chain', ['branch0']), ('chain', ['branch1.0', 'branch1.1', 'branch1.2']), ('max', 'branch2')],
    'Block17': [('chain', ['branch0']), ('chain', ['branch1.0', 'branch1.1', 'branch1.2'])],
    'Mixed_7a': [('chain', ['branch0.0', 'branch0.1']), ('chain', ['branch1.0', 'branch1.1']),
                 ('chain', ['branch2.0', 'branch2.1', 'branch2.2']), ('max', 'branch3')],
    'Block8': [('chain', ['branch0']), ('chain', ['branch1.0', 'branch1.1', 'branch1.2'])],
    'InceptionA': [('chain', ['branch1x1']), ('chain', ['branch5x5_1', 'branch5x5_2']),
                   ('chain', ['branch3x3dbl_1', 'branch3x3dbl_2', 'branch3x3dbl_3']), ('avg', ['branch_pool'], True)],
    'InceptionB': [('chain', ['branch3x3']), ('chain', ['branch3x3dbl_1', 'branch3x3dbl_2', 'branch3x3dbl_3']), ('max', None)],
    'InceptionC': [('chain', ['branch1x1']), ('chain', ['branch7x7_1', 'branch7x7_2', 'branch7x7_3']),
                   ('chain', ['branch7x7dbl_1', 'branch7x7dbl_2', 'branch7x7dbl_3', 'branch7x7dbl_4', 'branch7x7dbl_5']),
                   ('avg', ['branch_pool'], True)],
    'InceptionD': [('chain', ['branch3x3_1', 'branch3x3_2']), ('chain', ['branch7x7x3_1', 'branch7x7x3_2', 'branch7x7x3_3',
                                                                         'branch7x7x3_4']), ('max', None)],
    'InceptionE': [('chain', ['branch1x1']), ('fork', ['branch3x3_1'], ('branch3x3_2a', 'branch3x3_2b')),
                   ('fork', ['branch3x3dbl_1', 'branch3x3dbl_2'], ('branch3x3dbl_3a', 'branch3x3dbl_3b')),
                   ('avg', ['branch_pool'], True)],
}
RESIDUAL = ('Block35', 'Block17', 'Block8')
V3_KINDS = ('InceptionA', 'InceptionB', 'InceptionC', 'InceptionD', 'InceptionE')   # their classes are in models/inceptionv3.py


class _Block(engine.CacheOwner, nn.Module):
    kind = None


class Mixed_3a(_Block):
    def __init__(self):
        super().__init__()
        self.maxpool = nn.MaxPool2d(3, stride=2)
        self.conv = BasicConv2d(64, 96, kernel_size=3, stride=2)


class Mixed_4a(_Block):
    def __init__(self):
        super().__init__()
        self.branch0 = _seq((160, 64, 1, 1), (64, 96, 3, 1))
        self.branch1 = _seq((160, 64, 1, 1), (64, 64, (1, 7), 1, (0, 3)), (64, 64, (7, 1), 1, (3, 0)), (64, 96, (3, 3), 1))


class Mixed_5a(_Block):
    def __init__(self):
        super().__init__()
        self.conv = BasicConv2d(192, 192, kernel_size=3, stride=2)
        self.maxpool = nn.MaxPool2d(3, stride=2)


class Inception_A(_Block):
    def __init__(self):
        super().__init__()
        self.branch0 = BasicConv2d(384, 96, kernel_size=1, stride=1)
        self.branch1 = _seq((384, 64, 1, 1), (64, 96, 3, 1, 1))
        self.branch2 = _seq((384, 64, 1, 1), (64, 96, 3, 1, 1), (96, 96, 3, 1, 1))
        self.branch3 = _pool_branch(384, 96)


class Reduction_A(_Block):
    def __init__(self):
        super().__init__()
        self.branch0 = BasicConv2d(384, 384, kernel_size=3, stride=2)
        self.branch1 = _seq((384, 192, 1, 1), (192, 224, 3, 1, 1), (224, 256, 3, 2))
        self.branch2 = nn.MaxPool2d(3, stride=2)


class Inception_B(_Block):
    def __init__(self):
        super().__init__()
        self.branch0 = BasicConv2d(1024, 384, kernel_size=1, stride=1)
        self.branch1 = _seq((1024, 192, 1, 1), (192, 224, (1, 7), 1, (0, 3)), (224, 256, (7, 1), 1, (3, 0)))
        self.branch2 = _seq((1024, 192, 1, 1), (192, 192, (7, 1), 1, (3, 0)), (192, 224, (1, 7), 1, (0, 3)),
                            (224, 224, (7, 1), 1, (3, 0)), (224, 256, (1, 7), 1, (0, 3)))
        self.branch3 = _pool_branch(1024, 128)


class Reduction_B(_Block):
    def __init__(self):
        super().__init__()
        self.branch0 = _seq((1024, 192, 1, 1), (192, 192, 3, 2))
        self.branch1 = _seq((1024, 256, 1, 1), (256, 256, (1, 7), 1, (0, 3)), (256, 320, (7, 1), 1, (3, 0)), (320, 320, 3, 2))
        self.branch2 = nn.MaxPool2d(3, stride=2)


class Inception_C(_Block):
    def __init__(self):
        super().__init__()
        self.branch0 = BasicConv2d(1536, 256, kernel_size=1, stride=1)
        self.branch1_0 = BasicConv2d(1536, 384, kernel_size=1, stride=1)
        self.branch1_1a = BasicConv2d(384, 256, kernel_size=(1, 3), stride=1, padding=(0, 1))
        self.branch1_1b = BasicConv2d(384, 256, kernel_size=(3, 1), stride=1, padding=(1, 0))
        self.branch2_0 = BasicConv2d(1536, 384, kernel_size=1, stride=1)
        self.branch2_1 = BasicConv2d(384, 448, kernel_size=(3, 1), stride=1, padding=(1, 0))
        self.branch2_2 = BasicConv2d(448, 512, kernel_size=(1, 3), stride=1, padding=(0, 1))
        self.branch2_3a = BasicConv2d(512, 256, kernel_size=(1, 3), stride=1, padding=(0, 1))
        self.branch2_3b = BasicConv2d(512, 256, kernel_size=(3, 1), stride=1, padding=(1, 0))
        self.branch3 = _pool_branch(1536, 256)


class Mixed_5b(_Block):
    def __init__(self):
        super().__init__()
        self.branch0 = BasicConv2d(192, 96, kernel_size=1, stride=1)
        self.branch1 = _seq((192, 48, 1, 1), (48, 64, 5, 1, 2))
        self.branch2 = _seq((192, 64, 1, 1), (64, 96, 3, 1, 1), (96, 96, 3, 1, 1))
        self.branch3 = _pool_branch(192, 64)


class Block35(_Block):
    def __init__(self, scale=1.0):
        super().__init__()
        self.scale = scale
        self.branch0 = BasicConv2d(320, 32, kernel_size=1, stride=1)
        self.branch1 = _seq((320, 32, 1, 1), (32, 32, 3, 1, 1))
        self.branch2 = _seq((320, 32, 1, 1), (32, 48, 3, 1, 1), (48, 64, 3, 1, 1))
        self.conv2d = nn.Conv2d(128, 320, kernel_size=1, stride=1)
        self.relu = nn.ReLU(inplace=False)


class Mixed_6a(_Block):
    def __init__(self):
        super().__init__()
        self.branch0 = BasicConv2d(320, 384, kernel_size=3, stride=2)
        self.branch1 = _seq((320, 256, 1, 1), (256, 256, 3, 1, 1), (256, 384, 3, 2))
        self.branch2 = nn.MaxPool2d(3, stride=2)


class Block17(_Block):
    def __init__(self, scale=1.0):
        super().__init__()
        self.scale = scale
        self.branch0 = BasicConv2d(1088, 192, kernel_size=1, stride=1)
        self.branch1 = _seq((1088, 128, 1, 1), (128, 160, (1, 7), 1, (0, 3)), (160, 192, (7, 1), 1, (3, 0)))
        self.conv2d = nn.Conv2d(384, 1088, kernel_size=1, stride=1)
        self.relu = nn.ReLU(inplace=False)


class Mixed_7a(_Block):
    def __init__(self):
        super().__init__()
        self.branch0 = _seq((1088, 256, 1, 1), (256, 384, 3, 2))
        self.branch1 = _seq((1088, 256, 1, 1), (256, 288, 3, 2))
        self.branch2 = _seq((1088, 256, 1, 1), (256, 288, 3, 1, 1), (288, 320, 3, 2))
        self.branch3 = nn.MaxPool2d(3, stride=2)


class Block8(_Block):
    def __init__(self, scale=1.0, noReLU=False):
        super().__init__()
        self.scale = scale
        self.noReLU = noReLU
        self.branch0 = BasicConv2d(2080, 192, kernel_size=1, stride=1)
        self.branch1 = _seq((2080, 192, 1, 1), (192, 224, (1, 3), 1, (0, 1)), (224, 256, (3, 1), 1, (1, 0)))
        self.conv2d = nn.Conv2d(448, 2080, kernel_size=1, stride=1)
        if not self.noReLU:
            self.relu = nn.ReLU(inplace=False)


for _k in BRANCHES:
    if _k not in V3_KINDS:
        globals()[_k].kind = _k


class _Trunk(Trunk):
    """``InceptionV4.features`` (inceptionv4.py:273-296): the reference's Sequential.  Returns fp32 NCHW [B, 1536, 8, 8] for
    299x299 inputs."""

    _model = 'InceptionV4'

    def _run(self, x):
        return engine.run_inception_trunk(V4_STEM, list(self), x)


V4_STEM = 3         # features[0:3] are the stem's BasicConv2d units, features[3:] the blocks


def _final_pool(model, features):
    """avg_pool / avgpool_1a (AvgPool2d(8, count_include_pad=False)) -> view -> last_linear (inceptionv4.py:300-304).  On the
    8x8 map of a 299x299 input the pool is the global mean; any other final map raises instead of pooling differently."""
    a = features if isinstance(features, Act) else ops.from_ncdhw(features, pitch=ops._round_up(features.shape[1], 8))
    if (a.T, a.H, a.W) != (1, 8, 8):
        raise ValueError("%s's final pool is AvgPool2d(8): it needs an 8x8 final map (299x299 inputs), got %dx%d"
                         % (type(model).__name__, a.H, a.W))
    return engine.run_head(model, a, model.last_linear)


class InceptionV4(engine.CacheOwner, nn.Module):
    """inceptionv4.py:263-309."""

    def __init__(self, num_classes=1001):
        super().__init__()
        self.input_space = None
        self.input_size = (299, 299, 3)
        self.mean = None
        self.std = None
        self.features = _Trunk(
            BasicConv2d(3, 32, kernel_size=3, stride=2), BasicConv2d(32, 32, kernel_size=3, stride=1),
            BasicConv2d(32, 64, kernel_size=3, stride=1, padding=1), Mixed_3a(), Mixed_4a(), Mixed_5a(),
            *[Inception_A() for _ in range(4)], Reduction_A(), *[Inception_B() for _ in range(7)], Reduction_B(),
            *[Inception_C() for _ in range(3)])
        self.avg_pool = nn.AvgPool2d(8, count_include_pad=False)
        self.last_linear = nn.Linear(1536, num_classes)

    def features_act(self, x):
        """The trunk on the engine's native layout (fp16 NDHWC ``Act``)."""
        return self.features.run_act(x)

    def logits(self, features):
        return _final_pool(self, features)

    def forward(self, input):
        return self.logits(self.features_act(input))


class InceptionResNetV2(engine.CacheOwner, nn.Module):
    """inceptionresnetv2.py:234-331."""

    def __init__(self, num_classes=1001):
        super().__init__()
        self.input_space = None
        self.input_size = (299, 299, 3)
        self.mean = None
        self.std = None
        self.conv2d_1a = BasicConv2d(3, 32, kernel_size=3, stride=2)
        self.conv2d_2a = BasicConv2d(32, 32, kernel_size=3, stride=1)
        self.conv2d_2b = BasicConv2d(32, 64, kernel_size=3, stride=1, padding=1)
        self.maxpool_3a = nn.MaxPool2d(3, stride=2)
        self.conv2d_3b = BasicConv2d(64, 80, kernel_size=1, stride=1)
        self.conv2d_4a = BasicConv2d(80, 192, kernel_size=3, stride=1)
        self.maxpool_5a = nn.MaxPool2d(3, stride=2)
        self.mixed_5b = Mixed_5b()
        self.repeat = nn.Sequential(*[Block35(scale=0.17) for _ in range(10)])
        self.mixed_6a = Mixed_6a()
        self.repeat_1 = nn.Sequential(*[Block17(scale=0.10) for _ in range(20)])
        self.mixed_7a = Mixed_7a()
        self.repeat_2 = nn.Sequential(*[Block8(scale=0.20) for _ in range(9)])
        self.block8 = Block8(noReLU=True)
        self.conv2d_7b = BasicConv2d(2080, 1536, kernel_size=1, stride=1)
        self.avgpool_1a = nn.AvgPool2d(8, count_include_pad=False)
        self.last_linear = nn.Linear(1536, num_classes)

    def _units(self):
        stem = [self.conv2d_1a, self.conv2d_2a, self.conv2d_2b, self.maxpool_3a, self.conv2d_3b, self.conv2d_4a, self.maxpool_5a]
        return stem, [self.mixed_5b, *self.repeat, self.mixed_6a, *self.repeat_1, self.mixed_7a, *self.repeat_2, self.block8,
                      self.conv2d_7b]

    def features_act(self, x):
        """The trunk on the engine's native layout (fp16 NDHWC ``Act``)."""
        if self.training:
            raise RuntimeError("the forward engine is inference-only: call model.eval() first")
        stem, rest = self._units()
        return engine.run_inception_trunk(len(stem), stem + rest, x)

    def features(self, input):
        return ops.to_ncdhw(self.features_act(input)).squeeze(2)

    def logits(self, features):
        return _final_pool(self, features)

    def forward(self, input):
        return self.logits(self.features_act(input))


def _factory(cls, arch, num_classes, pretrained):
    """inceptionv4.py:312-335 / inceptionresnetv2.py:333-360: both rows load the 1001-class checkpoint; 'imagenet' drops row 0
    (the background class) of last_linear."""
    if not pretrained:
        return cls(num_classes=num_classes)
    settings = pretrained_settings[arch][pretrained]
    assert num_classes == settings['num_classes'], \
        "num_classes should be {}, but is {}".format(settings['num_classes'], num_classes)
    import torch.utils.model_zoo as model_zoo
    model = cls(num_classes=1001)
    model.load_state_dict(model_zoo.load_url(settings['url']))
    if pretrained == 'imagenet':
        new_last_linear = nn.Linear(1536, 1000)
        new_last_linear.weight.data = model.last_linear.weight.data[1:]
        new_last_linear.bias.data = model.last_linear.bias.data[1:]
        model.last_linear = new_last_linear
    _attach_settings(model, settings)
    return model


def inceptionv4(num_classes=1000, pretrained='imagenet'):
    """inceptionv4.py:312-335."""
    return _factory(InceptionV4, 'inceptionv4', num_classes, pretrained)


def inceptionresnetv2(num_classes=1000, pretrained='imagenet'):
    """inceptionresnetv2.py:333-360."""
    return _factory(InceptionResNetV2, 'inceptionresnetv2', num_classes, pretrained)
