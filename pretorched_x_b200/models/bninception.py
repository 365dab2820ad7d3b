"""BN-Inception (reference: pretorched/models/bninception.py), the backbone TRN and TSN were published with.

The modules are parameter containers created under the reference's names and in its order, so the ``state_dict`` keys, their
order and a seeded random init are the reference's and its checkpoint loads unchanged.  The forward runs on the engine
(engine.run_bninception_trunk): the 7x7 stem on the stem kernel, the ceil-mode pools on the pooling kernel, and every inception
block as one ``functions.frozen`` call whose branches write their columns of the concatenated block output in place -- the 1x1 heads
that read the block input as one split GEMM, the 3x3 branches as slice convolutions, the pool branch as a slice pool (+ its
projection GEMM).

Every ReLU of the reference is ``inplace=True`` on a BatchNorm output, so every ``*_bn_out`` it later reads -- including the inputs
of the stem pools and of each ``torch.cat`` -- is post-ReLU: each unit is conv -> BN -> ReLU.  Inference only: the trunk is frozen,
``last_linear`` is trainable on engine features; there is no ``fine_tune``.
"""
import torch.nn as nn

from .. import engine, ops
from ..ops import Act
from .resnet3d import _attach_settings

__all__ = ['BNInception', 'bninception']

# bninception.py:10-25
pretrained_settings = {
    'bninception': {
        'imagenet': {
            'url': 'http://pretorched-x.csail.mit.edu/models/bn_inception-f8309acd.pth',
            'input_space': 'BGR',
            'input_size': [3, 224, 224],
            'input_range': [0, 255],
            'mean': [104, 117, 128],
            'std': [1, 1, 1],
            'num_classes': 1000
        }
    }
}

# Inception blocks (bninception.py:43-250) in order: name, input channels, 1x1 head (None: none), 3x3 reduce -> 3x3,
# double 3x3 reduce -> 3x3 -> 3x3, pool branch.  Pool branch: ('avg', proj) = AvgPool2d(3, 1, 1) + 1x1 projection, ('max1', proj)
# = MaxPool2d(3, 1, 1) + projection (5b), ('max2', None) = MaxPool2d(3, 2, ceil_mode) pass-through of the block input, which
# also makes the two 3x3 branches stride 2 (3c, 4e).
BLOCKS = [
    ('3a', 192, 64, (64, 64), (64, 96), ('avg', 32)),
    ('3b', 256, 64, (64, 96), (64, 96), ('avg', 64)),
    ('3c', 320, None, (128, 160), (64, 96), ('max2', None)),
    ('4a', 576, 224, (64, 96), (96, 128), ('avg', 128)),
    ('4b', 576, 192, (96, 128), (96, 128), ('avg', 128)),
    ('4c', 576, 160, (128, 160), (128, 160), ('avg', 128)),
    ('4d', 608, 96, (128, 192), (160, 192), ('avg', 128)),
    ('4e', 608, None, (128, 192), (192, 256), ('max2', None)),
    ('5a', 1056, 352, (192, 320), (160, 224), ('avg', 128)),
    ('5b', 1024, 352, (192, 320), (192, 224), ('max1', 128)),
]


def block_out_channels(spec):
    """Channels of a block's concatenated output: 1x1 + 3x3 + double 3x3 + pool branch (bninception.py:288 and the other cats)."""
    _, cin, c1, (_, c3), (_, cd), (_, proj) = spec
    return (c1 or 0) + c3 + cd + (proj if proj is not None else cin)


def _unit(model, name, cin, cout, k, stride=1):
    """Conv2d (+bias) -> BatchNorm2d(eps=1e-5, momentum=0.9) -> ReLU, registered as the reference does."""
    pad = (k // 2, k // 2)
    setattr(model, name, nn.Conv2d(cin, cout, kernel_size=(k, k), stride=(stride, stride), **({'padding': pad} if k > 1 else {})))
    setattr(model, name + '_bn', nn.BatchNorm2d(cout, eps=1e-05, momentum=0.9, affine=True))


class BNInception(engine.CacheOwner, nn.Module):
    """bninception.py:27-495.  ``features`` returns fp32 NCHW [B, 1024, 7, 7] for 224x224 inputs."""

    def __init__(self, num_classes=1000):
        super().__init__()
        inplace = True
        _unit(self, 'conv1_7x7_s2', 3, 64, 7, 2)
        self.conv1_relu_7x7 = nn.ReLU(inplace)
        self.pool1_3x3_s2 = nn.MaxPool2d((3, 3), stride=(2, 2), dilation=(1, 1), ceil_mode=True)
        _unit(self, 'conv2_3x3_reduce', 64, 64, 1)
        self.conv2_relu_3x3_reduce = nn.ReLU(inplace)
        _unit(self, 'conv2_3x3', 64, 192, 3)
        self.conv2_relu_3x3 = nn.ReLU(inplace)
        self.pool2_3x3_s2 = nn.MaxPool2d((3, 3), stride=(2, 2), dilation=(1, 1), ceil_mode=True)
        for n, cin, c1, (c3r, c3), (cdr, cd), (pk, proj) in BLOCKS:
            p = 'inception_%s_' % n
            s = 2 if pk == 'max2' else 1
            if c1 is not None:
                _unit(self, p + '1x1', cin, c1, 1)
                setattr(self, p + 'relu_1x1', nn.ReLU(inplace))
            _unit(self, p + '3x3_reduce', cin, c3r, 1)
            setattr(self, p + 'relu_3x3_reduce', nn.ReLU(inplace))
            _unit(self, p + '3x3', c3r, c3, 3, s)
            setattr(self, p + 'relu_3x3', nn.ReLU(inplace))
            _unit(self, p + 'double_3x3_reduce', cin, cdr, 1)
            setattr(self, p + 'relu_double_3x3_reduce', nn.ReLU(inplace))
            _unit(self, p + 'double_3x3_1', cdr, cd, 3)
            setattr(self, p + 'relu_double_3x3_1', nn.ReLU(inplace))
            _unit(self, p + 'double_3x3_2', cd, cd, 3, s)
            setattr(self, p + 'relu_double_3x3_2', nn.ReLU(inplace))
            if pk == 'avg':
                setattr(self, p + 'pool', nn.AvgPool2d(3, stride=1, padding=1, ceil_mode=True, count_include_pad=True))
            elif pk == 'max1':
                setattr(self, p + 'pool', nn.MaxPool2d((3, 3), stride=(1, 1), padding=(1, 1), dilation=(1, 1), ceil_mode=True))
            else:
                setattr(self, p + 'pool', nn.MaxPool2d((3, 3), stride=(2, 2), dilation=(1, 1), ceil_mode=True))
            if proj is not None:
                _unit(self, p + 'pool_proj', cin, proj, 1)
                setattr(self, p + 'relu_pool_proj', nn.ReLU(inplace))
        self.global_pool = nn.AvgPool2d(7, stride=1, padding=0, ceil_mode=True, count_include_pad=True)
        self.last_linear = nn.Linear(1024, num_classes)

    def features_act(self, x):
        """The trunk on the engine's native layout (fp16 NDHWC ``Act``)."""
        if self.training:
            raise RuntimeError("the forward engine is inference-only: call model.eval() first")
        return engine.run_bninception_trunk(self, x)

    def features(self, input):
        return ops.to_ncdhw(self.features_act(input)).squeeze(2)

    def logits(self, features):
        """global_pool (AvgPool2d(7, stride=1, ceil_mode=True)) -> view -> last_linear (bninception.py:486-490).  The pool is
        fixed at 7x7: on a final map of another size the reference's ``view`` does not give one vector per image, so that case
        raises here instead of pooling differently."""
        a = features if isinstance(features, Act) else ops.from_ncdhw(features, pitch=ops._round_up(features.shape[1], 8))
        if (a.T, a.H, a.W) != (1, 7, 7):
            raise ValueError("BNInception.global_pool is AvgPool2d(7, stride=1): it needs a 7x7 final map (224x224 inputs), got "
                             "%dx%d" % (a.H, a.W))
        return engine.run_head(self, a, self.last_linear)

    def forward(self, input):
        return self.logits(self.features_act(input))


def bninception(num_classes=1000, pretrained='imagenet'):
    """bninception.py:497-511."""
    model = BNInception(num_classes=num_classes)
    if pretrained is not None:
        settings = pretrained_settings['bninception'][pretrained]
        assert num_classes == settings['num_classes'], \
            "num_classes should be {}, but is {}".format(settings['num_classes'], num_classes)
        import torch.utils.model_zoo as model_zoo
        model.load_state_dict(model_zoo.load_url(settings['url']))
        _attach_settings(model, settings)
    return model
