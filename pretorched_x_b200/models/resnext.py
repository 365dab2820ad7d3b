"""ResNeXt-101 32x4d / 64x4d (reference: pretorched/models/resnext.py and resnext_features/), Cadene's Torch7-converted models.

The reference writes the trunk as one ``nn.Sequential`` of Torch7 tables, so its ``state_dict`` keys are positional:
``features.<stage>.<block>.0.0.0.<k>`` for conv1 / bn1 / conv2 / bn2 (k = 0, 1, 3, 4), ``.0.0.1`` / ``.0.0.2`` for conv3 / bn3 and
``.0.1.0`` / ``.0.1.1`` for the projection shortcut.  Here each block is a ``ResNeXt101Bottleneck``, an ``nn.Sequential`` with those
child indices (so the keys, their order and a seeded init are the reference's and Cadene's checkpoints load unchanged) that
exposes ``conv1 .. bn3`` and ``downsample`` as read-only views of its children: the engine runs it as the torchvision-style
bottleneck it is (stride on the grouped 3x3 conv2, a 1x1 projection with BatchNorm as shortcut).  Likewise the model exposes
``conv1 / bn1 / maxpool / layer1 .. layer4`` as views of ``features[0 .. 7]`` (``ResNeXt101Features``, whose call runs the trunk on the engine).

One reference quirk is not kept: ``resnext101_*_features`` is a module-level ``nn.Sequential`` there, so every reference instance
shares (and trains) the same trunk, initialised once at import.  Here each instance owns its modules, initialised in the
reference's module order when the model is built.
"""
import torch.nn as nn

from .. import engine, ops
from ..ops import Act
from .resnet3d import FineTunable, _attach_settings

__all__ = ['ResNeXt101', 'ResNeXt101Features', 'ResNeXt101Bottleneck', 'resnext101_32x4d', 'resnext101_64x4d']

_URLS = {
    'resnext101_32x4d': 'http://pretorched-x.csail.mit.edu/models/resnext101_32x4d-429f0673.pth',
    'resnext101_64x4d': 'http://pretorched-x.csail.mit.edu/models/resnext101_64x4d-d75443fc.pth',
}

# resnext.py:12-35
pretrained_settings = {
    name: {'imagenet': {'url': url, 'input_space': 'RGB', 'input_size': [3, 224, 224], 'input_range': [0, 1],
                        'mean': [0.485, 0.456, 0.406], 'std': [0.229, 0.224, 0.225], 'num_classes': 1000}}
    for name, url in _URLS.items()
}

# name -> groups; both have 4 channels per group in layer1, doubling per stage (cg = 4, 8, 16, 32)
_GROUPS = {'resnext101_32x4d': 32, 'resnext101_64x4d': 64}
_LAYERS = (3, 4, 23, 3)


class CAddTable(nn.Module):
    """Torch7's CAddTable (the residual sum).  Parameterless: only keeps the block's child indices; the engine adds the shortcut
    in the closing convolution's epilogue."""

    def forward(self, pair):
        return pair[0] + pair[1]


class ResNeXt101Bottleneck(engine.CacheOwner, nn.Sequential):
    """One block of resnext101_*_features.py: ConcatTable(main, shortcut) -> CAddTable -> ReLU, where main is
    (conv1 1x1 -> bn1 -> ReLU -> conv2 grouped 3x3 (stride) -> bn2 -> ReLU) -> conv3 1x1 -> bn3 and shortcut is a strided 1x1
    projection + BatchNorm or the identity (an empty Sequential, Torch7's Identity)."""

    def __init__(self, inplanes, width, planes, groups, stride, project):
        main = nn.Sequential(
            nn.Sequential(
                nn.Conv2d(inplanes, width, 1, 1, 0, bias=False), nn.BatchNorm2d(width), nn.ReLU(),
                nn.Conv2d(width, width, 3, stride, 1, groups=groups, bias=False), nn.BatchNorm2d(width), nn.ReLU()),
            nn.Conv2d(width, planes, 1, 1, 0, bias=False), nn.BatchNorm2d(planes))
        shortcut = nn.Sequential(nn.Conv2d(inplanes, planes, 1, stride, 0, bias=False), nn.BatchNorm2d(planes)) if project \
            else nn.Sequential()
        super().__init__(nn.ModuleList([main, shortcut]), CAddTable(), nn.ReLU())

    conv1 = property(lambda self: self[0][0][0][0])
    bn1 = property(lambda self: self[0][0][0][1])
    conv2 = property(lambda self: self[0][0][0][3])
    bn2 = property(lambda self: self[0][0][0][4])
    conv3 = property(lambda self: self[0][0][1])
    bn3 = property(lambda self: self[0][0][2])
    downsample = property(lambda self: self[0][1] if len(self[0][1]) else None)

    def forward(self, x):
        if isinstance(x, Act):
            return engine.run_bottleneck(self, x)
        return ops.to_ncdhw(engine.run_bottleneck(self, ops.from_ncdhw(x, pitch=ops._round_up(x.shape[1], 8)))).squeeze(2)


class ResNeXt101Features(engine.CacheOwner, nn.Sequential):
    """resnext101_*_features: conv1 7x7/2 -> BN -> ReLU -> MaxPool2d(3, 2, 1) -> four stages of ``ResNeXt101Bottleneck``.  Calling
    it runs the trunk on the engine and returns the final map as NCHW fp16, where the reference's returns fp32."""

    conv1 = property(lambda self: self[0])
    bn1 = property(lambda self: self[1])
    maxpool = property(lambda self: self[3])
    layer1 = property(lambda self: self[4])
    layer2 = property(lambda self: self[5])
    layer3 = property(lambda self: self[6])
    layer4 = property(lambda self: self[7])

    def forward(self, x):
        if self.training:
            raise RuntimeError("the forward engine is inference-only: call model.eval() first")
        return ops.to_ncdhw(engine.run_trunk(self, x)).squeeze(2)


class ResNeXt101(engine.CacheOwner, FineTunable, nn.Module):
    """ResNeXt101_32x4d / ResNeXt101_64x4d (resnext.py:37-83): features (7x7 stem, max-pool, 3 + 4 + 23 + 3 bottlenecks) ->
    AvgPool2d(7, 1) -> last_linear.

    ``fine_tune(k)`` has the contract of ``ResNet2D.fine_tune`` (frozen BatchNorm, model in ``eval()``, 1 <= k <= 5): stage k is
    ``features.{3 + k}`` and k = 5 trains ``last_linear`` only.  The grouped 3x3 conv2 trains on the group-aware input-gradient
    kernel and the diagonal-block weight-gradient kernel (b2_conv_grouped_ndhwc_dgrad, b2_conv_wgrad_grouped)."""

    stem_desc = '7x7 convolution'

    def __init__(self, groups, num_classes=1000):
        super().__init__()
        self.num_classes = num_classes
        stem = [nn.Conv2d(3, 64, 7, 2, 3, bias=False), nn.BatchNorm2d(64), nn.ReLU(), nn.MaxPool2d(3, 2, 1)]
        stages, inplanes = [], 64
        for i, n in enumerate(_LAYERS):
            width, planes = groups * 4 << i, 256 << i
            stages.append(nn.Sequential(*[ResNeXt101Bottleneck(inplanes if b == 0 else planes, width, planes, groups,
                                                               2 if b == 0 and i > 0 else 1, b == 0) for b in range(n)]))
            inplanes = planes
        self.features = ResNeXt101Features(*stem, *stages)
        self.avg_pool = nn.AvgPool2d((7, 7), (1, 1))
        self.last_linear = nn.Linear(2048, num_classes)

    # the views the engine's trunk walk and FineTunable read
    conv1 = property(lambda self: self.features.conv1)
    bn1 = property(lambda self: self.features.bn1)
    maxpool = property(lambda self: self.features.maxpool)
    layer1 = property(lambda self: self.features.layer1)
    layer2 = property(lambda self: self.features.layer2)
    layer3 = property(lambda self: self.features.layer3)
    layer4 = property(lambda self: self.features.layer4)

    def _stage_prefix(self, i):
        return 'features.%d.' % (3 + i)

    def logits(self, input):
        """avg_pool (AvgPool2d(7, 1)) -> view -> last_linear (resnext.py:45-49).  The reference's pool is fixed at 7x7: on a
        final map of another size its output is not one vector per image and ``last_linear`` rejects it, so that case raises
        here instead of pooling differently."""
        a = input if isinstance(input, Act) else ops.from_ncdhw(input, pitch=ops._round_up(input.shape[1], 8))
        if (a.T, a.H, a.W) != (1, 7, 7):
            raise ValueError("ResNeXt101.avg_pool is AvgPool2d(7, 1): it needs a 7x7 final map (224x224 inputs), got %dx%d"
                             % (a.H, a.W))
        return engine.run_head(self, a, self.last_linear)

    def forward(self, input):
        return self.logits(self.features_act(input))


def _factory(name):
    def build(num_classes=1000, pretrained='imagenet'):
        model = ResNeXt101(_GROUPS[name], num_classes=num_classes)
        if pretrained is not None:
            settings = pretrained_settings[name][pretrained]
            assert num_classes == settings['num_classes'], \
                "num_classes should be {}, but is {}".format(settings['num_classes'], num_classes)
            import torch.utils.model_zoo as model_zoo
            model.load_state_dict(model_zoo.load_url(settings['url']))
            _attach_settings(model, settings)
        return model

    build.__name__ = name
    build.__doc__ = "Constructs a %s (resnext.py:86-112)." % name
    return build


resnext101_32x4d = _factory('resnext101_32x4d')
resnext101_64x4d = _factory('resnext101_64x4d')
