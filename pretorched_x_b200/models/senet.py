"""SE-ResNet and SE-ResNeXt (reference: pretorched/models/senet.py), the Caffe-layout SENets of Cadene's model zoo.

The modules are parameter containers created in the reference's order (``layer0`` as an ``OrderedDict`` Sequential, the
downsample projection of a stage before its first block, inside a block conv1 .. bn3 then the SE module), so the
``state_dict`` keys, their order and a seeded random init are the reference's and the zoo checkpoints load unchanged.  The
forward runs on the engine (engine.run_senet_trunk): the 7x7 stem on the stem kernel, the ceil-mode stem pool on the pooling
kernel with an explicit output extent, and every bottleneck as conv1 -> conv2 -> squeeze-excite (csrc/b2_se.cu) -> the closing
1x1 GEMM with the excitation folded into its per-sample affine.

``senet154`` is not offered: its three-conv 3x3 stem, 64-group convolutions with 2 channels per group and 3x3 projections are
outside the engine's kernels.
"""
import math
from collections import OrderedDict

import torch.nn as nn

from .. import engine, ops
from ..ops import Act
from .resnet3d import _attach_settings

__all__ = ['SENet', 'se_resnet50', 'se_resnet101', 'se_resnet152', 'se_resnext50_32x4d', 'se_resnext101_32x4d']

_URLS = {
    'se_resnet50': 'http://pretorched-x.csail.mit.edu/models/se_resnet50-8049f9c4.pth',
    'se_resnet101': 'http://pretorched-x.csail.mit.edu/models/se_resnet101-af4def2b.pth',
    'se_resnet152': 'http://pretorched-x.csail.mit.edu/models/se_resnet152-457c373d.pth',
    'se_resnext50_32x4d': 'http://pretorched-x.csail.mit.edu/models/se_resnext50_32x4d-377ad789.pth',
    'se_resnext101_32x4d': 'http://pretorched-x.csail.mit.edu/models/se_resnext101_32x4d-bcc25309.pth',
}

# senet.py:15-82 (the senet154 row aside)
pretrained_settings = {
    name: {'imagenet': {'url': url, 'input_space': 'RGB', 'input_size': [3, 224, 224], 'input_range': [0, 1],
                        'mean': [0.485, 0.456, 0.406], 'std': [0.229, 0.224, 0.225], 'num_classes': 1000}}
    for name, url in _URLS.items()
}


class SEModule(nn.Module):
    """senet.py:85-104: avgpool -> fc1 (1x1, reduction) -> ReLU -> fc2 -> sigmoid, a per-sample channel scale.  Its arithmetic
    runs inside the enclosing block (engine._se_bottleneck_body)."""

    def __init__(self, channels, reduction):
        super().__init__()
        self.avg_pool = nn.AdaptiveAvgPool2d(1)
        self.fc1 = nn.Conv2d(channels, channels // reduction, kernel_size=1, padding=0)
        self.relu = nn.ReLU(inplace=True)
        self.fc2 = nn.Conv2d(channels // reduction, channels, kernel_size=1, padding=0)
        self.sigmoid = nn.Sigmoid()


class SEBottleneckBase(engine.CacheOwner, nn.Module):
    """Bottleneck.forward (senet.py:107-131): conv1-bn1-relu, conv2-bn2-relu, conv3-bn3, se_module, + shortcut, relu."""

    def forward(self, x):
        if isinstance(x, Act):
            return engine.run_se_bottleneck(self, x)
        return ops.to_ncdhw(engine.run_se_bottleneck(self, ops.from_ncdhw(x, pitch=ops._round_up(x.shape[1], 8)))).squeeze(2)


class SEResNetBottleneck(SEBottleneckBase):
    """senet.py:158-180: the Caffe layout, stride on the 1x1 conv1."""
    expansion = 4

    def __init__(self, inplanes, planes, groups, reduction, stride=1, downsample=None):
        super().__init__()
        self.conv1 = nn.Conv2d(inplanes, planes, kernel_size=1, bias=False, stride=stride)
        self.bn1 = nn.BatchNorm2d(planes)
        self.conv2 = nn.Conv2d(planes, planes, kernel_size=3, padding=1, groups=groups, bias=False)
        self.bn2 = nn.BatchNorm2d(planes)
        self.conv3 = nn.Conv2d(planes, planes * 4, kernel_size=1, bias=False)
        self.bn3 = nn.BatchNorm2d(planes * 4)
        self.relu = nn.ReLU(inplace=True)
        self.se_module = SEModule(planes * 4, reduction=reduction)
        self.downsample = downsample
        self.stride = stride


class SEResNeXtBottleneck(SEBottleneckBase):
    """senet.py:183-204: ResNeXt bottleneck type C, stride on the grouped 3x3 conv2."""
    expansion = 4

    def __init__(self, inplanes, planes, groups, reduction, stride=1, downsample=None, base_width=4):
        super().__init__()
        width = math.floor(planes * (base_width / 64)) * groups
        self.conv1 = nn.Conv2d(inplanes, width, kernel_size=1, bias=False, stride=1)
        self.bn1 = nn.BatchNorm2d(width)
        self.conv2 = nn.Conv2d(width, width, kernel_size=3, stride=stride, padding=1, groups=groups, bias=False)
        self.bn2 = nn.BatchNorm2d(width)
        self.conv3 = nn.Conv2d(width, planes * 4, kernel_size=1, bias=False)
        self.bn3 = nn.BatchNorm2d(planes * 4)
        self.relu = nn.ReLU(inplace=True)
        self.se_module = SEModule(planes * 4, reduction=reduction)
        self.downsample = downsample
        self.stride = stride


class SENet(engine.CacheOwner, nn.Module):
    """senet.py:207-366 for the SE-ResNet / SE-ResNeXt configurations (7x7 stem, 1x1 projections, no dropout)."""

    def __init__(self, block, layers, groups, reduction, dropout_p=0.2, inplanes=128, input_3x3=True, downsample_kernel_size=3,
                 downsample_padding=1, num_classes=1000):
        super().__init__()
        if input_3x3 or downsample_kernel_size != 1 or downsample_padding != 0:
            raise NotImplementedError("the engine runs the SENets with a 7x7 stem and 1x1 projections (SE-ResNet, SE-ResNeXt); "
                                      "senet154's 3x3 stem and 3x3 projections are outside its scope")
        self.inplanes = inplanes
        layer0_modules = [
            ('conv1', nn.Conv2d(3, inplanes, kernel_size=7, stride=2, padding=3, bias=False)),
            ('bn1', nn.BatchNorm2d(inplanes)),
            ('relu1', nn.ReLU(inplace=True)),
        ]
        # ceil_mode=True instead of padding=1, for compatibility with the Caffe weights (senet.py:279-282)
        layer0_modules.append(('pool', nn.MaxPool2d(3, stride=2, ceil_mode=True)))
        self.layer0 = nn.Sequential(OrderedDict(layer0_modules))
        self.layer1 = self._make_layer(block, planes=64, blocks=layers[0], groups=groups, reduction=reduction,
                                       downsample_kernel_size=1, downsample_padding=0)
        self.layer2 = self._make_layer(block, planes=128, blocks=layers[1], stride=2, groups=groups, reduction=reduction,
                                       downsample_kernel_size=downsample_kernel_size, downsample_padding=downsample_padding)
        self.layer3 = self._make_layer(block, planes=256, blocks=layers[2], stride=2, groups=groups, reduction=reduction,
                                       downsample_kernel_size=downsample_kernel_size, downsample_padding=downsample_padding)
        self.layer4 = self._make_layer(block, planes=512, blocks=layers[3], stride=2, groups=groups, reduction=reduction,
                                       downsample_kernel_size=downsample_kernel_size, downsample_padding=downsample_padding)
        self.avg_pool = nn.AvgPool2d(7, stride=1)
        self.dropout = nn.Dropout(dropout_p) if dropout_p is not None else None
        self.last_linear = nn.Linear(512 * block.expansion, num_classes)

    def _make_layer(self, block, planes, blocks, groups, reduction, stride=1, downsample_kernel_size=1, downsample_padding=0):
        downsample = None
        if stride != 1 or self.inplanes != planes * block.expansion:
            downsample = nn.Sequential(
                nn.Conv2d(self.inplanes, planes * block.expansion, kernel_size=downsample_kernel_size, stride=stride,
                          padding=downsample_padding, bias=False),
                nn.BatchNorm2d(planes * block.expansion),
            )
        layers = [block(self.inplanes, planes, groups, reduction, stride, downsample)]
        self.inplanes = planes * block.expansion
        for _ in range(1, blocks):
            layers.append(block(self.inplanes, planes, groups, reduction))
        return nn.Sequential(*layers)

    def features_act(self, x):
        """layer0 .. layer4 on the engine's native layout (fp16 NDHWC ``Act``)."""
        if self.training:
            raise RuntimeError("the forward engine is inference-only: call model.eval() first")
        return engine.run_senet_trunk(self, x)

    def features(self, x):
        return ops.to_ncdhw(self.features_act(x)).squeeze(2)

    def logits(self, x):
        """avg_pool (AvgPool2d(7, stride=1)) -> dropout (the identity in eval mode) -> view -> last_linear (senet.py:355-361).
        The reference's pool is fixed at 7x7: on a final map of another size its output is not one vector per image and
        ``last_linear`` rejects it, so that case raises here instead of pooling differently."""
        a = x if isinstance(x, Act) else ops.from_ncdhw(x, pitch=ops._round_up(x.shape[1], 8))
        if (a.T, a.H, a.W) != (1, 7, 7):
            raise ValueError("SENet.avg_pool is AvgPool2d(7, stride=1): it needs a 7x7 final map (224x224 inputs), got %dx%d"
                             % (a.H, a.W))
        return engine.run_head(self, a, self.last_linear)

    def forward(self, x):
        return self.logits(self.features_act(x))


def _factory(name, block, layers, groups, doc):
    def build(num_classes=1000, pretrained='imagenet'):
        model = SENet(block, layers, groups=groups, reduction=16, dropout_p=None, inplanes=64, input_3x3=False,
                      downsample_kernel_size=1, downsample_padding=0, num_classes=num_classes)
        if pretrained is not None:
            settings = pretrained_settings[name][pretrained]
            assert num_classes == settings['num_classes'], \
                'num_classes should be {}, but is {}'.format(settings['num_classes'], num_classes)
            import torch.utils.model_zoo as model_zoo
            model.load_state_dict(model_zoo.load_url(settings['url']))
            _attach_settings(model, settings)
        return model

    build.__name__ = name
    build.__doc__ = doc
    return build


se_resnet50 = _factory('se_resnet50', SEResNetBottleneck, [3, 4, 6, 3], 1, "senet.py:390-398")
se_resnet101 = _factory('se_resnet101', SEResNetBottleneck, [3, 4, 23, 3], 1, "senet.py:401-409")
se_resnet152 = _factory('se_resnet152', SEResNetBottleneck, [3, 8, 36, 3], 1, "senet.py:412-420")
se_resnext50_32x4d = _factory('se_resnext50_32x4d', SEResNeXtBottleneck, [3, 4, 6, 3], 32, "senet.py:423-431")
se_resnext101_32x4d = _factory('se_resnext101_32x4d', SEResNeXtBottleneck, [3, 4, 23, 3], 32, "senet.py:434-442")
