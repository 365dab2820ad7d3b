"""MobileNetV2 (reference: pretorched/models/mobilenet.py:1-150), pretorched-x's own ImageNet model.

The modules are parameter containers created in the reference's order with the reference's ``_initialize_weights``, so the
``state_dict`` keys, their order and a seeded random init are the reference's.  The forward runs on the engine: the
depthwise 3x3 convolutions on their own CUDA-core kernel (csrc/b2_dwconv.cu), the 1x1 convolutions (with the folded BN and
the residual) on the persistent GEMM, the stem's 3x3 stride-2 convolution on the generic convolution path
(engine.run_mobilenet_features).  ``features`` stays an ``nn.Sequential`` attribute; calling it walks the engine.
"""
import math

import torch.nn as nn

from .. import engine, ops
from ..ops import Act
from .resnet3d import _attach_settings

__all__ = ['MobileNetV2', 'InvertedResidual', 'conv_bn', 'conv_1x1_bn', 'mobilenetv2', 'pretrained_settings']

pretrained_settings = {
    'mobilenetv2': {
        'imagenet': {
            'url': 'http://pretorched-x.csail.mit.edu/models/mobilenetv2-b190fe5f.pth',
            'input_space': 'RGB',
            'input_size': [3, 224, 224],
            'input_range': [0, 1],
            'mean': [0.485, 0.456, 0.406],
            'std': [0.229, 0.224, 0.225],
            'num_classes': 1000
        },
    }
}


def conv_bn(inp, oup, stride):
    return nn.Sequential(
        nn.Conv2d(inp, oup, 3, stride, 1, bias=False),
        nn.BatchNorm2d(oup),
        nn.ReLU6(inplace=True)
    )


def conv_1x1_bn(inp, oup):
    return nn.Sequential(
        nn.Conv2d(inp, oup, 1, 1, 0, bias=False),
        nn.BatchNorm2d(oup),
        nn.ReLU6(inplace=True)
    )


class InvertedResidual(nn.Module):
    """mobilenet.py:38-76; the body runs in engine._inverted_residual_body."""

    def __init__(self, inp, oup, stride, expand_ratio):
        super(InvertedResidual, self).__init__()
        self.stride = stride
        assert stride in [1, 2]

        hidden_dim = round(inp * expand_ratio)
        self.use_res_connect = self.stride == 1 and inp == oup

        if expand_ratio == 1:
            self.conv = nn.Sequential(
                # dw
                nn.Conv2d(hidden_dim, hidden_dim, 3, stride, 1, groups=hidden_dim, bias=False),
                nn.BatchNorm2d(hidden_dim),
                nn.ReLU6(inplace=True),
                # pw-linear
                nn.Conv2d(hidden_dim, oup, 1, 1, 0, bias=False),
                nn.BatchNorm2d(oup),
            )
        else:
            self.conv = nn.Sequential(
                # pw
                nn.Conv2d(inp, hidden_dim, 1, 1, 0, bias=False),
                nn.BatchNorm2d(hidden_dim),
                nn.ReLU6(inplace=True),
                # dw
                nn.Conv2d(hidden_dim, hidden_dim, 3, stride, 1, groups=hidden_dim, bias=False),
                nn.BatchNorm2d(hidden_dim),
                nn.ReLU6(inplace=True),
                # pw-linear
                nn.Conv2d(hidden_dim, oup, 1, 1, 0, bias=False),
                nn.BatchNorm2d(oup),
            )


class MobileNetFeatures(nn.Sequential):
    """``MobileNetV2.features``: the reference's ``nn.Sequential`` (same children, same keys) whose call walks the engine.
    fp32 [B, 3, H, W] in, fp32 [B, last_channel, H/32, W/32] out."""

    def forward(self, x):
        if self.training:
            raise RuntimeError("the forward engine is inference-only: call model.eval() first")
        return ops.to_ncdhw(engine.run_mobilenet_features(self, x)).squeeze(2)


class MobileNetV2(engine.CacheOwner, nn.Module):
    def __init__(self, num_classes=1000, input_size=224, width_mult=1.):
        super(MobileNetV2, self).__init__()
        block = InvertedResidual
        input_channel = 32
        last_channel = 1280
        interverted_residual_setting = [
            # t, c, n, s
            [1, 16, 1, 1],
            [6, 24, 2, 2],
            [6, 32, 3, 2],
            [6, 64, 4, 2],
            [6, 96, 3, 1],
            [6, 160, 3, 2],
            [6, 320, 1, 1],
        ]

        # building first layer
        assert input_size % 32 == 0
        input_channel = int(input_channel * width_mult)
        self.last_channel = int(last_channel * width_mult) if width_mult > 1.0 else last_channel
        self.features = [conv_bn(3, input_channel, 2)]
        # building inverted residual blocks
        for t, c, n, s in interverted_residual_setting:
            output_channel = int(c * width_mult)
            for i in range(n):
                if i == 0:
                    self.features.append(block(input_channel, output_channel, s, expand_ratio=t))
                else:
                    self.features.append(block(input_channel, output_channel, 1, expand_ratio=t))
                input_channel = output_channel
        # building last several layers
        self.features.append(conv_1x1_bn(input_channel, self.last_channel))
        # make it nn.Sequential (whose call runs on the engine)
        self.features = MobileNetFeatures(*self.features)

        # building classifier
        self.dropout = nn.Dropout(0.2)
        self.last_linear = nn.Linear(self.last_channel, num_classes)

        self._initialize_weights()
        widths = sorted({m.out_channels for m in self.features.modules() if isinstance(m, nn.Conv2d)})
        if any(c % 8 for c in widths):
            raise NotImplementedError("the engine needs every channel count to be a multiple of 8; width_mult=%r gives %s"
                                      % (width_mult, [c for c in widths if c % 8]))

    def features_act(self, x):
        if self.training:
            raise RuntimeError("the forward engine is inference-only: call model.eval() first")
        return engine.run_mobilenet_features(self.features, x)

    def logits(self, features):
        """Global average -> dropout (the identity in eval mode) -> ``last_linear`` (mobilenet.py:121-126)."""
        a = features if isinstance(features, Act) else ops.from_ncdhw(features, pitch=ops._round_up(features.shape[1], 8))
        return engine.run_head(self, a, self.last_linear)

    def forward(self, x):
        return self.logits(self.features_act(x))

    def _initialize_weights(self):
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                n = m.kernel_size[0] * m.kernel_size[1] * m.out_channels
                m.weight.data.normal_(0, math.sqrt(2. / n))
                if m.bias is not None:
                    m.bias.data.zero_()
            elif isinstance(m, nn.BatchNorm2d):
                m.weight.data.fill_(1)
                m.bias.data.zero_()
            elif isinstance(m, nn.Linear):
                n = m.weight.size(1)
                m.weight.data.normal_(0, 0.01)
                m.bias.data.zero_()


def mobilenetv2(num_classes=1000, pretrained='imagenet'):
    """Constructs mobilenetv2 model (mobilenet.py:144-150)."""
    model = MobileNetV2(num_classes=num_classes)
    if pretrained is not None:
        settings = pretrained_settings['mobilenetv2'][pretrained]
        assert num_classes == settings['num_classes'], \
            "num_classes should be {}, but is {}".format(settings['num_classes'], num_classes)
        import torch.utils.model_zoo as model_zoo
        model.load_state_dict(model_zoo.load_url(settings['url']))
        _attach_settings(model, settings)
    return model
