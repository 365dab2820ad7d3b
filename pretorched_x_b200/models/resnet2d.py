"""2-D ResNets behind the reference's wrapper API (reference: pretorched/models/torchvision_models.py).

The reference builds ``torchvision.models.resnetXX`` and then ``modify_resnets`` renames ``fc`` to
``last_linear`` and patches ``features / logits / forward`` (torchvision_models.py:443-492).  Here the
parameters still come from torchvision's constructor (same tensors, same init), but the three methods run
on the engine: a 2-D image is a clip with T = 1, so the stem / 3x3 / 1x1 convolutions are the same
implicit-GEMM kernel as the video models (BASELINE.json config #1, examples/imagenet_logits.py).
"""
import torch.nn as nn
import torchvision.models.resnet as tvresnet

from .. import engine, ops
from ..ops import Act
from .resnet3d import FineTunable, _attach_settings

__all__ = ['ResNet2D', 'resnet18', 'resnet34', 'resnet50', 'resnet101', 'resnet152']

_URLS = {
    'resnet18': 'https://download.pytorch.org/models/resnet18-5c106cde.pth',
    'resnet34': 'https://download.pytorch.org/models/resnet34-333f7ec4.pth',
    'resnet50': 'https://download.pytorch.org/models/resnet50-19c8e357.pth',
    'resnet101': 'https://download.pytorch.org/models/resnet101-5d3b4d8f.pth',
    'resnet152': 'https://download.pytorch.org/models/resnet152-b121ed2d.pth',
}


def _row(url, num_classes):
    return {'url': url, 'input_space': 'RGB', 'input_size': [3, 224, 224], 'input_range': [0, 1],
            'mean': [0.485, 0.456, 0.406], 'std': [0.229, 0.224, 0.225], 'num_classes': num_classes}


pretrained_settings = {name: {'imagenet': _row(url, 1000)} for name, url in _URLS.items()}
pretrained_settings['resnet50']['moments'] = _row('http://moments.csail.mit.edu/moments_models/resnet50_moments-fd0c4436.pth', 339)
pretrained_settings['resnet18']['places365'] = _row('http://pretorched-x.csail.mit.edu/models/resnet18_places365-dbad67aa.pth', 365)
pretrained_settings['resnet50']['places365'] = _row('http://pretorched-x.csail.mit.edu/models/resnet50_places365-a570fcfc.pth', 365)


class ResNet2D(engine.CacheOwner, FineTunable, tvresnet.ResNet):
    """torchvision ResNet parameters + engine forward; ``last_linear`` replaces ``fc``.

    ``fine_tune(k)`` trains ``layer{k}..layer4`` and ``last_linear`` on the engine, with the contract of
    ``ResNet3D.fine_tune`` (frozen BatchNorm, model in ``eval()``, 1 <= k <= 5)."""

    stem_desc = '7x7 convolution'

    def __init__(self, block, layers, num_classes=1000):
        super().__init__(block, layers, num_classes=num_classes)
        self.last_linear = self.fc
        self.fc = None
        self._register_load_state_dict_pre_hook(self._accept_fc_keys)

    @staticmethod
    def _accept_fc_keys(state_dict, prefix, *args):
        for leaf in ('weight', 'bias'):
            src, dst = prefix + 'fc.' + leaf, prefix + 'last_linear.' + leaf
            if src in state_dict and dst not in state_dict:
                state_dict[dst] = state_dict.pop(src)

    def features(self, input):
        self._refuse_features_in_fine_tune_mode()
        return ops.to_ncdhw(self.features_act(input)).squeeze(2)

    def logits(self, features):
        a = features if isinstance(features, Act) else ops.from_ncdhw(features, pitch=ops._round_up(features.shape[1], 8))
        return engine.run_head(self, a, self.last_linear)

    def forward(self, input):
        return self.logits(self.features_act(input))


_SPECS = {
    'resnet18': (tvresnet.BasicBlock, [2, 2, 2, 2]),
    'resnet34': (tvresnet.BasicBlock, [3, 4, 6, 3]),
    'resnet50': (tvresnet.Bottleneck, [3, 4, 6, 3]),
    'resnet101': (tvresnet.Bottleneck, [3, 4, 23, 3]),
    'resnet152': (tvresnet.Bottleneck, [3, 8, 36, 3]),
}


def _factory(name):
    block, layers = _SPECS[name]

    def build(num_classes=1000, pretrained='imagenet'):
        model = ResNet2D(block, layers, num_classes=num_classes)
        if pretrained is not None:
            settings = pretrained_settings[name][pretrained]
            assert num_classes == settings['num_classes'], \
                "num_classes should be {}, but is {}".format(settings['num_classes'], num_classes)
            import torch.utils.model_zoo as model_zoo
            model.load_state_dict(model_zoo.load_url(settings['url']))
            _attach_settings(model, settings)
        return model

    build.__name__ = name
    build.__doc__ = "Constructs a %s (torchvision_models.py:484-532)." % name
    return build


resnet18, resnet34, resnet50, resnet101, resnet152 = (_factory(n) for n in _SPECS)
