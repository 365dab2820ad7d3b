"""VGG and AlexNet behind the reference's wrapper API (reference: pretorched/models/torchvision_models.py:195-248, 597-725).

The reference builds ``torchvision.models.vgg*`` / ``alexnet`` and ``modify_vggs`` / ``modify_alexnet`` move ``features`` to
``_features`` and the classifier's layers to ``linear0 / relu0 / dropout0 / linear1 / relu1 / dropout1 / last_linear``.  Here the
parameters come from torchvision's own constructors (same keys, key order and seeded init) with the same moves, and the forward
runs on the engine:

* the trunk (``_features``) is one Function: every convolution on the convolution path with its bias (or bias + folded BatchNorm)
  and ReLU in the epilogue, the max pools on the pooling kernel; VGG's 3-channel input is stored at pitch 8;
* AlexNet's 11x11 stride-4 conv1 is a valid 3x3 convolution over a 4x4 space-to-depth image of the input
  (``ops_vgg.space_to_depth4``) with the filter zero-padded to 12x12 and regrouped (``ops_vgg.s2d_filter``);
* the classifier reads the last map [N*H*W][C] as [N][H*W*C]: fc6's weight columns are permuted once, at pack time, from the
  reference's (c, h, w) flatten order to (h, w, c), so no transpose runs.  fc6 applies bias + ReLU and writes fp16, fc7 applies
  its bias and writes fp32 -- ``features()``'s tensor; where the output tiles leave SMs idle the GEMMs run split-K
  (``ops_vgg.gemm_splitk``).

Inference only: the trunk and fc6 / fc7 are frozen, ``last_linear`` is trainable on engine features; there is no ``fine_tune``.

Reference behaviour not kept: ``modify_vggs`` / ``modify_alexnet`` patch torchvision's classes for the whole process (here the
methods belong to this module's classes), and the VGG factories ignore ``num_classes`` when ``pretrained=None`` (here it is
honoured).  An input other than 224x224, which breaks the reference's ``view``, raises ``ValueError``.
"""
from collections import OrderedDict

from torchvision.models.alexnet import AlexNet as _TVAlexNet
import torchvision.models.vgg as tvvgg

from .. import engine
from .resnet3d import _attach_settings
from .utils import Trunk

__all__ = ['VGG', 'AlexNet', 'alexnet', 'vgg11', 'vgg11_bn', 'vgg13', 'vgg13_bn', 'vgg16', 'vgg16_bn', 'vgg19', 'vgg19_bn']

_URLS = {
    'alexnet': 'https://download.pytorch.org/models/alexnet-owt-4df8aa71.pth',
    'vgg11': 'https://download.pytorch.org/models/vgg11-bbd30ac9.pth',
    'vgg13': 'https://download.pytorch.org/models/vgg13-c768596a.pth',
    'vgg16': 'https://download.pytorch.org/models/vgg16-397923af.pth',
    'vgg19': 'https://download.pytorch.org/models/vgg19-dcbb9e9d.pth',
    'vgg11_bn': 'https://download.pytorch.org/models/vgg11_bn-6002323d.pth',
    'vgg13_bn': 'https://download.pytorch.org/models/vgg13_bn-abd245e5.pth',
    'vgg16_bn': 'https://download.pytorch.org/models/vgg16_bn-6c64b313.pth',
    'vgg19_bn': 'https://download.pytorch.org/models/vgg19_bn-c79401a0.pth',
}


def _row(url, num_classes):
    return {'url': url, 'input_space': 'RGB', 'input_size': [3, 224, 224], 'input_range': [0, 1],
            'mean': [0.485, 0.456, 0.406], 'std': [0.229, 0.224, 0.225], 'num_classes': num_classes}


# torchvision_models.py:64-119
pretrained_settings = {name: {'imagenet': _row(url, 1000)} for name, url in _URLS.items()}
pretrained_settings['alexnet']['places365'] = _row('http://pretorched-x.csail.mit.edu/models/alexnet_places365-0c3a7b83.pth', 365)

# torchvision's configuration letter of each VGG
_CFG = {'vgg11': 'A', 'vgg13': 'B', 'vgg16': 'D', 'vgg19': 'E'}


class _VGGTrunk(Trunk):
    """``_features``: torchvision's Sequential of 3x3 convolutions (+ BatchNorm), ReLUs and 2x2 max pools.  Returns the last pool's
    output, fp32 NCHW [B, 512, 7, 7] for 224x224 inputs."""

    _model = 'VGG'

    def _run(self, x):
        return engine.run_vgg_trunk(self, x)


class _AlexNetTrunk(Trunk):
    """``_features`` of AlexNet.  Returns the last pool's output, fp32 NCHW [B, 256, 6, 6] for 224x224 inputs."""

    _model = 'AlexNet'

    def _run(self, x):
        return engine.run_alexnet_trunk(self, x)


class _Classifier:
    """``features`` / ``logits`` / ``forward`` of both families (torchvision_models.py:211-229, 613-631)."""

    def features(self, input):
        """_features -> view -> linear0 -> relu0 -> linear1 (dropouts: the identity in eval): fp32 [B, 4096], fc7 before its ReLU."""
        return engine.run_vgg_classifier(self, self._features.run_act(input))

    def logits(self, features):
        """relu1 -> last_linear on ``features()``'s tensor."""
        return engine.run_vgg_logits(self, features)

    def forward(self, input):
        return self.logits(self.features(input))


class VGG(_Classifier, engine.CacheOwner, tvvgg.VGG):
    """torchvision VGG parameters + engine forward, with the reference's module names (torchvision_models.py:600-611)."""

    def __init__(self, cfg, batch_norm, num_classes=1000):
        super().__init__(tvvgg.make_layers(tvvgg.cfgs[cfg], batch_norm=batch_norm), num_classes=num_classes)
        # ``features`` is a method of this class: the Sequential torchvision registered under that name is reached through _modules
        self._features = _VGGTrunk(OrderedDict(self._modules['features']._modules))
        del self._modules['features']
        cls = self.classifier
        self.linear0, self.relu0, self.dropout0 = cls[0], cls[1], cls[2]
        self.linear1, self.relu1, self.dropout1 = cls[3], cls[4], cls[5]
        self.last_linear = cls[6]
        del self.classifier


class AlexNet(_Classifier, engine.CacheOwner, _TVAlexNet):
    """torchvision AlexNet parameters + engine forward, with the reference's module names (torchvision_models.py:198-209)."""

    def __init__(self, num_classes=1000):
        super().__init__(num_classes=num_classes)
        # ``features`` is a method of this class: the Sequential torchvision registered under that name is reached through _modules
        self._features = _AlexNetTrunk(OrderedDict(self._modules['features']._modules))
        del self._modules['features']
        cls = self.classifier
        self.dropout0, self.linear0, self.relu0 = cls[0], cls[1], cls[2]
        self.dropout1, self.linear1, self.relu1 = cls[3], cls[4], cls[5]
        self.last_linear = cls[6]
        del self.classifier


# classifier index -> module name of each family (modify_vggs / modify_alexnet)
_VGG_KEYS = {'0': 'linear0', '3': 'linear1', '6': 'last_linear'}
_ALEXNET_KEYS = {'1': 'linear0', '4': 'linear1', '6': 'last_linear'}


def _rename(state_dict, keys):
    """A checkpoint in torchvision's layout (``features.*``, ``classifier.<i>.*``) -> the reference's (``_features.*``,
    ``linear0.*`` ...); keys already in the reference's layout pass through."""
    out = OrderedDict()
    for k, v in state_dict.items():
        if k.startswith('features.'):
            k = '_' + k
        elif k.startswith('classifier.'):
            idx, leaf = k[len('classifier.'):].split('.', 1)
            k = keys[idx] + '.' + leaf
        out[k] = v
    return out


def _load(model, name, num_classes, pretrained, keys):
    if pretrained is not None:
        settings = pretrained_settings[name][pretrained]
        assert num_classes == settings['num_classes'], \
            "num_classes should be {}, but is {}".format(settings['num_classes'], num_classes)
        import torch.utils.model_zoo as model_zoo
        model.load_state_dict(_rename(model_zoo.load_url(settings['url']), keys))
        _attach_settings(model, settings)
    return model


def _vgg_factory(name):
    cfg, bn = _CFG[name.replace('_bn', '')], name.endswith('_bn')

    def build(num_classes=1000, pretrained='imagenet'):
        return _load(VGG(cfg, bn, num_classes=num_classes), name, num_classes, pretrained, _VGG_KEYS)

    build.__name__ = name
    build.__doc__ = "Constructs a %s (torchvision_models.py:640-725)." % name
    return build


vgg11, vgg11_bn, vgg13, vgg13_bn, vgg16, vgg16_bn, vgg19, vgg19_bn = (
    _vgg_factory(n) for n in ('vgg11', 'vgg11_bn', 'vgg13', 'vgg13_bn', 'vgg16', 'vgg16_bn', 'vgg19', 'vgg19_bn'))


def alexnet(num_classes=1000, pretrained='imagenet'):
    """AlexNet (torchvision_models.py:238-248); ``pretrained='places365'``: the project's Places365 checkpoint, 365 classes."""
    return _load(AlexNet(num_classes=num_classes), 'alexnet', num_classes, pretrained, _ALEXNET_KEYS)
