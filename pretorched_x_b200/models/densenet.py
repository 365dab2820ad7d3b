"""DenseNets behind the reference's wrapper API (reference: pretorched/models/torchvision_models.py:254-380).

The reference builds ``torchvision.models.densenetXXX`` and ``modify_densenets`` renames ``classifier`` to ``last_linear`` and
patches ``logits / forward`` onto torchvision's ``DenseNet`` class.  Here the parameters still come from torchvision's constructor
(same keys, order and seeded init), and the forward runs on the engine (engine.run_densenet_trunk):

* every dense block is one fp16 [M][C_final] matrix: the stem's max-pool or the previous transition writes its first columns, and
  each dense layer reads its input columns in place and writes its k new ones -- no concatenation is ever copied;
* a dense layer is two launches: its 1x1 convolution on the pre-activated GEMM (norm1 + ReLU applied to the A operand on chip,
  norm2 + ReLU in the epilogue), and its 3x3 convolution on the slab kernel's slice entry, written into the block matrix;
* a transition is BatchNorm + ReLU + 2x2 average pool in one pass, then its 1x1 convolution on a quarter of the positions;
* the head applies norm5 + ReLU inside the 7x7 mean that feeds ``last_linear``.

Inference only: the trunk is frozen, ``last_linear`` is trainable on engine features; there is no ``fine_tune``.
"""
import re
from collections import OrderedDict

import torchvision.models.densenet as tvdensenet

from .. import engine, ops
from ..ops import Act
from .resnet3d import _attach_settings
from .utils import Trunk

__all__ = ['DenseNet', 'densenet121', 'densenet161', 'densenet169', 'densenet201']

_URLS = {
    'densenet121': 'https://download.pytorch.org/models/densenet121-241335ed.pth',
    'densenet169': 'https://download.pytorch.org/models/densenet169-6f0f7f60.pth',
    'densenet201': 'https://download.pytorch.org/models/densenet201-4c113574.pth',
    'densenet161': 'https://download.pytorch.org/models/densenet161-17b70270.pth',
}


def _row(url, num_classes):
    return {'url': url, 'input_space': 'RGB', 'input_size': [3, 224, 224], 'input_range': [0, 1],
            'mean': [0.485, 0.456, 0.406], 'std': [0.229, 0.224, 0.225], 'num_classes': num_classes}


# torchvision_models.py:80-130
pretrained_settings = {name: {'imagenet': _row(url, 1000)} for name, url in _URLS.items()}
pretrained_settings['densenet161']['places365'] = _row('http://pretorched-x.csail.mit.edu/models/densenet161_places365-62bbf0d4.pth', 365)

# growth rate, block config, initial features (torchvision densenet.py)
_SPECS = {
    'densenet121': (32, (6, 12, 24, 16), 64),
    'densenet161': (48, (6, 12, 36, 24), 96),
    'densenet169': (32, (6, 12, 32, 32), 64),
    'densenet201': (32, (6, 12, 48, 32), 64),
}

# checkpoints written before '.' was disallowed in module names keep 'norm.1', 'conv.2', ... (torchvision_models.py:283-297)
_LEGACY_KEY = re.compile(r'^(.*denselayer\d+\.(?:norm|relu|conv))\.((?:[12])\.(?:weight|bias|running_mean|running_var))$')


class _DenseTrunk(Trunk):
    """``DenseNet.features``: torchvision's Sequential (conv0 .. denseblock4, norm5).  Returns the norm5 output, fp32 NCHW
    [B, C, 7, 7] for 224x224 inputs, with no ReLU, as the reference's ``features``."""

    _model = 'DenseNet'

    def _run(self, x):
        return engine.densenet_norm5(self, self.run_blocks(x))

    def run_blocks(self, x):
        """The last dense block's output before norm5 (an Act): what the head reads."""
        self.check_runnable()
        return engine.run_densenet_trunk(self, x)


class DenseNet(engine.CacheOwner, tvdensenet.DenseNet):
    """torchvision DenseNet parameters + engine forward; ``last_linear`` replaces ``classifier`` (torchvision_models.py:254-274)."""

    def __init__(self, growth_rate, block_config, num_init_features, num_classes=1000):
        super().__init__(growth_rate=growth_rate, block_config=block_config, num_init_features=num_init_features,
                         num_classes=num_classes)
        self.features = _DenseTrunk(OrderedDict(self.features._modules))
        self.last_linear = self.classifier
        del self.classifier

    def logits(self, features):
        """F.relu -> F.avg_pool2d(7, stride=1) -> view -> last_linear on ``features()``'s tensor (torchvision_models.py:261-266);
        the ReLU runs inside the pool.  A final map other than 7x7 raises."""
        a = features if isinstance(features, Act) else ops.from_ncdhw(features, pitch=ops._round_up(features.shape[1], 8))
        return engine.run_densenet_head(self, a)

    def forward(self, input):
        return engine.run_densenet_head(self, self.features.run_blocks(input), self.features.norm5)


def _factory(name):
    growth, blocks, init = _SPECS[name]

    def build(num_classes=1000, pretrained='imagenet'):
        model = DenseNet(growth, blocks, init, num_classes=num_classes)
        if pretrained is not None:
            settings = pretrained_settings[name][pretrained]
            import torch.utils.model_zoo as model_zoo
            state_dict = model_zoo.load_url(settings['url'])
            for key in list(state_dict.keys()):
                res = _LEGACY_KEY.match(key)
                if res:
                    state_dict[res.group(1) + res.group(2)] = state_dict.pop(key)
            for leaf in ('weight', 'bias'):     # the checkpoints name the head as torchvision does
                if 'classifier.' + leaf in state_dict:
                    state_dict['last_linear.' + leaf] = state_dict.pop('classifier.' + leaf)
            model.load_state_dict(state_dict)
            # deviation: the reference's DenseNet factories attach no preprocessing attributes; here they are attached as for
            # every other family, so TRN and data pipelines read them from the model
            _attach_settings(model, settings)
        return model

    build.__name__ = name
    build.__doc__ = "Constructs a %s (torchvision_models.py:280-380)." % name
    return build


densenet121, densenet161, densenet169, densenet201 = (_factory(n) for n in ('densenet121', 'densenet161', 'densenet169', 'densenet201'))
