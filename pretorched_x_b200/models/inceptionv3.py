"""Inception-v3 behind the reference's wrapper API (reference: pretorched/models/torchvision_models.py:380-437).

The reference builds ``torchvision.models.inception_v3(pretrained=False)``, renames ``fc`` to ``last_linear`` and binds its own
``features / logits / forward``.  Here the parameters still come from torchvision's ``Inception3`` constructor (same keys, order
and seeded init; the blocks are torchvision's InceptionA-E classes, subclassed only to carry their row of
models.inception.BRANCHES), and the forward runs on the engine (engine.run_inception_trunk), exactly as Inception-v4's:

* the stem (Conv2d_1a_3x3 .. maxpool2) is Inception-ResNet-v2's stem, unit for unit;
* every block is one ``functions.frozen`` call whose branches write their columns of the concatenated output in place: the 1x1
  units that read the block input as one split GEMM, every convolution with taps (3x3, 5x5, 1x7 / 7x1, 1x3 / 3x1) on the slab
  kernel's slice entry, the average-pool branches (F.avg_pool2d(3, 1, 1), padding counted) as a slice pool into a matrix that
  ``branch_pool`` reads, the max-pool branches (F.max_pool2d(3, 2)) as a slice pool into the pass-through columns;
* the head is the 8x8 global mean and ``last_linear`` (models.inception._final_pool).

``AuxLogits`` stays in the ``state_dict`` and never runs: the reference computes it only in training, and the engine is
inference-only.  ``transform_input`` is not applied, as the reference's ``features`` bypasses it.  The trunk is frozen,
``last_linear`` is trainable on engine features; there is no ``fine_tune``.  Inputs must be 299x299.
"""
import torchvision.models.inception as tvinception

from .. import engine, ops
from .inception import _final_pool
from .resnet3d import _attach_settings

__all__ = ['Inception3', 'inceptionv3']

# torchvision_models.py:39, 74-92
pretrained_settings = {
    'inceptionv3': {'imagenet': {'url': 'https://download.pytorch.org/models/inception_v3_google-1a9a5a14.pth', 'input_space': 'RGB',
                                 'input_size': [3, 299, 299], 'input_range': [0, 1], 'mean': [0.5, 0.5, 0.5],
                                 'std': [0.5, 0.5, 0.5], 'num_classes': 1000}},
}


class InceptionA(engine.CacheOwner, tvinception.InceptionA):
    kind = 'InceptionA'


class InceptionB(engine.CacheOwner, tvinception.InceptionB):
    kind = 'InceptionB'


class InceptionC(engine.CacheOwner, tvinception.InceptionC):
    kind = 'InceptionC'


class InceptionD(engine.CacheOwner, tvinception.InceptionD):
    kind = 'InceptionD'


class InceptionE(engine.CacheOwner, tvinception.InceptionE):
    kind = 'InceptionE'


class Inception3(engine.CacheOwner, tvinception.Inception3):
    """torchvision's Inception3 parameters (1000 classes, AuxLogits kept, no transform_input, torchvision's weight init) and the
    engine forward; ``last_linear`` replaces ``fc`` (torchvision_models.py:384-392)."""

    def __init__(self):
        super().__init__(num_classes=1000, aux_logits=True, transform_input=False, init_weights=True,
                         inception_blocks=[tvinception.BasicConv2d, InceptionA, InceptionB, InceptionC, InceptionD, InceptionE,
                                           tvinception.InceptionAux])
        self.last_linear = self.fc
        del self.fc

    def _units(self):
        stem = [self.Conv2d_1a_3x3, self.Conv2d_2a_3x3, self.Conv2d_2b_3x3, self.maxpool1, self.Conv2d_3b_1x1, self.Conv2d_4a_3x3,
                self.maxpool2]
        return stem, [self.Mixed_5b, self.Mixed_5c, self.Mixed_5d, self.Mixed_6a, self.Mixed_6b, self.Mixed_6c, self.Mixed_6d,
                      self.Mixed_6e, self.Mixed_7a, self.Mixed_7b, self.Mixed_7c]

    def features_act(self, x):
        """The trunk on the engine's native layout (fp16 NDHWC ``Act``)."""
        if self.training:
            raise RuntimeError("the forward engine is inference-only: call model.eval() first")
        stem, blocks = self._units()
        return engine.run_inception_trunk(len(stem), stem + blocks, x)

    def features(self, input):
        """Conv2d_1a_3x3 .. Mixed_7c (torchvision_models.py:396-419): fp32 NCHW [B, 2048, 8, 8] for 299x299 inputs."""
        return ops.to_ncdhw(self.features_act(input)).squeeze(2)

    def logits(self, features):
        """F.avg_pool2d(8) -> dropout (identity in eval) -> view -> last_linear (torchvision_models.py:421-430)."""
        return _final_pool(self, features)

    def forward(self, input):
        return self.logits(self.features_act(input))


def _head_keys(state_dict):
    """torchvision's zoo layout names the head ``fc``; the reference's own ``state_dict`` names it ``last_linear``.  Only the
    top-level ``fc.`` prefix is renamed: ``AuxLogits.fc.*`` keeps its name."""
    return {('last_linear.' + k[3:] if k.startswith('fc.') else k): v for k, v in state_dict.items()}


def inceptionv3(num_classes=1000, pretrained='imagenet'):
    """torchvision_models.py:380-437.  As in the reference, ``pretrained=None`` ignores ``num_classes`` and builds the 1000-class
    head; ``'imagenet'`` asserts ``num_classes == 1000``, loads the checkpoint and attaches the preprocessing attributes."""
    model = Inception3()
    if pretrained is not None:
        settings = pretrained_settings['inceptionv3'][pretrained]
        assert num_classes == settings['num_classes'], \
            "num_classes should be {}, but is {}".format(settings['num_classes'], num_classes)
        import torch.utils.model_zoo as model_zoo
        model.load_state_dict(_head_keys(model_zoo.load_url(settings['url'])))
        _attach_settings(model, settings)
    return model
