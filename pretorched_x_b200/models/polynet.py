"""PolyNet (reference: pretorched/models/polynet.py, Cadene's ``polynet-f71d82a5.pth``, 331x331 inputs).

The modules are parameter containers created under the reference's names and in its order, so the ``state_dict`` keys (3104),
their order and a seeded random init are the reference's and its checkpoint loads unchanged.  The forward runs on the engine
(engine.run_polynet_trunk), one ``functions.frozen`` call per module, on the Inception block path of models/inception.py:

* the stem and the two reductions are rows of ``BRANCHES`` below, walked by engine._inception_block_body: their 1x1 heads as
  one split GEMM, every convolution with taps on the slab kernel's slice entry, the max pools into their pass-through columns;
* a 2-way module (``MultiWay``: out = relu(x + s * A(x) + s * B(x))) runs the branches of both blocks into two concatenation
  matrices and closes with ONE two-operand GEMM: both closing BatchNorm scales, times s, are folded into the fp16 filters, so
  x + s * A(x) never reaches HBM;
* a poly-3 module (out = x; for i in 0..2: f = F_i(x_i); out += s * f; x_{i+1} = relu(f); relu(out)) applies the same filters
  three times with a different BatchNorm each time.  Each application closes with the dual GEMM (b2_gemm_dual_f16): from one
  accumulator it writes the running sum out + s * f and relu(f), the next application's input; the last application is the
  plain residual GEMM with ReLU.  The shared filters are packed once; only the folded BatchNorm differs per application.

``BasicConv2d`` is conv (no bias) -> BatchNorm2d (eps 1e-5, the reference's default) -> ReLU (none on the closing 1x1s).
Inference only: the trunk is frozen, ``last_linear`` is trainable on engine features; there is no ``fine_tune``.  The final
pool is the reference's fixed AvgPool2d(9): inputs must be 331x331.
"""
import torch.nn as nn

from .. import engine, ops
from ..ops import Act
from .resnet3d import _attach_settings

__all__ = ['PolyNet', 'polynet']

# polynet.py:8-21
pretrained_settings = {
    'polynet': {
        'imagenet': {
            'url': 'http://data.lip6.fr/cadene/pretrainedmodels/polynet-f71d82a5.pth',
            'input_space': 'RGB',
            'input_size': [3, 331, 331],
            'input_range': [0, 1],
            'mean': [0.485, 0.456, 0.406],
            'std': [0.229, 0.224, 0.225],
            'num_classes': 1000
        },
    }
}

# Blocks as data, in the format of models.inception.BRANCHES (see there), in the reference's concatenation order.  The stem is
# three concatenations of one module (polynet.py:91-105): the pool branch comes first in both stride-2 stages, and conv2_long is
# (7, 1) before (1, 7) -- the reverse of Inception-v4's Mixed_4a.  The Block rows are the branches of one half of a 2-way
# module; its closing ``conv2d`` (1x1 + BatchNorm, no ReLU) is the module's two-operand GEMM.  The Poly rows are one application
# of a poly-3 module (its PolyConv2d units with BatchNorm ``bn_blocks[i]``), closed by ``conv2d_blocks[i]``.
BRANCHES = {
    'Stem1': [('max', 'conv1_pool_branch'), ('chain', ['conv1_branch'])],
    'Stem2': [('chain', ['conv2_short.0', 'conv2_short.1']),
              ('chain', ['conv2_long.0', 'conv2_long.1', 'conv2_long.2', 'conv2_long.3'])],
    'Stem3': [('max', 'conv2_pool_branch'), ('chain', ['conv2_branch'])],
    'BlockA': [('chain', ['path0.0', 'path0.1', 'path0.2']), ('chain', ['path1.0', 'path1.1']), ('chain', ['path2'])],
    'BlockB': [('chain', ['path0.0', 'path0.1', 'path0.2']), ('chain', ['path1'])],
    'BlockC': [('chain', ['path0.0', 'path0.1', 'path0.2']), ('chain', ['path1'])],
    'ReductionA': [('chain', ['path0.0', 'path0.1', 'path0.2']), ('chain', ['path1']), ('max', 'path2')],
    'ReductionB': [('chain', ['path0.0', 'path0.1', 'path0.2']), ('chain', ['path1.0', 'path1.1']),
                   ('chain', ['path2.0', 'path2.1']), ('max', 'path3')],
    'PolyB': [('chain', ['path0_1x1', 'path0_1x7', 'path0_7x1']), ('chain', ['path1'])],
    'PolyC': [('chain', ['path0_1x1', 'path0_1x3', 'path0_3x1']), ('chain', ['path1'])],
}


class BasicConv2d(nn.Module):
    """conv (no bias) -> BatchNorm2d -> ReLU (none when ``output_relu`` is False) (polynet.py:24-41)."""

    def __init__(self, in_planes, out_planes, kernel_size, stride=1, padding=0, output_relu=True):
        super().__init__()
        self.conv = nn.Conv2d(in_planes, out_planes, kernel_size=kernel_size, stride=stride, padding=padding, bias=False)
        self.bn = nn.BatchNorm2d(out_planes)
        self.relu = nn.ReLU() if output_relu else None


class PolyConv2d(nn.Module):
    """A convolution shared by the applications of a poly-N module, with one BatchNorm per application (polynet.py:44-68)."""

    def __init__(self, in_planes, out_planes, kernel_size, num_blocks, stride=1, padding=0):
        super().__init__()
        self.conv = nn.Conv2d(in_planes, out_planes, kernel_size=kernel_size, stride=stride, padding=padding, bias=False)
        self.bn_blocks = nn.ModuleList([nn.BatchNorm2d(out_planes) for _ in range(num_blocks)])
        self.relu = nn.ReLU()


class _Module(engine.CacheOwner, nn.Module):
    pass


class Stem(_Module):
    """polynet.py:71-106."""

    def __init__(self):
        super().__init__()
        self.conv1 = nn.Sequential(BasicConv2d(3, 32, kernel_size=3, stride=2), BasicConv2d(32, 32, kernel_size=3),
                                   BasicConv2d(32, 64, kernel_size=3, padding=1))
        self.conv1_pool_branch = nn.MaxPool2d(3, stride=2)
        self.conv1_branch = BasicConv2d(64, 96, kernel_size=3, stride=2)
        self.conv2_short = nn.Sequential(BasicConv2d(160, 64, kernel_size=1), BasicConv2d(64, 96, kernel_size=3))
        self.conv2_long = nn.Sequential(BasicConv2d(160, 64, kernel_size=1), BasicConv2d(64, 64, kernel_size=(7, 1), padding=(3, 0)),
                                        BasicConv2d(64, 64, kernel_size=(1, 7), padding=(0, 3)), BasicConv2d(64, 96, kernel_size=3))
        self.conv2_pool_branch = nn.MaxPool2d(3, stride=2)
        self.conv2_branch = BasicConv2d(192, 192, kernel_size=3, stride=2)


class BlockA(_Module):
    """Inception-ResNet-A block (polynet.py:109-131)."""

    def __init__(self):
        super().__init__()
        self.path0 = nn.Sequential(BasicConv2d(384, 32, kernel_size=1), BasicConv2d(32, 48, kernel_size=3, padding=1),
                                   BasicConv2d(48, 64, kernel_size=3, padding=1))
        self.path1 = nn.Sequential(BasicConv2d(384, 32, kernel_size=1), BasicConv2d(32, 32, kernel_size=3, padding=1))
        self.path2 = BasicConv2d(384, 32, kernel_size=1)
        self.conv2d = BasicConv2d(128, 384, kernel_size=1, output_relu=False)


class BlockB(_Module):
    """Inception-ResNet-B block (polynet.py:134-151)."""

    def __init__(self):
        super().__init__()
        self.path0 = nn.Sequential(BasicConv2d(1152, 128, kernel_size=1), BasicConv2d(128, 160, kernel_size=(1, 7), padding=(0, 3)),
                                   BasicConv2d(160, 192, kernel_size=(7, 1), padding=(3, 0)))
        self.path1 = BasicConv2d(1152, 192, kernel_size=1)
        self.conv2d = BasicConv2d(384, 1152, kernel_size=1, output_relu=False)


class BlockC(_Module):
    """Inception-ResNet-C block (polynet.py:154-171)."""

    def __init__(self):
        super().__init__()
        self.path0 = nn.Sequential(BasicConv2d(2048, 192, kernel_size=1), BasicConv2d(192, 224, kernel_size=(1, 3), padding=(0, 1)),
                                   BasicConv2d(224, 256, kernel_size=(3, 1), padding=(1, 0)))
        self.path1 = BasicConv2d(2048, 192, kernel_size=1)
        self.conv2d = BasicConv2d(448, 2048, kernel_size=1, output_relu=False)


class ReductionA(_Module):
    """polynet.py:174-196."""
    kind = 'ReductionA'

    def __init__(self):
        super().__init__()
        self.path0 = nn.Sequential(BasicConv2d(384, 256, kernel_size=1), BasicConv2d(256, 256, kernel_size=3, padding=1),
                                   BasicConv2d(256, 384, kernel_size=3, stride=2))
        self.path1 = BasicConv2d(384, 384, kernel_size=3, stride=2)
        self.path2 = nn.MaxPool2d(3, stride=2)


class ReductionB(_Module):
    """polynet.py:199-228."""
    kind = 'ReductionB'

    def __init__(self):
        super().__init__()
        self.path0 = nn.Sequential(BasicConv2d(1152, 256, kernel_size=1), BasicConv2d(256, 256, kernel_size=3, padding=1),
                                   BasicConv2d(256, 256, kernel_size=3, stride=2))
        self.path1 = nn.Sequential(BasicConv2d(1152, 256, kernel_size=1), BasicConv2d(256, 256, kernel_size=3, stride=2))
        self.path2 = nn.Sequential(BasicConv2d(1152, 256, kernel_size=1), BasicConv2d(256, 384, kernel_size=3, stride=2))
        self.path3 = nn.MaxPool2d(3, stride=2)


class InceptionResNetBPoly(_Module):
    """polynet.py:231-277."""
    kind = 'PolyB'

    def __init__(self, scale, num_blocks):
        super().__init__()
        assert num_blocks >= 1, 'num_blocks should be greater or equal to 1'
        self.scale = scale
        self.num_blocks = num_blocks
        self.path0_1x1 = PolyConv2d(1152, 128, kernel_size=1, num_blocks=self.num_blocks)
        self.path0_1x7 = PolyConv2d(128, 160, kernel_size=(1, 7), num_blocks=self.num_blocks, padding=(0, 3))
        self.path0_7x1 = PolyConv2d(160, 192, kernel_size=(7, 1), num_blocks=self.num_blocks, padding=(3, 0))
        self.path1 = PolyConv2d(1152, 192, kernel_size=1, num_blocks=self.num_blocks)
        self.conv2d_blocks = nn.ModuleList([BasicConv2d(384, 1152, kernel_size=1, output_relu=False) for _ in range(self.num_blocks)])
        self.relu = nn.ReLU()


class InceptionResNetCPoly(_Module):
    """polynet.py:280-326."""
    kind = 'PolyC'

    def __init__(self, scale, num_blocks):
        super().__init__()
        assert num_blocks >= 1, 'num_blocks should be greater or equal to 1'
        self.scale = scale
        self.num_blocks = num_blocks
        self.path0_1x1 = PolyConv2d(2048, 192, kernel_size=1, num_blocks=self.num_blocks)
        self.path0_1x3 = PolyConv2d(192, 224, kernel_size=(1, 3), num_blocks=self.num_blocks, padding=(0, 1))
        self.path0_3x1 = PolyConv2d(224, 256, kernel_size=(3, 1), num_blocks=self.num_blocks, padding=(1, 0))
        self.path1 = PolyConv2d(2048, 192, kernel_size=1, num_blocks=self.num_blocks)
        self.conv2d_blocks = nn.ModuleList([BasicConv2d(448, 2048, kernel_size=1, output_relu=False) for _ in range(self.num_blocks)])
        self.relu = nn.ReLU()


class MultiWay(_Module):
    """N-way module: out = relu(x + sum_b scale * block_b(x)) (polynet.py:329-344)."""

    def __init__(self, scale, block_cls, num_blocks):
        super().__init__()
        assert num_blocks >= 1, 'num_blocks should be greater or equal to 1'
        self.scale = scale
        self.blocks = nn.ModuleList([block_cls() for _ in range(num_blocks)])
        self.relu = nn.ReLU()


class InceptionResNetA2Way(MultiWay):
    def __init__(self, scale):
        super().__init__(scale, block_cls=BlockA, num_blocks=2)


class InceptionResNetB2Way(MultiWay):
    def __init__(self, scale):
        super().__init__(scale, block_cls=BlockB, num_blocks=2)


class InceptionResNetC2Way(MultiWay):
    def __init__(self, scale):
        super().__init__(scale, block_cls=BlockC, num_blocks=2)


class InceptionResNetBPoly3(InceptionResNetBPoly):
    def __init__(self, scale):
        super().__init__(scale, num_blocks=3)


class InceptionResNetCPoly3(InceptionResNetCPoly):
    def __init__(self, scale):
        super().__init__(scale, num_blocks=3)


_A_SCALES = (1, 0.992308, 0.984615, 0.976923, 0.969231, 0.961538, 0.953846, 0.946154, 0.938462, 0.930769)
_B_SCALES = (0.923077, 0.915385, 0.907692, 0.9, 0.892308, 0.884615, 0.876923, 0.869231, 0.861538, 0.853846, 0.846154, 0.838462,
             0.830769, 0.823077, 0.815385, 0.807692, 0.8, 0.792308, 0.784615, 0.776923)
_C_SCALES = (0.769231, 0.761538, 0.753846, 0.746154, 0.738462, 0.730769, 0.723077, 0.715385, 0.707692, 0.7)


class PolyNet(engine.CacheOwner, nn.Module):
    """polynet.py:374-457."""

    def __init__(self, num_classes=1000):
        super().__init__()
        self.stem = Stem()
        self.stage_a = nn.Sequential(*[InceptionResNetA2Way(scale=s) for s in _A_SCALES])
        self.reduction_a = ReductionA()
        self.stage_b = nn.Sequential(*[(InceptionResNetBPoly3 if i % 2 == 0 else InceptionResNetB2Way)(scale=s)
                                       for i, s in enumerate(_B_SCALES)])
        self.reduction_b = ReductionB()
        self.stage_c = nn.Sequential(*[(InceptionResNetCPoly3 if i % 2 == 0 else InceptionResNetC2Way)(scale=s)
                                       for i, s in enumerate(_C_SCALES)])
        self.avg_pool = nn.AvgPool2d(9, stride=1)
        self.dropout = nn.Dropout(0.2)
        self.last_linear = nn.Linear(2048, num_classes)

    def modules_in_order(self):
        """The trunk's modules, each one ``functions.frozen`` call: stem, stage_a, reduction_a, stage_b, reduction_b, stage_c."""
        return [self.stem, *self.stage_a, self.reduction_a, *self.stage_b, self.reduction_b, *self.stage_c]

    def features_act(self, x):
        """The trunk on the engine's native layout (fp16 NDHWC ``Act``)."""
        if self.training:
            raise RuntimeError("the forward engine is inference-only: call model.eval() first")
        return engine.run_polynet_trunk(self, x)

    def features(self, x):
        """stem .. stage_c (polynet.py:440-447): fp32 NCHW [B, 2048, 9, 9] for 331x331 inputs."""
        return ops.to_ncdhw(self.features_act(x)).squeeze(2)

    def logits(self, x):
        """AvgPool2d(9) -> dropout (identity in eval) -> view -> last_linear (polynet.py:449-454).  On the 9x9 map of a 331x331
        input the pool is the global mean; any other final map raises instead of pooling differently."""
        T, H, W = (x.T, x.H, x.W) if isinstance(x, Act) else (1,) + tuple(x.shape[-2:])
        if (T, H, W) != (1, 9, 9):
            raise ValueError("PolyNet's final pool is AvgPool2d(9): it needs a 9x9 final map (331x331 inputs), got %dx%d" % (H, W))
        a = x if isinstance(x, Act) else ops.from_ncdhw(x, pitch=ops._round_up(x.shape[1], 8))
        return engine.run_head(self, a, self.last_linear)

    def forward(self, x):
        return self.logits(self.features_act(x))


def polynet(num_classes=1000, pretrained='imagenet'):
    """polynet.py:460-481: 'PolyNet: A Pursuit of Structural Diversity in Very Deep Networks' (arXiv:1611.05725)."""
    if pretrained:
        settings = pretrained_settings['polynet'][pretrained]
        assert num_classes == settings['num_classes'], \
            'num_classes should be {}, but is {}'.format(settings['num_classes'], num_classes)
        import torch.utils.model_zoo as model_zoo
        model = PolyNet(num_classes=num_classes)
        model.load_state_dict(model_zoo.load_url(settings['url']))
        _attach_settings(model, settings)
    else:
        model = PolyNet(num_classes=num_classes)
    return model
