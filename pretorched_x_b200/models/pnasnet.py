"""PNASNet-5-Large (reference: pretorched/models/pnasnet.py; Liu et al., "Progressive Neural Architecture Search"), 331x331 inputs.

The modules keep the reference's names, ``state_dict`` keys (1380), key order and seeded init: every convolution and BatchNorm is
built in the reference's construction order (a cell's ``conv_prev_1x1`` and ``conv_1x1`` before its ``comb_iter_*`` branches, left
before right), with BatchNorm eps 1e-3.  Cadene's checkpoint and the reference's own ``state_dict`` load unchanged.

The forward runs on the engine (engine.run_pnasnet_trunk): conv_0 on the slab kernel; every separable branch as a depthwise pass
of max(x, 0) (ops_pnasnet.dwconv_kxk_relu_in, K = 3 / 5 / 7) followed by the pointwise GEMM with the BatchNorm; each combination's
second operand (a max-pool, another branch, ``x_right`` or a 1x1 convolution) joins as the closing GEMM's residual; ReLU -> 1x1 ->
BatchNorm on the pre-activation GEMM; FactorizedReduction as two offset gathers (ops_pnasnet.gather_offset) and one two-operand
GEMM.  ``features`` returns cell_11's output before any ReLU; ``logits`` applies the ReLU and the 11x11 mean in one pass, then
``last_linear`` (dropout is the identity in eval).  Inputs must be 331x331 (the reference's fixed AvgPool2d(11)).  The trunk is
frozen, ``last_linear`` is trainable on engine features; there is no ``fine_tune``.
"""
from collections import OrderedDict

import torch.nn as nn

from .. import engine, ops
from ..ops import Act
from .resnet3d import _attach_settings

__all__ = ['PNASNet5Large', 'pnasnet5large']

_URL = 'http://data.lip6.fr/cadene/pretrainedmodels/pnasnet5large-bf079911.pth'
# pnasnet.py:9-30
pretrained_settings = {
    'pnasnet5large': {
        name: {'url': _URL, 'input_space': 'RGB', 'input_size': [3, 331, 331], 'input_range': [0, 1], 'mean': [0.5, 0.5, 0.5],
               'std': [0.5, 0.5, 0.5], 'num_classes': classes}
        for name, classes in (('imagenet', 1000), ('imagenet+background', 1001))
    }
}


def _bn(c):
    return nn.BatchNorm2d(c, eps=0.001)


class _OnEngine(nn.Module):
    """A PNASNet part: it runs inside its cell on the engine."""

    def forward(self, *args):
        raise NotImplementedError("a %s runs inside its PNASNet cell on the engine" % type(self).__name__)


class MaxPool(_OnEngine):
    """MaxPool2d(k, stride, padding), after ZeroPad2d((1, 0, 1, 0)) and before a [1:, 1:] crop when ``zero_pad`` (pnasnet.py:33-46)."""

    def __init__(self, kernel_size, stride=1, padding=1, zero_pad=False):
        super().__init__()
        self.zero_pad = nn.ZeroPad2d((1, 0, 1, 0)) if zero_pad else None
        self.pool = nn.MaxPool2d(kernel_size, stride=stride, padding=padding)


class SeparableConv2d(_OnEngine):
    """Depthwise ``depthwise_conv2d`` (groups = in_channels) then the 1x1 ``pointwise_conv2d`` (pnasnet.py:49-64)."""

    def __init__(self, in_channels, out_channels, dw_kernel_size, dw_stride, dw_padding):
        super().__init__()
        self.depthwise_conv2d = nn.Conv2d(in_channels, in_channels, dw_kernel_size, stride=dw_stride, padding=dw_padding,
                                          groups=in_channels, bias=False)
        self.pointwise_conv2d = nn.Conv2d(in_channels, out_channels, 1, bias=False)


class BranchSeparables(_OnEngine):
    """ReLU -> [ZeroPad2d((1, 0, 1, 0))] -> SeparableConv2d (stride) -> [crop] -> BN -> ReLU -> SeparableConv2d -> BN
    (pnasnet.py:67-97).  The middle width is the output width in a stem cell, the input width otherwise."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, stem_cell=False, zero_pad=False):
        super().__init__()
        mid = out_channels if stem_cell else in_channels
        self.zero_pad = nn.ZeroPad2d((1, 0, 1, 0)) if zero_pad else None
        self.relu_1 = nn.ReLU()
        self.separable_1 = SeparableConv2d(in_channels, mid, kernel_size, stride, kernel_size // 2)
        self.bn_sep_1 = _bn(mid)
        self.relu_2 = nn.ReLU()
        self.separable_2 = SeparableConv2d(mid, out_channels, kernel_size, 1, kernel_size // 2)
        self.bn_sep_2 = _bn(out_channels)


class ReluConvBn(_OnEngine):
    """ReLU -> Conv2d(kernel_size, stride, no bias) -> BN (pnasnet.py:100-114)."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1):
        super().__init__()
        self.relu = nn.ReLU()
        self.conv = nn.Conv2d(in_channels, out_channels, kernel_size, stride=stride, bias=False)
        self.bn = _bn(out_channels)


class FactorizedReduction(_OnEngine):
    """ReLU, then two 1x1 convolutions of half the width on x[2i, 2j] (path_1) and x[2i + 1, 2j + 1] (path_2, zero past the far
    edge), concatenated, then ``final_path_bn`` (pnasnet.py:117-146)."""

    def __init__(self, in_channels, out_channels):
        super().__init__()
        self.relu = nn.ReLU()
        self.path_1 = nn.Sequential(OrderedDict([
            ('avgpool', nn.AvgPool2d(1, stride=2, count_include_pad=False)),
            ('conv', nn.Conv2d(in_channels, out_channels // 2, 1, bias=False))]))
        self.path_2 = nn.Sequential(OrderedDict([
            ('pad', nn.ZeroPad2d((0, 1, 0, 1))),
            ('avgpool', nn.AvgPool2d(1, stride=2, count_include_pad=False)),
            ('conv', nn.Conv2d(in_channels, out_channels // 2, 1, bias=False))]))
        self.final_path_bn = _bn(out_channels)


class CellStem0(_OnEngine):
    """The first stem cell (pnasnet.py:181-223): x_right = conv_1x1(x_left); five stride-2 combinations."""

    def __init__(self, in_channels_left, out_channels_left, in_channels_right, out_channels_right):
        super().__init__()
        cl, cr = out_channels_left, out_channels_right
        self.conv_1x1 = ReluConvBn(in_channels_right, cr, 1)
        self.comb_iter_0_left = BranchSeparables(in_channels_left, cl, 5, 2, stem_cell=True)
        self.comb_iter_0_right = nn.Sequential(OrderedDict([
            ('max_pool', MaxPool(3, stride=2)),
            ('conv', nn.Conv2d(in_channels_left, cl, 1, bias=False)),
            ('bn', _bn(cl))]))
        self.comb_iter_1_left = BranchSeparables(cr, cr, 7, 2)
        self.comb_iter_1_right = MaxPool(3, stride=2)
        self.comb_iter_2_left = BranchSeparables(cr, cr, 5, 2)
        self.comb_iter_2_right = BranchSeparables(cr, cr, 3, 2)
        self.comb_iter_3_left = BranchSeparables(cr, cr, 3)
        self.comb_iter_3_right = MaxPool(3, stride=2)
        self.comb_iter_4_left = BranchSeparables(in_channels_right, cr, 3, 2, stem_cell=True)
        self.comb_iter_4_right = ReluConvBn(cr, cr, 1, stride=2)


class Cell(_OnEngine):
    """A normal or reduction cell (pnasnet.py:226-288): x_left = conv_prev_1x1(prev) (a FactorizedReduction when the previous map is
    twice as large), x_right = conv_1x1(x); five combinations at stride 2 (reduction) or 1."""

    def __init__(self, in_channels_left, out_channels_left, in_channels_right, out_channels_right, is_reduction=False,
                 zero_pad=False, match_prev_layer_dimensions=False):
        super().__init__()
        s, cl, cr = (2 if is_reduction else 1), out_channels_left, out_channels_right
        self.match_prev_layer_dimensions = match_prev_layer_dimensions
        self.conv_prev_1x1 = (FactorizedReduction(in_channels_left, cl) if match_prev_layer_dimensions
                              else ReluConvBn(in_channels_left, cl, 1))
        self.conv_1x1 = ReluConvBn(in_channels_right, cr, 1)
        self.comb_iter_0_left = BranchSeparables(cl, cl, 5, s, zero_pad=zero_pad)
        self.comb_iter_0_right = MaxPool(3, stride=s, zero_pad=zero_pad)
        self.comb_iter_1_left = BranchSeparables(cr, cr, 7, s, zero_pad=zero_pad)
        self.comb_iter_1_right = MaxPool(3, stride=s, zero_pad=zero_pad)
        self.comb_iter_2_left = BranchSeparables(cr, cr, 5, s, zero_pad=zero_pad)
        self.comb_iter_2_right = BranchSeparables(cr, cr, 3, s, zero_pad=zero_pad)
        self.comb_iter_3_left = BranchSeparables(cr, cr, 3)
        self.comb_iter_3_right = MaxPool(3, stride=s, zero_pad=zero_pad)
        self.comb_iter_4_left = BranchSeparables(cl, cl, 3, s, zero_pad=zero_pad)
        self.comb_iter_4_right = ReluConvBn(cr, cr, 1, stride=s) if is_reduction else None


# (name, in_left, out_left, in_right, out_right, is_reduction, zero_pad, match_prev_layer_dimensions): pnasnet.py:302-334
CELLS = [
    ('cell_stem_1', 96, 108, 270, 108, True, False, True),
    ('cell_0', 270, 216, 540, 216, False, False, True),
    ('cell_1', 540, 216, 1080, 216, False, False, False),
    ('cell_2', 1080, 216, 1080, 216, False, False, False),
    ('cell_3', 1080, 216, 1080, 216, False, False, False),
    ('cell_4', 1080, 432, 1080, 432, True, True, False),
    ('cell_5', 1080, 432, 2160, 432, False, False, True),
    ('cell_6', 2160, 432, 2160, 432, False, False, False),
    ('cell_7', 2160, 432, 2160, 432, False, False, False),
    ('cell_8', 2160, 864, 2160, 864, True, False, False),
    ('cell_9', 2160, 864, 4320, 864, False, False, True),
    ('cell_10', 4320, 864, 4320, 864, False, False, False),
    ('cell_11', 4320, 864, 4320, 864, False, False, False),
]


class PNASNet5Large(engine.CacheOwner, nn.Module):
    """PNASNet-5-Large for ImageNet (pnasnet.py:291-369): conv_0 (3x3 stride 2, valid) + BN, CellStem0, 13 cells, ReLU, 11x11 mean,
    dropout and ``last_linear``."""

    def __init__(self, num_classes=1001):
        super().__init__()
        self.num_classes = num_classes
        self.conv_0 = nn.Sequential(OrderedDict([('conv', nn.Conv2d(3, 96, 3, stride=2, bias=False)), ('bn', _bn(96))]))
        self.cell_stem_0 = CellStem0(96, 54, 96, 54)
        for name, il, ol, ir, orr, red, zp, match in CELLS:
            setattr(self, name, Cell(il, ol, ir, orr, is_reduction=red, zero_pad=zp, match_prev_layer_dimensions=match))
        self.relu = nn.ReLU()
        self.avg_pool = nn.AvgPool2d(11, stride=1, padding=0)
        self.dropout = nn.Dropout(0.5)
        self.last_linear = nn.Linear(4320, num_classes)

    def features_act(self, input):
        """The trunk on the engine's native layout (fp16 NHWC ``Act``): cell_11's output."""
        if self.training:
            raise RuntimeError("the forward engine is inference-only: call model.eval() first")
        return engine.run_pnasnet_trunk(self, input)

    def features(self, input):
        """conv_0 .. cell_11 (pnasnet.py:340-356): fp32 NCHW [B, 4320, 11, 11], before the head's ReLU."""
        return ops.to_ncdhw(self.features_act(input)).squeeze(2)

    def logits(self, features):
        """ReLU -> AvgPool2d(11) -> view -> dropout -> last_linear (pnasnet.py:358-364)."""
        a = features if isinstance(features, Act) else ops.from_ncdhw(features, pitch=ops._round_up(features.shape[1], 8))
        return engine.run_pnasnet_head(self, a)

    def forward(self, input):
        return self.logits(self.features_act(input))


def pnasnet5large(num_classes=1000, pretrained='imagenet'):
    """pnasnet.py:372-401: with ``pretrained``, asserts ``num_classes`` against the registry row, loads the 1001-class checkpoint
    and, for 'imagenet', drops the background row of ``last_linear``."""
    if not pretrained:
        return PNASNet5Large(num_classes=num_classes)
    settings = pretrained_settings['pnasnet5large'][pretrained]
    assert num_classes == settings['num_classes'], \
        'num_classes should be {}, but is {}'.format(settings['num_classes'], num_classes)
    import torch.utils.model_zoo as model_zoo
    model = PNASNet5Large(num_classes=1001)
    model.load_state_dict(model_zoo.load_url(settings['url']))
    if pretrained == 'imagenet':
        head = nn.Linear(model.last_linear.in_features, 1000)
        head.weight.data = model.last_linear.weight.data[1:]
        head.bias.data = model.last_linear.bias.data[1:]
        model.last_linear = head
    _attach_settings(model, settings)
    return model
