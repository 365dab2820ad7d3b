"""Xception (reference: pretorched/models/xception.py; Chollet, "Xception: Deep Learning with Depthwise Separable Convolutions").

The modules keep the reference's names, ``state_dict`` keys, key order and seeded init: every convolution and BatchNorm is built
in the reference's construction order, a block's ``skip`` / ``skipbn`` before its ``rep``, and ``rep`` has the reference's indices,
the parameter-free ReLU and MaxPool2d slots included (``start_with_relu=False`` drops block1's leading ReLU).  ``fc`` is
``last_linear`` (xception.py:231-233); checkpoints with ``fc.*`` keys (the zoo file) load as well as the reference's own
``state_dict``.

The forward runs on the engine (engine.run_xception_trunk): the stem's two valid 3x3 convolutions on the slab kernel, every
separable convolution as a depthwise pass (which applies the ReLU that opens it, if one does, to its input:
ops_xception.dwconv3x3_relu_in) followed by the pointwise GEMM with the BatchNorm and the next ReLU or the block's residual in its
epilogue, and the strided blocks' MaxPool2d(3, 2, 1) on the pooling kernel with the skip's projection GEMM adding the pooled tensor.  ``features`` returns bn4's
output before any ReLU; ``logits`` applies the ReLU and the global mean in one pass, then ``last_linear``, so any input of at
least 7x7 works (the reference's pool is adaptive).  The trunk is frozen, ``last_linear`` is trainable on engine features; there is
no ``fine_tune``.
"""
import torch.nn as nn

from .. import engine, ops
from .. import functions as Fn
from ..ops import Act
from .resnet3d import _attach_settings

__all__ = ['Xception', 'xception']

# xception.py:33-47
pretrained_settings = {
    'xception': {
        'imagenet': {
            'url': 'http://pretorched-x.csail.mit.edu/models/xception-b429252d.pth',
            'input_space': 'RGB',
            'input_size': [3, 299, 299],
            'input_range': [0, 1],
            'mean': [0.5, 0.5, 0.5],
            'std': [0.5, 0.5, 0.5],
            'num_classes': 1000,
            'scale': 0.8975,
        }
    }
}


class SeparableConv2d(nn.Module):
    """Depthwise ``conv1`` (groups = in_channels) then the 1x1 ``pointwise`` (xception.py:50-60).  It runs inside its block on the
    engine, with the BatchNorm that follows it."""

    def __init__(self, in_channels, out_channels, kernel_size=1, stride=1, padding=0, dilation=1, bias=False):
        super().__init__()
        self.conv1 = nn.Conv2d(in_channels, in_channels, kernel_size, stride, padding, dilation, groups=in_channels, bias=bias)
        self.pointwise = nn.Conv2d(in_channels, out_channels, 1, 1, 0, 1, 1, bias=bias)

    def forward(self, x):
        raise NotImplementedError("a SeparableConv2d runs inside its Xception block (with the BatchNorm after it) on the engine")


class Block(nn.Module):
    """``reps`` x (ReLU -> SeparableConv2d 3x3 -> BatchNorm2d), MaxPool2d(3, strides, 1) when strided, plus the skip: a 1x1
    convolution (stride ``strides``) + BatchNorm when the width or the map changes, the input itself otherwise (xception.py:63-112).
    The widening happens in the first repetition (``grow_first``) or the last."""

    def __init__(self, in_filters, out_filters, reps, strides=1, start_with_relu=True, grow_first=True):
        super().__init__()
        if out_filters != in_filters or strides != 1:
            self.skip = nn.Conv2d(in_filters, out_filters, 1, stride=strides, bias=False)
            self.skipbn = nn.BatchNorm2d(out_filters)
        else:
            self.skip = None
        self.relu = nn.ReLU(inplace=True)
        if grow_first:
            widths = [(in_filters, out_filters)] + [(out_filters, out_filters)] * (reps - 1)
        else:
            widths = [(in_filters, in_filters)] * (reps - 1) + [(in_filters, out_filters)]
        rep = []
        for cin, cout in widths:
            rep += [self.relu, SeparableConv2d(cin, cout, 3, stride=1, padding=1, bias=False), nn.BatchNorm2d(cout)]
        # the block input is the previous block's residual sum, which the skip reads unchanged: its ReLU is not in place
        rep = [nn.ReLU(inplace=False)] + rep[1:] if start_with_relu else rep[1:]
        if strides != 1:
            rep.append(nn.MaxPool2d(3, strides, 1))
        self.rep = nn.Sequential(*rep)

    def forward(self, x):
        if isinstance(x, Act):
            return Fn.frozen(lambda a, o: engine._xception_block_body(self, a, o), x)
        a = ops.from_ncdhw(x, pitch=ops._round_up(x.shape[1], 8))
        return ops.to_ncdhw(Fn.frozen(lambda a, o: engine._xception_block_body(self, a, o), a)).squeeze(2)


class Xception(engine.CacheOwner, nn.Module):
    """Xception for ImageNet (xception.py:115-210): a 3x3 stride-2 and a 3x3 convolution, 12 blocks (entry flow 1-3, middle flow
    4-11, exit block 12), two separable convolutions (conv3, conv4), ReLU, global mean and ``last_linear``."""

    def __init__(self, num_classes=1000):
        super().__init__()
        self.num_classes = num_classes
        self.conv1 = nn.Conv2d(3, 32, 3, 2, 0, bias=False)
        self.bn1 = nn.BatchNorm2d(32)
        self.relu = nn.ReLU(inplace=True)
        self.conv2 = nn.Conv2d(32, 64, 3, bias=False)
        self.bn2 = nn.BatchNorm2d(64)
        self.block1 = Block(64, 128, 2, 2, start_with_relu=False, grow_first=True)
        self.block2 = Block(128, 256, 2, 2, start_with_relu=True, grow_first=True)
        self.block3 = Block(256, 728, 2, 2, start_with_relu=True, grow_first=True)
        for i in range(4, 12):
            setattr(self, 'block%d' % i, Block(728, 728, 3, 1, start_with_relu=True, grow_first=True))
        self.block12 = Block(728, 1024, 2, 2, start_with_relu=True, grow_first=False)
        self.conv3 = SeparableConv2d(1024, 1536, 3, 1, 1)
        self.bn3 = nn.BatchNorm2d(1536)
        self.conv4 = SeparableConv2d(1536, 2048, 3, 1, 1)
        self.bn4 = nn.BatchNorm2d(2048)
        self.last_linear = nn.Linear(2048, num_classes)
        self._register_load_state_dict_pre_hook(self._accept_fc_keys)

    @staticmethod
    def _accept_fc_keys(state_dict, prefix, *args):
        """The zoo checkpoint was saved before the reference renamed ``fc`` to ``last_linear``."""
        for leaf in ('weight', 'bias'):
            src, dst = prefix + 'fc.' + leaf, prefix + 'last_linear.' + leaf
            if src in state_dict and dst not in state_dict:
                state_dict[dst] = state_dict.pop(src)

    def features_act(self, input):
        """The trunk on the engine's native layout (fp16 NDHWC ``Act``): bn4's output."""
        if self.training:
            raise RuntimeError("the forward engine is inference-only: call model.eval() first")
        return engine.run_xception_trunk(self, input)

    def features(self, input):
        """conv1 .. bn4 (xception.py:163-193): fp32 NCHW [B, 2048, h, w], before the head's ReLU."""
        return ops.to_ncdhw(self.features_act(input)).squeeze(2)

    def logits(self, features):
        """ReLU -> adaptive_avg_pool2d(1) -> view -> last_linear (xception.py:195-202)."""
        a = features if isinstance(features, Act) else ops.from_ncdhw(features, pitch=ops._round_up(features.shape[1], 8))
        return engine.run_xception_head(self, a)

    def forward(self, input):
        return self.logits(self.features_act(input))


def xception(num_classes=1000, pretrained='imagenet'):
    """xception.py:213-233: with ``pretrained``, asserts ``num_classes == 1000``, loads the checkpoint (``fc.*`` keys) and attaches
    the preprocessing attributes."""
    model = Xception(num_classes=num_classes)
    if pretrained:
        settings = pretrained_settings['xception'][pretrained]
        assert num_classes == settings['num_classes'], \
            "num_classes should be {}, but is {}".format(settings['num_classes'], num_classes)
        import torch.utils.model_zoo as model_zoo
        model.load_state_dict(model_zoo.load_url(settings['url']))
        _attach_settings(model, settings)
    return model
