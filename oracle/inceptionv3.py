"""CPU restatement of the reference's Inception-v3 forward (pretorched/models/torchvision_models.py:380-437 over torchvision's
Inception3 blocks) -- TEST INFRASTRUCTURE.

Plain functional torch over a ``state_dict``, like oracle/inception.py, whose BasicConv2d restatement it reuses, walking the block
rows of models.inception.BRANCHES in torchvision's concatenation order (average pools with the padding counted, as the row says;
max pools functional, 3x3 stride 2).  Pinned bit for bit against the unmodified reference by oracle/make_golden_inceptionv3.py.
Works in the dtype of its inputs (fp32 for the fixtures, fp64 for the block tests).
"""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle.inception import unit

STEM = ['Conv2d_1a_3x3', 'Conv2d_2a_3x3', 'Conv2d_2b_3x3', 'maxpool1', 'Conv2d_3b_1x1', 'Conv2d_4a_3x3', 'maxpool2']
BLOCKS = ['Mixed_5b', 'Mixed_5c', 'Mixed_5d', 'Mixed_6a', 'Mixed_6b', 'Mixed_6c', 'Mixed_6d', 'Mixed_6e', 'Mixed_7a', 'Mixed_7b',
          'Mixed_7c']


def fan_in_scale_(module):
    """Multiply every Conv2d weight by sqrt(2 / fan_in) / 0.1, in place.  torchvision's Inception3 init draws every convolution
    from N(0, 0.1^2) whatever its fan-in, so with BatchNorm statistics near 1 (oracle.functional.randomize_bn_) the activations
    grow about 3x per layer, to ~1e14 at Mixed_7c: past fp16's range, where no trained checkpoint goes.  Rescaled to the
    fan-in-scaled (He) standard deviation, Mixed_7c stays within a few hundred.  Applied by the fixtures and the GPU tests after
    the seeded init (whose digest the fixture records first)."""
    with torch.no_grad():
        for m in module.modules():
            if isinstance(m, nn.Conv2d):
                m.weight.mul_(math.sqrt(2.0 / m.weight[0].numel()) / 0.1)
    return module


def build_package_model(pkg, fx):
    """The package-under-test's model for an Inception-v3 fixture: same constructor call, seeds and weight scaling as
    oracle/make_golden_inceptionv3.py applied to the reference."""
    from oracle import functional as OF
    torch.manual_seed(fx["seeds"]["init"])
    if fx["kind"] == "trn_inception":
        m = pkg.TRN(10, num_segments=fx["segments"], arch=fx["arch"], consensus="MSTRN", pretrained=None, **fx["kwargs"])
    else:
        m = pkg.__dict__[fx["arch"]](pretrained=None, **fx["kwargs"])
    fan_in_scale_(m)
    OF.randomize_bn_(m, fx["seeds"]["bn"])
    return m.eval()


def block(x, sd, mod, prefix):
    """One InceptionA-E block (``mod``: the package's container, ``prefix``: its state_dict prefix with the trailing dot)."""
    from pretorched_x_b200.models.inception import BRANCHES
    u = lambda h, path: unit(h, sd, prefix + path + '.', mod.get_submodule(path).conv)
    outs = []
    for br in BRANCHES[type(mod).kind]:
        if br[0] == 'max':
            outs.append(F.max_pool2d(x, kernel_size=3, stride=2))
        elif br[0] == 'avg':
            outs.append(u(F.avg_pool2d(x, kernel_size=3, stride=1, padding=1, count_include_pad=br[2]), br[1][-1]))
        else:
            h = x
            for p in br[1]:
                h = u(h, p)
            outs.extend([u(h, p) for p in br[2]] if br[0] == 'fork' else [h])
    return torch.cat(outs, 1)


def features(x, sd, model, stages=None):
    """Conv2d_1a_3x3 .. Mixed_7c; ``model``: a package Inception3 (module geometry only).  ``stages`` receives every unit's output."""
    h = x
    for name in STEM + BLOCKS:
        if name.startswith('maxpool'):
            h = F.max_pool2d(h, kernel_size=3, stride=2)
        elif name in STEM:
            h = unit(h, sd, name + '.', model.get_submodule(name).conv)
        else:
            h = block(h, sd, model.get_submodule(name), name + '.')
        if stages is not None:
            stages[name] = h
    return h


def logits(h, sd):
    """F.avg_pool2d(8) -> dropout (eval: identity) -> view -> last_linear (torchvision_models.py:421-430)."""
    h = F.avg_pool2d(h, kernel_size=8)
    return F.linear(h.view(h.size(0), -1), sd['last_linear.weight'], sd['last_linear.bias'])


def forward(x, sd, model, stages=None):
    return logits(features(x, sd, model, stages), sd)
