"""CPU restatement of the reference's PolyNet forward (pretorched/models/polynet.py) -- TEST INFRASTRUCTURE.

Plain functional torch over a ``state_dict``, like oracle/inception.py, walking the rows of models.polynet.BRANCHES in the
reference's concatenation order for the stem, the reductions and the blocks of a 2-way module, and restating the poly-3 loop
(polynet.py:258-277).  Each unit's stride / padding is read from the module it restates.  Pinned bit for bit against the
unmodified reference by oracle/make_golden_polynet.py.  Works in the dtype of its inputs (fp32 for the fixtures, fp64 for the
block tests).
"""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F

BN_EPS = 1e-5
STAGES = ['stem', 'stage_a', 'reduction_a', 'stage_b', 'reduction_b', 'stage_c']


def rescale_(model, close=0.5):
    """Weights that make a fixture able to tell a wrong branch from a right one, applied after the seeded init (whose digest the
    fixture records first) and before ``oracle.functional.randomize_bn_``:

    * every Conv2d weight times sqrt(6): PyTorch's default init has std 1 / sqrt(3 fan_in), which with ReLU shrinks the
      activations about 2.4x per layer -- at seed 0 the stem's output stays below 0.09 and the 20 stage_b modules move their input
      by under 1 %.  Times sqrt(6) it is He's sqrt(2 / fan_in), which keeps their scale through a chain;
    * the residual branches' closing 1x1 convolutions (``conv2d`` of BlockA / B / C, ``conv2d_blocks``) a further ``close``, so
      that each module's scaled branch sum is a sizeable fraction of its input while 40 modules of residual growth stay well
      inside fp16's range (``module_report`` measures both)."""
    with torch.no_grad():
        for name, m in model.named_modules():
            if isinstance(m, nn.Conv2d):
                f = math.sqrt(6.0)
                if '.conv2d.' in name + '.' or '.conv2d_blocks.' in name:
                    f *= close
                m.weight.mul_(f)
    return model


def unit(x, sd, p, conv, relu=True, bn=None):
    """conv (no bias) -> eval-mode BatchNorm2d (eps 1e-5; ``bn``: its state_dict prefix, ``p + 'bn.'`` by default) -> ReLU."""
    bn = p + 'bn.' if bn is None else bn
    h = F.conv2d(x, sd[p + 'conv.weight'], None, conv.stride, conv.padding)
    h = F.batch_norm(h, sd[bn + 'running_mean'], sd[bn + 'running_var'], sd[bn + 'weight'], sd[bn + 'bias'], False, 0.0, BN_EPS)
    return F.relu(h) if relu else h


def branches(x, sd, mod, prefix, row):
    """The concatenation of one row of models.polynet.BRANCHES (``mod``: the package's container, ``prefix``: its state_dict
    prefix with the trailing dot)."""
    u = lambda h, path: unit(h, sd, prefix + path + '.', mod.get_submodule(path).conv)
    outs = []
    for br in row:
        if br[0] == 'max':
            outs.append(F.max_pool2d(x, kernel_size=3, stride=2))
        else:
            h = x
            for p in br[1]:
                h = u(h, p)
            outs.append(h)
    return torch.cat(outs, 1)


def stem(x, sd, mod, prefix='stem.'):
    from pretorched_x_b200.models.polynet import BRANCHES
    for i, c in enumerate(mod.conv1):
        x = unit(x, sd, prefix + 'conv1.%d.' % i, c.conv)
    for k in ('Stem1', 'Stem2', 'Stem3'):
        x = branches(x, sd, mod, prefix, BRANCHES[k])
    return x


def block_branch(x, sd, blk, prefix):
    """One half of a 2-way module before its scale: conv2d(cat) with its BatchNorm and no ReLU (BlockA / B / C.forward)."""
    from pretorched_x_b200.models.polynet import BRANCHES
    h = branches(x, sd, blk, prefix, BRANCHES[type(blk).__name__])
    return unit(h, sd, prefix + 'conv2d.', blk.conv2d.conv, relu=False)


def multiway(x, sd, mod, prefix):
    """MultiWay.forward (polynet.py:338-344)."""
    out = x
    for i, blk in enumerate(mod.blocks):
        out = out + block_branch(x, sd, blk, prefix + 'blocks.%d.' % i) * mod.scale
    return F.relu(out)


def poly_application(x, sd, mod, prefix, i):
    """forward_block(x, i) of InceptionResNetB/CPoly (polynet.py:258-267): f_i before its ReLU."""
    from pretorched_x_b200.models.polynet import BRANCHES
    outs = []
    for br in BRANCHES[mod.kind]:
        h = x
        for p in br[1]:
            h = unit(h, sd, prefix + p + '.', mod.get_submodule(p).conv, bn=prefix + p + '.bn_blocks.%d.' % i)
        outs.append(h)
    h = torch.cat(outs, 1)
    return unit(h, sd, prefix + 'conv2d_blocks.%d.' % i, mod.conv2d_blocks[i].conv, relu=False)


def poly(x, sd, mod, prefix):
    """InceptionResNetB/CPoly.forward (polynet.py:269-277)."""
    out = x
    for i in range(mod.num_blocks):
        x = poly_application(x, sd, mod, prefix, i)
        out = out + x * mod.scale
        x = F.relu(x)
    return F.relu(out)


def module(x, sd, mod, prefix):
    """One module of PolyNet.modules_in_order()."""
    from pretorched_x_b200.models import polynet as PN
    if isinstance(mod, PN.Stem):
        return stem(x, sd, mod, prefix)
    if isinstance(mod, PN.MultiWay):
        return multiway(x, sd, mod, prefix)
    if isinstance(mod, (PN.InceptionResNetBPoly, PN.InceptionResNetCPoly)):
        return poly(x, sd, mod, prefix)
    return branches(x, sd, mod, prefix, PN.BRANCHES[mod.kind])


def module_names(model):
    """state_dict prefixes (without the dot) of PolyNet.modules_in_order()."""
    return (['stem'] + ['stage_a.%d' % i for i in range(len(model.stage_a))] + ['reduction_a']
            + ['stage_b.%d' % i for i in range(len(model.stage_b))] + ['reduction_b'] + ['stage_c.%d' % i for i in range(len(model.stage_c))])


def features(x, sd, model, stages=None):
    """stem .. stage_c; ``model``: a package PolyNet (module geometry only).  ``stages`` receives every module's output."""
    h = x
    for name in module_names(model):
        h = module(h, sd, model.get_submodule(name), name + '.')
        if stages is not None:
            stages[name] = h
    return h


def logits(h, sd):
    """AvgPool2d(9, stride=1) -> dropout (eval: identity) -> view -> last_linear (polynet.py:449-454)."""
    h = F.avg_pool2d(h, kernel_size=9, stride=1)
    return F.linear(h.view(h.size(0), -1), sd['last_linear.weight'], sd['last_linear.bias'])


def forward(x, sd, model, stages=None):
    return logits(features(x, sd, model, stages), sd)


def module_report(x, sd, model):
    """Per residual module: (name, |scaled branch sum| / |input| in the L2 norm, max |activation| of its output), and the
    largest activation anywhere in the trunk -- what ``rescale_`` is tuned by."""
    from pretorched_x_b200.models import polynet as PN
    rows, h, peak = [], x, 0.0
    for name in module_names(model):
        mod = model.get_submodule(name)
        p = name + '.'
        if isinstance(mod, PN.MultiWay):
            br = sum(block_branch(h, sd, b, p + 'blocks.%d.' % i) * mod.scale for i, b in enumerate(mod.blocks))
            out = F.relu(h + br)
        elif isinstance(mod, (PN.InceptionResNetBPoly, PN.InceptionResNetCPoly)):
            xi, br = h, 0
            for i in range(mod.num_blocks):
                f = poly_application(xi, sd, mod, p, i)
                br, xi = br + f * mod.scale, F.relu(f)
                peak = max(peak, float(f.abs().max()))
            out = F.relu(h + br)
        else:
            h = module(h, sd, mod, p)
            peak = max(peak, float(h.abs().max()))
            continue
        rows.append((name, float(br.norm() / h.norm()), float(out.abs().max())))
        peak = max(peak, float((h + br).abs().max()))
        h = out
    return rows, peak


def build_package_model(pkg, fx):
    """The package-under-test's model for a PolyNet fixture: same constructor call, seeds and weight scaling as
    oracle/make_golden_polynet.py applied to the reference."""
    from oracle import functional as OF
    torch.manual_seed(fx["seeds"]["init"])
    if fx["kind"] == "trn_inception":
        m = pkg.TRN(10, num_segments=fx["segments"], arch=fx["arch"], consensus="MSTRN", pretrained=None, **fx["kwargs"])
    else:
        m = pkg.__dict__[fx["arch"]](pretrained=None, **fx["kwargs"])
    rescale_(m, fx["close"])
    OF.randomize_bn_(m, fx["seeds"]["bn"])
    return m.eval()
