"""CPU restatement of the reference's ResNeXt-101 32x4d / 64x4d forward (pretorched/models/resnext.py and
resnext_features/resnext101_*_features.py) -- TEST INFRASTRUCTURE.

Plain functional torch over a ``state_dict`` with the reference's positional Torch7 keys; pinned bit for bit against the unmodified
reference by oracle/make_golden_resnext.py.  Works in the dtype of its inputs (fp32 for the fixtures, fp64 for the audits).
"""
import torch
import torch.nn.functional as F

BN_EPS = 1e-5
LAYERS = (3, 4, 23, 3)
# name -> groups: conv2 widths groups * 4 * 2^stage, 4 / 8 / 16 / 32 channels per group in layer1 .. layer4
ARCHS = {'resnext101_32x4d': 32, 'resnext101_64x4d': 64}
STAGES = ('layer0', 'layer1', 'layer2', 'layer3', 'layer4')     # features[3] (the max-pool), features[4] .. features[7]


def _bn(x, sd, p):
    return F.batch_norm(x, sd[p + '.running_mean'], sd[p + '.running_var'], sd[p + '.weight'], sd[p + '.bias'], False, 0.0, BN_EPS)


def _conv(x, sd, p, stride=1, padding=0, groups=1):
    return F.conv2d(x, sd[p + '.weight'], None, stride, padding, 1, groups)


def block(x, sd, p, groups, stride, project):
    """ConcatTable(main, shortcut) -> CAddTable -> ReLU: main = 1x1 -> BN -> ReLU -> grouped 3x3 (stride) -> BN -> ReLU -> 1x1 -> BN,
    shortcut = strided 1x1 -> BN or the identity."""
    h = F.relu(_bn(_conv(x, sd, p + '.0.0.0.0'), sd, p + '.0.0.0.1'))
    h = F.relu(_bn(_conv(h, sd, p + '.0.0.0.3', stride, 1, groups), sd, p + '.0.0.0.4'))
    h = _bn(_conv(h, sd, p + '.0.0.1'), sd, p + '.0.0.2')
    r = _bn(_conv(x, sd, p + '.0.1.0', stride), sd, p + '.0.1.1') if project else x
    return F.relu(h + r)


def features(x, sd, arch, stages=None, prefix=''):
    """``features`` (resnext101_*_features.py).  ``stages``: dict receiving layer0 (after the max-pool) .. layer4."""
    groups = ARCHS[arch]
    h = F.relu(_bn(_conv(x, sd, prefix + 'features.0', 2, 3), sd, prefix + 'features.1'))
    h = F.max_pool2d(h, 3, 2, 1)
    if stages is not None:
        stages['layer0'] = h
    for i, n in enumerate(LAYERS):
        for b in range(n):
            h = block(h, sd, prefix + 'features.%d.%d' % (4 + i, b), groups, 2 if b == 0 and i > 0 else 1, b == 0)
        if stages is not None:
            stages['layer%d' % (i + 1)] = h
    return h


def forward(x, sd, arch, stages=None):
    """ResNeXt101_*.forward (resnext.py:51-54): features -> AvgPool2d(7, 1) -> view -> last_linear."""
    h = F.avg_pool2d(features(x, sd, arch, stages), 7, 1)
    return F.linear(h.view(h.size(0), -1), sd['last_linear.weight'], sd['last_linear.bias'])


def trn_forward(x, sd, arch, num_segments, stages=None):
    """TRN.forward (trn.py:246-263) with consensus 'MSTRN' on a ResNeXt-101 backbone in eval mode (see oracle/senet.py)."""
    from oracle import functional as OF
    base = {k[len('base_model.'):]: v for k, v in sd.items() if k.startswith('base_model.')}
    b = x.size(0)
    frames = x.view((-1, 3) + tuple(x.shape[-2:]))
    rep = F.avg_pool2d(features(frames, base, arch), 7, 1)
    rep = rep.view(rep.size(0), -1)
    fdim = rep.size(-1)
    t_in = rep.view(b, -1, num_segments, fdim).view(-1, 1, num_segments, fdim)
    v = OF.multiscale_relation(t_in, sd, num_segments, fdim, p='temporal_relation.').squeeze()
    if stages is not None:
        stages['features'] = v
    return F.linear(v, sd['last_linear.weight'], sd['last_linear.bias'])


def reseed_modules_(module):
    """Re-run every convolution's, BatchNorm's and Linear's own initialiser in module order.  The package's constructor draws the
    same numbers when it is called under the same seed (each instance initialises its modules in that order); the reference's
    shared trunk is initialised once at import, so oracle/make_golden_resnext.py re-initialises it with this pass."""
    for m in module.modules():
        if isinstance(m, (torch.nn.Conv2d, torch.nn.BatchNorm2d, torch.nn.Linear)):
            m.reset_parameters()
    return module


def build_package_model(pkg, fx):
    """The package-under-test's model for a ``kind == 'resnext101'`` / ``'trn_resnext101'`` fixture: same constructor call and seeds as
    oracle/make_golden_resnext.py applied to the reference."""
    from oracle import functional as OF
    torch.manual_seed(fx["seeds"]["init"])
    if fx["kind"] == "trn_resnext101":
        m = pkg.TRN(10, num_segments=fx["segments"], arch=fx["arch"], consensus="MSTRN", pretrained=None, **fx["kwargs"])
    else:
        m = pkg.__dict__[fx["arch"]](pretrained=None, **fx["kwargs"])
    OF.randomize_bn_(m, fx["seeds"]["bn"])
    return m.eval()
