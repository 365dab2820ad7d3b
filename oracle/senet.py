"""CPU restatement of the reference's SE-ResNet / SE-ResNeXt forward (pretorched/models/senet.py:85-366) -- TEST INFRASTRUCTURE.

Plain functional torch over a ``state_dict``, like oracle/functional.py; pinned bit for bit against the unmodified reference by
oracle/make_golden_senet.py.  Works in the dtype of its inputs (fp32 for the fixtures, fp64 for the block tests).
"""
import math

import torch
import torch.nn.functional as F

BN_EPS = 1e-5

# name -> (layers, groups); reduction 16, inplanes 64, 7x7 stem, 1x1 projections (senet.py:390-442)
ARCHS = {
    'se_resnet50': ([3, 4, 6, 3], 1),
    'se_resnet101': ([3, 4, 23, 3], 1),
    'se_resnet152': ([3, 8, 36, 3], 1),
    'se_resnext50_32x4d': ([3, 4, 6, 3], 32),
    'se_resnext101_32x4d': ([3, 4, 23, 3], 32),
}


def _bn(x, sd, p):
    return F.batch_norm(x, sd[p + '.running_mean'], sd[p + '.running_var'], sd[p + '.weight'], sd[p + '.bias'], False, 0.0, BN_EPS)


def _conv(x, sd, p, stride=1, padding=0, groups=1):
    return F.conv2d(x, sd[p + '.weight'], sd.get(p + '.bias'), stride, padding, 1, groups)


def se_module(x, sd, p):
    """SEModule.forward (senet.py:97-104)."""
    s = F.adaptive_avg_pool2d(x, 1)
    s = F.relu(_conv(s, sd, p + '.fc1'))
    s = torch.sigmoid(_conv(s, sd, p + '.fc2'))
    return x * s


def block(x, sd, p, resnext, groups, stride, has_downsample):
    """Bottleneck.forward (senet.py:111-131) of SEResNetBottleneck (stride on conv1) / SEResNeXtBottleneck (stride on conv2)."""
    out = F.relu(_bn(_conv(x, sd, p + '.conv1', 1 if resnext else stride), sd, p + '.bn1'))
    out = F.relu(_bn(_conv(out, sd, p + '.conv2', stride if resnext else 1, 1, groups), sd, p + '.bn2'))
    out = _bn(_conv(out, sd, p + '.conv3'), sd, p + '.bn3')
    residual = _bn(_conv(x, sd, p + '.downsample.0', stride), sd, p + '.downsample.1') if has_downsample else x
    return F.relu(se_module(out, sd, p + '.se_module') + residual)


def features(x, sd, arch, stages=None, prefix=''):
    """SENet.features (senet.py:347-353).  ``stages``: dict receiving layer0 .. layer4."""
    layers, groups = ARCHS[arch]
    resnext = groups > 1
    h = F.relu(_bn(_conv(x, sd, prefix + 'layer0.conv1', 2, 3), sd, prefix + 'layer0.bn1'))
    h = F.max_pool2d(h, 3, 2, ceil_mode=True)
    if stages is not None:
        stages['layer0'] = h
    inplanes = 64
    for li, (planes, n) in enumerate(zip((64, 128, 256, 512), layers)):
        stride = 1 if li == 0 else 2
        for bi in range(n):
            p = prefix + 'layer%d.%d' % (li + 1, bi)
            ds = bi == 0 and (stride != 1 or inplanes != planes * 4)
            h = block(h, sd, p, resnext, groups, stride if bi == 0 else 1, ds)
        inplanes = planes * 4
        if stages is not None:
            stages['layer%d' % (li + 1)] = h
    return h


def forward(x, sd, arch, stages=None):
    """SENet.forward (senet.py:355-366) in eval mode: features -> AvgPool2d(7, stride 1) -> view -> last_linear."""
    h = F.avg_pool2d(features(x, sd, arch, stages), 7, 1)
    return F.linear(h.view(h.size(0), -1), sd['last_linear.weight'], sd['last_linear.bias'])


def trn_forward(x, sd, arch, num_segments, stages=None):
    """TRN.forward (trn.py:246-263) with consensus 'MSTRN' on an SENet backbone in eval mode: frames folded into the batch,
    ``base_model.features`` -> AvgPool2d(7) (its ``last_linear`` is a Dropout, the identity), regrouped [B, 1, T, F],
    ``MultiScaleRelation`` (tuples drawn from NumPy's global RNG as the reference does), ``.squeeze()``, final Linear."""
    from oracle import functional as OF
    base = {k[len('base_model.'):]: v for k, v in sd.items() if k.startswith('base_model.')}
    b = x.size(0)
    frames = x.view((-1, 3) + tuple(x.shape[-2:]))
    rep = F.avg_pool2d(features(frames, base, arch), 7, 1)
    rep = rep.view(rep.size(0), -1)
    fdim = rep.size(-1)
    rep = rep.view(b, -1, num_segments, fdim)
    t_in = rep.view(-1, rep.size(1), num_segments, fdim)
    v = OF.multiscale_relation(t_in, sd, num_segments, fdim, p='temporal_relation.').squeeze()
    if stages is not None:
        stages['features'] = v
    return F.linear(v, sd['last_linear.weight'], sd['last_linear.bias'])


def se_width(planes, groups):
    """conv1 / conv2 width of a block of stage ``planes`` (senet.py:190 for SE-ResNeXt, ``planes`` for SE-ResNet)."""
    return math.floor(planes * (4 / 64)) * groups if groups > 1 else planes


def build_package_model(pkg, fx):
    """The package-under-test's model for a ``kind == 'senet'`` / ``'trn_senet'`` fixture: same constructor call and seeds as
    oracle/make_golden_senet.py applied to the reference."""
    from oracle import functional as OF
    torch.manual_seed(fx["seeds"]["init"])
    if fx["kind"] == "trn_senet":
        m = pkg.TRN(10, num_segments=fx["segments"], arch=fx["arch"], consensus="MSTRN", pretrained=None, **fx["kwargs"])
    else:
        m = pkg.__dict__[fx["arch"]](pretrained=None, **fx["kwargs"])
    OF.randomize_bn_(m, fx["seeds"]["bn"])
    return m.eval()
