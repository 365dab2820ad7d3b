"""CPU restatement of the reference's BNInception forward (pretorched/models/bninception.py:254-495) -- TEST INFRASTRUCTURE.

Plain functional torch over a ``state_dict``, like oracle/senet.py; pinned bit for bit against the unmodified reference by
oracle/make_golden_bninception.py.  Every ReLU of the reference is in place on a BatchNorm output, so each unit is
conv -> BN -> ReLU and every tensor the reference later reads (pool inputs, ``torch.cat`` operands) is post-ReLU.  Works in the
dtype of its inputs (fp32 for the fixtures, fp64 for the block tests).
"""
import torch
import torch.nn.functional as F

BN_EPS = 1e-5

# name, input channels, 1x1 (None: none), (3x3 reduce, 3x3), (double reduce, double 3x3), (pool kind, projection)
# pool kinds: 'avg' AvgPool2d(3, 1, 1, ceil, count_include_pad), 'max1' MaxPool2d(3, 1, 1, ceil), 'max2' MaxPool2d(3, 2, ceil)
# with no projection, which also makes both 3x3 branches stride 2 (bninception.py:43-250)
BLOCKS = [
    ('3a', 192, 64, (64, 64), (64, 96), ('avg', 32)),
    ('3b', 256, 64, (64, 96), (64, 96), ('avg', 64)),
    ('3c', 320, None, (128, 160), (64, 96), ('max2', None)),
    ('4a', 576, 224, (64, 96), (96, 128), ('avg', 128)),
    ('4b', 576, 192, (96, 128), (96, 128), ('avg', 128)),
    ('4c', 576, 160, (128, 160), (128, 160), ('avg', 128)),
    ('4d', 608, 96, (128, 192), (160, 192), ('avg', 128)),
    ('4e', 608, None, (128, 192), (192, 256), ('max2', None)),
    ('5a', 1056, 352, (192, 320), (160, 224), ('avg', 128)),
    ('5b', 1024, 352, (192, 320), (192, 224), ('max1', 128)),
]
STAGES = ['stem'] + [b[0] for b in BLOCKS]


def unit(x, sd, p, stride=1, padding=0):
    """conv (+bias) -> eval-mode BatchNorm -> ReLU."""
    h = F.conv2d(x, sd[p + '.weight'], sd[p + '.bias'], stride, padding)
    h = F.batch_norm(h, sd[p + '_bn.running_mean'], sd[p + '_bn.running_var'], sd[p + '_bn.weight'], sd[p + '_bn.bias'], False, 0.0,
                     BN_EPS)
    return F.relu(h)


def stem(x, sd):
    """bninception.py:255-265."""
    h = F.max_pool2d(unit(x, sd, 'conv1_7x7_s2', 2, 3), 3, 2, ceil_mode=True)
    h = unit(unit(h, sd, 'conv2_3x3_reduce'), sd, 'conv2_3x3', 1, 1)
    return F.max_pool2d(h, 3, 2, ceil_mode=True)


def block(x, sd, spec):
    """One inception block (bninception.py:266-288 and its siblings): the branches concatenated in the reference's order."""
    n, _, c1, _, _, (pk, proj) = spec
    p = 'inception_%s_' % n
    s = 2 if pk == 'max2' else 1
    outs = [unit(x, sd, p + '1x1')] if c1 is not None else []
    outs.append(unit(unit(x, sd, p + '3x3_reduce'), sd, p + '3x3', s, 1))
    d = unit(unit(x, sd, p + 'double_3x3_reduce'), sd, p + 'double_3x3_1', 1, 1)
    outs.append(unit(d, sd, p + 'double_3x3_2', s, 1))
    if pk == 'avg':
        pooled = F.avg_pool2d(x, 3, 1, 1, ceil_mode=True, count_include_pad=True)
    elif pk == 'max1':
        pooled = F.max_pool2d(x, 3, 1, 1, ceil_mode=True)
    else:
        pooled = F.max_pool2d(x, 3, 2, ceil_mode=True)
    outs.append(unit(pooled, sd, p + 'pool_proj') if proj is not None else pooled)
    return torch.cat(outs, 1)


def features(x, sd, stages=None, prefix=''):
    """BNInception.features.  ``stages``: dict receiving the stem output and every block output."""
    if prefix:
        sd = {k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)}
    h = stem(x, sd)
    if stages is not None:
        stages['stem'] = h
    for spec in BLOCKS:
        h = block(h, sd, spec)
        if stages is not None:
            stages[spec[0]] = h
    return h


def logits(h, sd):
    """global_pool (AvgPool2d(7, stride=1, ceil_mode=True)) -> view -> last_linear (bninception.py:486-490)."""
    h = F.avg_pool2d(h, 7, 1, 0, ceil_mode=True, count_include_pad=True)
    return F.linear(h.view(h.size(0), -1), sd['last_linear.weight'], sd['last_linear.bias'])


def forward(x, sd, stages=None):
    return logits(features(x, sd, stages), sd)


def trn_forward(x, sd, num_segments, stages=None):
    """TRN.forward (trn.py:246-263) with consensus 'MSTRN' on a BNInception backbone in eval mode: frames folded into the batch,
    ``base_model`` (its ``last_linear`` a Dropout, the identity), regrouped [B, 1, T, F], ``MultiScaleRelation`` (tuples drawn
    from NumPy's global RNG as the reference does), ``.squeeze()``, final Linear."""
    from oracle import functional as OF
    base = {k[len('base_model.'):]: v for k, v in sd.items() if k.startswith('base_model.')}
    b = x.size(0)
    frames = x.view((-1, 3) + tuple(x.shape[-2:]))
    rep = F.avg_pool2d(features(frames, base), 7, 1, 0, ceil_mode=True, count_include_pad=True)
    rep = rep.view(rep.size(0), -1)
    fdim = rep.size(-1)
    t_in = rep.view(b, -1, num_segments, fdim).view(-1, 1, num_segments, fdim)
    v = OF.multiscale_relation(t_in, sd, num_segments, fdim, p='temporal_relation.').squeeze()
    if stages is not None:
        stages['features'] = v
    return F.linear(v, sd['last_linear.weight'], sd['last_linear.bias'])


def build_package_model(pkg, fx):
    """The package-under-test's model for a ``kind == 'bninception'`` / ``'trn_bninception'`` fixture: same constructor call and
    seeds as oracle/make_golden_bninception.py applied to the reference."""
    from oracle import functional as OF
    torch.manual_seed(fx["seeds"]["init"])
    if fx["kind"] == "trn_bninception":
        m = pkg.TRN(10, num_segments=fx["segments"], arch="bninception", consensus="MSTRN", pretrained=None, **fx["kwargs"])
    else:
        m = pkg.bninception(pretrained=None, **fx["kwargs"])
    OF.randomize_bn_(m, fx["seeds"]["bn"])
    return m.eval()
