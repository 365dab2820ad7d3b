"""CPU fp32 restatement of the reference's MobileNetV2 forward (pretorched/models/mobilenet.py:22-126) -- TEST INFRASTRUCTURE.

Plain functional torch over a ``state_dict``, like oracle/functional.py; pinned bit for bit against the unmodified reference by
oracle/make_golden_mobilenet.py.  Also holds the deterministic conditioning the fixtures and the tests share.
"""
import torch
import torch.nn.functional as F

BN_EPS = 1e-5

# t, c, n, s (mobilenet.py:85-94)
SETTING = [[1, 16, 1, 1], [6, 24, 2, 2], [6, 32, 3, 2], [6, 64, 4, 2], [6, 96, 3, 1], [6, 160, 3, 2], [6, 320, 1, 1]]


def blocks(width_mult=1.0):
    """[(inp, oup, stride, expand_ratio)] of features.1 .. features.17, in order."""
    out, inp = [], int(32 * width_mult)
    for t, c, n, s in SETTING:
        oup = int(c * width_mult)
        for i in range(n):
            out.append((inp, oup, s if i == 0 else 1, t))
            inp = oup
    return out


def _bn(x, sd, p):
    return F.batch_norm(x, sd[p + '.running_mean'], sd[p + '.running_var'], sd[p + '.weight'], sd[p + '.bias'], False, 0.0, BN_EPS)


def _conv(x, sd, p, stride=1, padding=0, groups=1):
    return F.conv2d(x, sd[p + '.weight'], None, stride, padding, 1, groups)


def conv_bn(x, sd, p, stride):
    """conv_bn (mobilenet.py:22-27): 3x3 conv (padding 1) -> BN -> ReLU6."""
    return F.relu6(_bn(_conv(x, sd, p + '.0', stride, 1), sd, p + '.1'))


def conv_1x1_bn(x, sd, p):
    """conv_1x1_bn (mobilenet.py:30-35)."""
    return F.relu6(_bn(_conv(x, sd, p + '.0'), sd, p + '.1'))


def inverted_residual(x, sd, p, inp, oup, stride, expand_ratio, taps=None):
    """InvertedResidual.forward (mobilenet.py:72-76).  ``taps``: a dict that receives the post-ReLU6 expansion and depthwise
    outputs (the generator checks that the clamps bind)."""
    hidden = round(inp * expand_ratio)
    h, i = x, 0
    if expand_ratio != 1:
        h = F.relu6(_bn(_conv(h, sd, p + '.conv.0'), sd, p + '.conv.1'))
        i = 3
        if taps is not None:
            taps['expand'] = h
    h = F.relu6(_bn(_conv(h, sd, p + '.conv.%d' % i, stride, 1, hidden), sd, p + '.conv.%d' % (i + 1)))
    if taps is not None:
        taps['dw'] = h
    h = _bn(_conv(h, sd, p + '.conv.%d' % (i + 3)), sd, p + '.conv.%d' % (i + 4))
    return x + h if stride == 1 and inp == oup else h


def features(x, sd, stages=None, taps=None, prefix='features.'):
    """``model.features`` (mobilenet.py:100-113).  ``stages``: dict receiving every block output (``features.<i>``)."""
    h = conv_bn(x, sd, prefix + '0', 2)
    if stages is not None:
        stages['features.0'] = h
    for i, (inp, oup, s, t) in enumerate(blocks(), start=1):
        tp = {} if taps is not None else None
        h = inverted_residual(h, sd, prefix + '%d' % i, inp, oup, s, t, tp)
        if taps is not None:
            taps[i] = tp
        if stages is not None:
            stages['features.%d' % i] = h
    h = conv_1x1_bn(h, sd, prefix + '18')
    if stages is not None:
        stages['features.18'] = h
    return h


def forward(x, sd, stages=None, taps=None):
    """MobileNetV2.forward in eval mode (mobilenet.py:121-126): features -> mean over H, W -> dropout (identity) -> last_linear."""
    h = features(x, sd, stages, taps)
    h = h.mean(3).mean(2)
    return F.linear(h, sd['last_linear.weight'], sd['last_linear.bias'])


def trn_forward(x, sd, num_segments, stages=None):
    """TRN.forward (trn.py:246-263) with consensus 'TRN' on a MobileNetV2 backbone in eval mode: frames folded into the batch,
    ``base_model`` features -> mean over H, W (its ``last_linear`` is a Dropout, the identity), regrouped [B, 1, T, F],
    ``Relation``, ``.squeeze()``, final Linear."""
    from oracle import functional as OF
    base = {k[len('base_model.'):]: v for k, v in sd.items() if k.startswith('base_model.')}
    b = x.size(0)
    frames = x.view((-1, 3) + tuple(x.shape[-2:]))
    rep = features(frames, base).mean(3).mean(2)
    fdim = rep.size(-1)
    rep = rep.view(b, -1, num_segments, fdim)
    t_in = rep.view(-1, rep.size(1), num_segments, fdim)
    v = OF.relation(t_in, sd, 'temporal_relation.', num_segments, fdim).squeeze()
    if stages is not None:
        stages['features'] = v
    return F.linear(v, sd['last_linear.weight'], sd['last_linear.bias'])


def calibrate_bn_(model, x, target_std=3.0):
    """Scale the affine (weight and bias) of every BatchNorm, in execution order, so that its output on ``x`` has standard
    deviation ``target_std``.  At the reference's random init the activations shrink layer by layer and no ReLU6 ever reaches
    its upper clamp; at std 3 a few percent of every activated tensor sits at 6.  Works on the reference's model and on
    pretorched_x_b200's alike (both compute the forward on the CPU here).  Returns the factors (``apply_bn_factors_``)."""
    bns = [m for _, m in model.named_modules() if isinstance(m, torch.nn.BatchNorm2d)]
    factors = []

    def hook(m, inp, out):
        f = target_std / max(float(out.double().std()), 1e-12)
        with torch.no_grad():
            m.weight.mul_(f)
            m.bias.mul_(f)
        factors.append(f)
        return F.batch_norm(inp[0], m.running_mean, m.running_var, m.weight, m.bias, False, 0.0, m.eps)

    handles = [b.register_forward_hook(hook) for b in bns]
    try:
        with torch.no_grad():
            h = x
            for m in model.features:
                h = m(h) if not hasattr(m, 'use_res_connect') else _ref_block(m, h)
    finally:
        for hd in handles:
            hd.remove()
    assert len(factors) == len(bns)
    return factors


def _ref_block(block, x):
    return x + block.conv(x) if block.use_res_connect else block.conv(x)


def build_package_model(pkg, fx):
    """The package-under-test's model for a ``kind == 'mobilenetv2'`` / ``'trn_mobilenetv2'`` fixture: same constructor call,
    seeds and BatchNorm conditioning as oracle/make_golden_mobilenet.py applied to the reference."""
    from oracle import functional as OF
    torch.manual_seed(fx["seeds"]["init"])
    if fx["kind"] == "trn_mobilenetv2":
        m = pkg.TRN(10, num_segments=fx["segments"], arch="mobilenetv2", consensus=fx["consensus"], pretrained=None, **fx["kwargs"])
        OF.randomize_bn_(m, fx["seeds"]["bn"])
        apply_bn_factors_(m.base_model, fx["bn_factors"])
    else:
        m = pkg.mobilenetv2(pretrained=None, **fx["kwargs"])
        OF.randomize_bn_(m, fx["seeds"]["bn"])
        apply_bn_factors_(m, fx["bn_factors"])
    return m.eval()


def apply_bn_factors_(model, factors):
    """Apply ``calibrate_bn_``'s factors to a model with the same BatchNorm sequence."""
    bns = [m for _, m in model.named_modules() if isinstance(m, torch.nn.BatchNorm2d)]
    assert len(bns) == len(factors)
    with torch.no_grad():
        for m, f in zip(bns, factors):
            m.weight.mul_(f)
            m.bias.mul_(f)
    return model
