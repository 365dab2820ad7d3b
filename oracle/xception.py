"""CPU restatement of the reference's Xception forward (pretorched/models/xception.py:50-210) -- TEST INFRASTRUCTURE.

Plain functional torch over a ``state_dict`` in the reference's layout (``conv1``, ``bn1``, ``conv2``, ``bn2``, ``block{1..12}.skip /
skipbn / rep.<i>.*``, ``conv3`` / ``conv4`` as ``conv1`` (depthwise) + ``pointwise``, ``bn3``, ``bn4``, ``last_linear``), in the
reference's order of operations.  A block's ``rep`` is read from its keys: every index with a ``conv1.weight`` is a separable
convolution, the index after it its BatchNorm, and every separable convolution but one at index 0 (block1, built with
start_with_relu=False) is preceded by a ReLU; a block with a ``skip`` convolution closes ``rep`` with MaxPool2d(3, 2, 1) (in Xception
every projecting block is strided).  Pinned bit for bit against the unmodified reference by oracle/make_golden_xception.py; the
GPU tests run it in fp64, and tools/bench_xception.py in fp16 channels_last on cuDNN.
"""
import torch
import torch.nn.functional as F

BN_EPS = 1e-5
BLOCKS = ['block%d' % i for i in range(1, 13)]


def _bn(x, sd, p):
    return F.batch_norm(x, sd[p + 'running_mean'], sd[p + 'running_var'], sd[p + 'weight'], sd[p + 'bias'], False, 0.0, BN_EPS)


def separable(x, sd, p):
    """SeparableConv2d ``p`` (3x3 depthwise, padding 1, then the 1x1 pointwise; no biases)."""
    x = F.conv2d(x, sd[p + 'conv1.weight'], None, 1, 1, 1, x.shape[1])
    return F.conv2d(x, sd[p + 'pointwise.weight'])


def block(x, sd, p):
    """Block ``p`` (with the trailing dot): rep(x) + skip(x)."""
    seps = sorted(int(k[len(p) + 4:].split('.')[0]) for k in sd if k.startswith(p + 'rep.') and k.endswith('.conv1.weight'))
    h = x
    for i in seps:
        if i > 0:
            h = F.relu(h)
        h = _bn(separable(h, sd, '%srep.%d.' % (p, i)), sd, '%srep.%d.' % (p, i + 1))
    if p + 'skip.weight' in sd:
        h = F.max_pool2d(h, 3, 2, 1)
        skip = _bn(F.conv2d(x, sd[p + 'skip.weight'], stride=2), sd, p + 'skipbn.')
    else:
        skip = x
    return h + skip


def features(x, sd, stages=None):
    """conv1 .. bn4: bn4's output, before the head's ReLU.  ``stages``: optional dict that receives the stem's output and every
    block's."""
    x = F.relu(_bn(F.conv2d(x, sd['conv1.weight'], stride=2), sd, 'bn1.'))
    x = F.relu(_bn(F.conv2d(x, sd['conv2.weight']), sd, 'bn2.'))
    if stages is not None:
        stages['stem'] = x
    for b in BLOCKS:
        x = block(x, sd, b + '.')
        if stages is not None:
            stages[b] = x
    x = F.relu(_bn(separable(x, sd, 'conv3.'), sd, 'bn3.'))
    return _bn(separable(x, sd, 'conv4.'), sd, 'bn4.')


def logits(f, sd):
    x = F.adaptive_avg_pool2d(F.relu(f), (1, 1)).view(f.size(0), -1)
    return F.linear(x, sd['last_linear.weight'], sd['last_linear.bias'])


def forward(x, sd):
    return logits(features(x, sd), sd)


def build_package_model(pkg, fx):
    """The package-under-test's model for a ``kind == 'xception'`` / ``'trn_xception'`` fixture: same constructor call and seeds as
    oracle/make_golden_xception.py applied to the reference."""
    from oracle import functional as OF
    torch.manual_seed(fx["seeds"]["init"])
    if fx["kind"] == "trn_xception":
        m = pkg.TRN(10, num_segments=fx["segments"], arch="xception", consensus="MSTRN", pretrained=None, **fx["kwargs"])
    else:
        m = pkg.xception(pretrained=None, **fx["kwargs"])
    OF.randomize_bn_(m, fx["seeds"]["bn"])
    return m.eval()
