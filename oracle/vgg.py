"""CPU restatement of the reference's VGG and AlexNet forwards (pretorched/models/torchvision_models.py:195-248, 597-725 over
torchvision's vgg.py / alexnet.py) -- TEST INFRASTRUCTURE.

Plain functional torch over a ``state_dict`` in the reference's layout (``_features.<i>.*``, ``linear0`` / ``linear1`` /
``last_linear``), in the reference's order of operations: the ``_features`` Sequential layer by layer, ``view(B, -1)`` (torchvision's
avgpool is skipped), linear0 -> ReLU -> linear1 for ``features`` (the dropouts are the identity in eval) and ReLU -> last_linear for
``logits``.  Pinned bit for bit against the unmodified reference by oracle/make_golden_vgg.py.
"""
import torch.nn.functional as F

BN_EPS = 1e-5

# torchvision's layer lists: 'M' a 2x2 stride-2 max pool, an int a 3x3 padding-1 convolution to that many channels (+ BN) + ReLU
CFGS = {
    'vgg11': [64, 'M', 128, 'M', 256, 256, 'M', 512, 512, 'M', 512, 512, 'M'],
    'vgg13': [64, 64, 'M', 128, 128, 'M', 256, 256, 'M', 512, 512, 'M', 512, 512, 'M'],
    'vgg16': [64, 64, 'M', 128, 128, 'M', 256, 256, 256, 'M', 512, 512, 512, 'M', 512, 512, 512, 'M'],
    'vgg19': [64, 64, 'M', 128, 128, 'M', 256, 256, 256, 256, 'M', 512, 512, 512, 512, 'M', 512, 512, 512, 512, 'M'],
}
# AlexNet's features: (kind, index, args)
ALEXNET = [('conv', 0, dict(stride=4, padding=2)), ('pool', 2, None), ('conv', 3, dict(padding=2)), ('pool', 5, None),
           ('conv', 6, dict(padding=1)), ('conv', 8, dict(padding=1)), ('conv', 10, dict(padding=1)), ('pool', 12, None)]


def _bn(x, sd, p):
    return F.batch_norm(x, sd[p + 'running_mean'], sd[p + 'running_var'], sd[p + 'weight'], sd[p + 'bias'], False, 0.0, BN_EPS)


def trunk(x, sd, arch, stages=None):
    """``_features``: the last pool's output.  ``stages``: optional dict that receives every pool's output."""
    if arch == 'alexnet':
        for kind, i, kw in ALEXNET:
            if kind == 'conv':
                x = F.relu(F.conv2d(x, sd['_features.%d.weight' % i], sd['_features.%d.bias' % i], **kw))
            else:
                x = F.max_pool2d(x, 3, 2)
                if stages is not None:
                    stages['pool%d' % i] = x
        return x
    bn = arch.endswith('_bn')
    i = 0
    for v in CFGS[arch.replace('_bn', '')]:
        if v == 'M':
            x = F.max_pool2d(x, 2, 2)
            if stages is not None:
                stages['pool%d' % i] = x
            i += 1
            continue
        x = F.conv2d(x, sd['_features.%d.weight' % i], sd['_features.%d.bias' % i], padding=1)
        if bn:
            x = _bn(x, sd, '_features.%d.' % (i + 1))
        x = F.relu(x)
        i += 3 if bn else 2
    return x


def features(x, sd, arch, stages=None):
    """fc7's output before its ReLU, fp32 [B, 4096]."""
    h = trunk(x, sd, arch, stages)
    h = h.view(h.size(0), -1)
    h = F.relu(F.linear(h, sd['linear0.weight'], sd['linear0.bias']))
    return F.linear(h, sd['linear1.weight'], sd['linear1.bias'])


def logits(f, sd):
    return F.linear(F.relu(f), sd['last_linear.weight'], sd['last_linear.bias'])
