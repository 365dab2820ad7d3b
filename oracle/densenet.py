"""CPU restatement of the reference's DenseNet forward (pretorched/models/torchvision_models.py:254-380 over torchvision's
densenet.py) -- TEST INFRASTRUCTURE.

Plain functional torch over a ``state_dict``, in the reference's order of operations: every dense layer concatenates its inputs
and runs norm1 -> ReLU -> conv1 -> norm2 -> ReLU -> conv2; a transition is norm -> ReLU -> conv -> AvgPool2d(2, 2); ``features``
ends with norm5 (no ReLU); ``logits`` is F.relu -> avg_pool2d(7, stride=1) -> view -> last_linear.  Pinned bit for bit against the
unmodified reference by oracle/make_golden_densenet.py.  Works in the dtype of its inputs (fp32 for the fixtures, fp64 for the
block tests).
"""
import torch
import torch.nn.functional as F

BN_EPS = 1e-5


def bn(x, sd, p):
    return F.batch_norm(x, sd[p + 'running_mean'], sd[p + 'running_var'], sd[p + 'weight'], sd[p + 'bias'], False, 0.0, BN_EPS)


def layer(inputs, sd, p):
    """One _DenseLayer: its k new channels from the list of the block's feature maps so far."""
    h = torch.cat(inputs, 1)
    h = F.conv2d(F.relu(bn(h, sd, p + 'norm1.')), sd[p + 'conv1.weight'])
    return F.conv2d(F.relu(bn(h, sd, p + 'norm2.')), sd[p + 'conv2.weight'], padding=1)


def n_layers(sd, p):
    n = 0
    while (p + 'denselayer%d.conv1.weight' % (n + 1)) in sd:
        n += 1
    return n


def block(x, sd, p):
    """One _DenseBlock (``p``: its state_dict prefix with the trailing dot): the concatenation of its input and every layer's output."""
    feats = [x]
    for i in range(n_layers(sd, p)):
        feats.append(layer(feats, sd, p + 'denselayer%d.' % (i + 1)))
    return torch.cat(feats, 1)


def transition(x, sd, p):
    h = F.conv2d(F.relu(bn(x, sd, p + 'norm.')), sd[p + 'conv.weight'])
    return F.avg_pool2d(h, 2, 2)


def features(x, sd, stages=None):
    """conv0 -> norm0 -> relu0 -> pool0, the dense blocks and transitions, norm5.  ``stages`` receives every block's and
    transition's output under its module name."""
    h = F.conv2d(x, sd['features.conv0.weight'], stride=2, padding=3)
    h = F.max_pool2d(F.relu(bn(h, sd, 'features.norm0.')), 3, 2, 1)
    b = 1
    while ('features.denseblock%d.denselayer1.conv1.weight' % b) in sd:
        h = block(h, sd, 'features.denseblock%d.' % b)
        if stages is not None:
            stages['denseblock%d' % b] = h
        if ('features.transition%d.conv.weight' % b) in sd:
            h = transition(h, sd, 'features.transition%d.' % b)
            if stages is not None:
                stages['transition%d' % b] = h
        b += 1
    return bn(h, sd, 'features.norm5.')


def logits(h, sd):
    """F.relu -> F.avg_pool2d(7, stride=1) -> view -> last_linear (torchvision_models.py:261-266)."""
    h = F.avg_pool2d(F.relu(h), kernel_size=7, stride=1)
    return F.linear(h.view(h.size(0), -1), sd['last_linear.weight'], sd['last_linear.bias'])


def forward(x, sd, stages=None):
    return logits(features(x, sd, stages), sd)


def build_package_model(pkg, fx):
    """The package-under-test's model for a ``densenet`` fixture: same constructor call and seeds as
    oracle/make_golden_densenet.py applied to the reference."""
    from oracle import functional as OF
    torch.manual_seed(fx["seeds"]["init"])
    if fx["kind"] == "trn_densenet":
        m = pkg.TRN(10, num_segments=fx["segments"], arch=fx["arch"], consensus="MSTRN", pretrained=None, **fx["kwargs"])
    else:
        m = pkg.__dict__[fx["arch"]](pretrained=None, **fx["kwargs"])
    OF.randomize_bn_(m, fx["seeds"]["bn"])
    return m.eval()
