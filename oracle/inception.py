"""CPU restatement of the reference's Inception-v4 and Inception-ResNet-v2 forwards (pretorched/models/inceptionv4.py:34-309,
inceptionresnetv2.py:34-331) -- TEST INFRASTRUCTURE.

Plain functional torch over a ``state_dict``, like oracle/bninception.py, walking the block table models.inception.BRANCHES in
the reference's concatenation order; each unit's stride / padding is read from the module it restates.  Pinned bit for bit
against the unmodified reference by oracle/make_golden_inception.py.  Works in the dtype of its inputs (fp32 for the fixtures,
fp64 for the block tests).
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

BN_EPS = 1e-3

# Convolution geometries of both networks at 299^2 inputs, shared by the tests and tools/bench_inception.py: every convolution with
# taps that is not "same"-padded (VALID; the stem's 3 input channels are stored with pitch 8, which is what the kernels read), and
# the 1xn / nx1 / 5x5 ones (ONE_BY_N).  Rows: (C, H = W, K, kh, kw, stride, ph, pw).
VALID = [(8, 299, 32, 3, 3, 2, 0, 0), (32, 149, 32, 3, 3, 1, 0, 0), (64, 147, 96, 3, 3, 2, 0, 0), (64, 73, 96, 3, 3, 1, 0, 0),
         (192, 71, 192, 3, 3, 2, 0, 0), (384, 35, 384, 3, 3, 2, 0, 0), (224, 35, 256, 3, 3, 2, 0, 0), (192, 17, 192, 3, 3, 2, 0, 0),
         (320, 17, 320, 3, 3, 2, 0, 0), (80, 73, 192, 3, 3, 1, 0, 0), (320, 35, 384, 3, 3, 2, 0, 0), (256, 35, 384, 3, 3, 2, 0, 0),
         (256, 17, 384, 3, 3, 2, 0, 0), (256, 17, 288, 3, 3, 2, 0, 0), (288, 17, 320, 3, 3, 2, 0, 0)]
ONE_BY_N = [(64, 73, 64, 1, 7, 1, 0, 3), (64, 73, 64, 7, 1, 1, 3, 0), (192, 17, 224, 1, 7, 1, 0, 3), (224, 17, 256, 7, 1, 1, 3, 0),
            (192, 17, 192, 7, 1, 1, 3, 0), (224, 17, 224, 7, 1, 1, 3, 0), (224, 17, 256, 1, 7, 1, 0, 3), (256, 17, 256, 1, 7, 1, 0, 3),
            (256, 17, 320, 7, 1, 1, 3, 0), (384, 8, 256, 1, 3, 1, 0, 1), (384, 8, 256, 3, 1, 1, 1, 0), (384, 8, 448, 3, 1, 1, 1, 0),
            (448, 8, 512, 1, 3, 1, 0, 1), (512, 8, 256, 1, 3, 1, 0, 1), (512, 8, 256, 3, 1, 1, 1, 0), (128, 17, 160, 1, 7, 1, 0, 3),
            (160, 17, 192, 7, 1, 1, 3, 0), (192, 8, 224, 1, 3, 1, 0, 1), (224, 8, 256, 3, 1, 1, 1, 0), (48, 35, 64, 5, 5, 1, 2, 2)]


def unit(x, sd, p, conv):
    """BasicConv2d: conv (no bias) -> eval-mode BatchNorm(eps 0.001) -> ReLU.  ``conv``: the nn.Conv2d whose geometry it uses."""
    h = F.conv2d(x, sd[p + 'conv.weight'], None, conv.stride, conv.padding)
    h = F.batch_norm(h, sd[p + 'bn.running_mean'], sd[p + 'bn.running_var'], sd[p + 'bn.weight'], sd[p + 'bn.bias'], False, 0.0,
                     BN_EPS)
    return F.relu(h)


def block(x, sd, mod, prefix):
    """One block (``mod``: the package's container, ``prefix``: its state_dict prefix with the trailing dot)."""
    from pretorched_x_b200.models.inception import BRANCHES, RESIDUAL
    kind = type(mod).kind
    u = lambda h, path: unit(h, sd, prefix + path + '.', mod.get_submodule(path).conv)
    outs = []
    for br in BRANCHES[kind]:
        if br[0] == 'max':
            outs.append(F.max_pool2d(x, 3, 2))
        elif br[0] == 'avg':
            outs.append(u(F.avg_pool2d(x, 3, 1, 1, count_include_pad=False), br[1][-1]))
        else:
            h = x
            for p in br[1]:
                h = u(h, p)
            outs.extend([u(h, p) for p in br[2]] if br[0] == 'fork' else [h])
    out = torch.cat(outs, 1)
    if kind not in RESIDUAL:
        return out
    out = F.conv2d(out, sd[prefix + 'conv2d.weight'], sd[prefix + 'conv2d.bias']) * mod.scale + x
    return out if getattr(mod, 'noReLU', False) else F.relu(out)


def _units(model):
    """(state_dict prefix, module) of the trunk's units in order."""
    if hasattr(model, 'conv2d_1a'):
        names = ['conv2d_1a', 'conv2d_2a', 'conv2d_2b', 'maxpool_3a', 'conv2d_3b', 'conv2d_4a', 'maxpool_5a', 'mixed_5b']
        names += ['repeat.%d' % i for i in range(10)] + ['mixed_6a'] + ['repeat_1.%d' % i for i in range(20)] + ['mixed_7a']
        names += ['repeat_2.%d' % i for i in range(9)] + ['block8', 'conv2d_7b']
    else:
        names = ['features.%d' % i for i in range(len(model.features))]
    return [(n + '.', model.get_submodule(n)) for n in names]


def features(x, sd, model, stages=None):
    """The trunk; ``model``: a package InceptionV4 / InceptionResNetV2 (module geometry only).  ``stages`` receives every unit's output."""
    from pretorched_x_b200.models.inception import BasicConv2d
    h = x
    for p, m in _units(model):
        if isinstance(m, nn.MaxPool2d):
            h = F.max_pool2d(h, 3, 2)
        elif isinstance(m, BasicConv2d):
            h = unit(h, sd, p, m.conv)
        else:
            h = block(h, sd, m, p)
        if stages is not None:
            stages[p[:-1]] = h
    return h


def logits(h, sd):
    """AvgPool2d(8, count_include_pad=False) -> view -> last_linear (inceptionv4.py:300-304)."""
    h = F.avg_pool2d(h, 8, count_include_pad=False)
    return F.linear(h.view(h.size(0), -1), sd['last_linear.weight'], sd['last_linear.bias'])


def forward(x, sd, model, stages=None):
    return logits(features(x, sd, model, stages), sd)


def build_package_model(pkg, fx):
    """The package-under-test's model for an ``inception`` fixture: same constructor call and seeds as
    oracle/make_golden_inception.py applied to the reference."""
    from oracle import functional as OF
    torch.manual_seed(fx["seeds"]["init"])
    if fx["kind"] == "trn_inception":
        m = pkg.TRN(10, num_segments=fx["segments"], arch=fx["arch"], consensus="MSTRN", pretrained=None, **fx["kwargs"])
    else:
        m = pkg.__dict__[fx["arch"]](pretrained=None, **fx["kwargs"])
    OF.randomize_bn_(m, fx["seeds"]["bn"])
    return m.eval()
