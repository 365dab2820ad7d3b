"""CPU: Inception-v4 and Inception-ResNet-v2 against the reference, as recorded in the fixtures (tests/golden/*_b2_299.pt, written
by oracle/make_golden_inception.py from the unmodified reference): state_dict keys, shapes and order, a seeded init bit-identical
to the reference's, the registry rows, the 'imagenet' head slicing, the oracle restatement against the reference's features and
logits, TRN on both backbones, the slab kernel's plans of every valid-padded and 1xn / nx1 shape of both networks, and the
refusals (partial ``features``, 1x1 slice convolutions, the exclude-pad pool's bad arguments)."""
import ctypes
import os

import pytest
import torch

import pretorched_x_b200 as P
from pretorched_x_b200 import _lib
from oracle import functional as OF
from oracle import inception as OI
from oracle.inception import ONE_BY_N, VALID
from oracle.make_golden import sample_of

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
B2_ERR_INVALID = -1
ARCHS = [("inceptionv4", 896, 42679816), ("inceptionresnetv2", 1306, 55843464)]


def _load(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


@pytest.mark.parametrize("arch,n_state,n_params", ARCHS)
def test_state_dict_layout_and_seeded_init_match_reference(arch, n_state, n_params):
    fx = _load("%s_b2_299.pt" % arch)
    torch.manual_seed(fx["seeds"]["init"])
    model = P.__dict__[arch](pretrained=None, **fx["kwargs"])
    sd = model.state_dict()
    assert len(sd) == n_state == fx["n_state"] and sum(p.numel() for p in model.parameters()) == n_params
    assert [(k, tuple(v.shape)) for k, v in sd.items()] == [tuple(kv) for kv in fx["keys"]]
    assert OF.digests_match(OF.state_digest(sd), fx["init_digest"])


@pytest.mark.parametrize("arch", [a[0] for a in ARCHS])
def test_pretrained_settings_rows_match_reference(arch):
    fx = _load("%s_b2_299.pt" % arch)
    assert P.pretrained_settings[arch] == fx["settings"][arch]
    assert arch in P.model_names


@pytest.mark.parametrize("arch", [a[0] for a in ARCHS])
@pytest.mark.parametrize("row,classes", [("imagenet", 1000), ("imagenet+background", 1001)])
def test_pretrained_head_slicing(monkeypatch, arch, row, classes):
    torch.manual_seed(5)
    ckpt = P.__dict__[arch](num_classes=1001, pretrained=None).state_dict()
    import torch.utils.model_zoo as model_zoo
    monkeypatch.setattr(model_zoo, "load_url", lambda url: ckpt)
    m = P.__dict__[arch](num_classes=classes, pretrained=row)
    assert m.last_linear.out_features == classes
    rows = slice(1, None) if row == "imagenet" else slice(None)
    assert torch.equal(m.last_linear.weight, ckpt["last_linear.weight"][rows])
    assert torch.equal(m.last_linear.bias, ckpt["last_linear.bias"][rows])
    assert (m.input_space, m.input_range, m.mean, m.std, list(m.input_size)) == ("RGB", [0, 1], [0.5] * 3, [0.5] * 3, [3, 299, 299])
    with pytest.raises(AssertionError):
        P.__dict__[arch](num_classes=1001 if row == "imagenet" else 1000, pretrained=row)


@pytest.mark.parametrize("arch", [a[0] for a in ARCHS])
def test_oracle_reproduces_reference_features_and_logits(arch):
    fx = _load("%s_b2_299.pt" % arch)
    model = OI.build_package_model(P, fx)
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    assert OF.digests_match(OF.state_digest(sd), fx["weight_digest"])
    x = OF.seeded_input(fx["input_shape"], fx["seeds"]["input"])
    with torch.no_grad():
        feats = OI.features(x, sd, model)
        logits = OI.logits(feats, sd)
    assert tuple(feats.shape) == tuple(fx["features"]["shape"]) == (2, 1536, 8, 8)
    s, step = sample_of(feats)
    assert step == fx["features"]["step"] and torch.equal(s, fx["features"]["sample"])
    assert torch.equal(logits, fx["logits"])


@pytest.mark.parametrize("arch", [a[0] for a in ARCHS])
def test_trn_builds_and_refuses_fine_tune(arch):
    m = P.TRN(10, num_segments=4, arch=arch, consensus="MSTRN", pretrained=None, frame_bottleneck_dim=128, video_feature_dim=64)
    assert m.frame_feature_dim == 1536
    # without a checkpoint the backbone keeps the reference constructor's attributes (input_space None, input_size (299, 299, 3)),
    # which TRN's getattr lookups prefer over the registry row, as the reference's TRN does
    assert (m.input_space, m.mean, m.std, list(m.input_size)) == (None, None, None, [299, 3])
    assert sum(len(g["params"]) for g in m.get_optim_policies()) > 0
    with pytest.raises(NotImplementedError, match="has none"):
        m.fine_tune(4)


def test_partial_features_refuse_to_run():
    m = P.inceptionv4(pretrained=None).eval()
    part = m.features[3:6]
    assert type(part) is type(m.features) and len(part) == 3
    with pytest.raises(NotImplementedError, match="whole trunk"):
        part(torch.zeros(1, 64, 147, 147))


def _args(N, C, H, K, kh, kw, s, ph, pw, ldy=None):
    a = _lib.ConvArgs()
    a.N, a.T, a.H, a.W, a.C, a.K, a.ldy = N, 1, H, H, C, K, ldy or K
    a.kt, a.kh, a.kw, a.st, a.sh, a.sw, a.pt, a.ph, a.pw = 1, kh, kw, 1, s, s, 0, ph, pw
    a.relu, a.mode = 1, _lib.B2_CONV_AUTO
    return a


def _plan(entry, shape, N=128):
    out = (ctypes.c_int * 10)()
    fn = getattr(_lib.load(), entry)
    fn.argtypes = [ctypes.POINTER(_lib.ConvArgs), ctypes.POINTER(ctypes.c_int)]
    assert fn(ctypes.byref(_args(N, *shape)), out) == 0
    return tuple(out)


@pytest.mark.parametrize("shape", VALID + ONE_BY_N, ids=lambda s: "%d-%d_%dx%d_s%d_p%d%d_%d" % (s[0], s[2], s[3], s[4], s[5], s[6], s[7], s[1]))
@pytest.mark.parametrize("N", [2, 128])
def test_slice_plan_covers_every_shape(shape, N):
    plan = _plan("b2_debug_slab_slice_plan", shape, N)
    assert plan[0] == 1 and plan[1] * plan[2] <= 192, plan


# the shapes the plain convolution's slab plan still declines at B = 128 (output widths 192 / 320 on runtime-N tiles; the slice
# entry takes 128-column tiles for them): the engine runs these networks' convolutions with taps through the slice entry
@pytest.mark.parametrize("shape", [(192, 71, 192, 3, 3, 2, 0, 0), (192, 17, 192, 7, 1, 1, 3, 0), (256, 17, 320, 7, 1, 1, 3, 0),
                                   (80, 73, 192, 3, 3, 1, 0, 0), (160, 17, 192, 7, 1, 1, 3, 0)])
def test_plain_plan_declines_and_slice_plan_takes_128(shape):
    assert _plan("b2_debug_slab_plan", shape)[0] == 0
    assert _plan("b2_debug_slab_slice_plan", shape)[:2] == (1, 128)


def test_valid_padding_keeps_same_padded_plans():
    """Centring the row offsets of a one-sided window leaves every "same" geometry as it was: 3x3 valid at stride 1 plans with the
    slab rows of the same-padded 3x3 on a map two pixels wider."""
    same = _plan("b2_debug_slab_plan", (64, 75, 96, 3, 3, 1, 1, 1))
    valid = _plan("b2_debug_slab_plan", (64, 77, 96, 3, 3, 1, 0, 0))
    assert valid[:4] == same[:4] and valid[4] == same[4]


@pytest.mark.parametrize("case,kw", [
    ("1x1 filter", dict(kh=1, kw=1, ph=0, pw=0)),
    ("even filter", dict(kh=2, kw=2, ph=0, pw=0)),
    ("padding over same", dict(ph=2, pw=2)),
    ("negative padding", dict(ph=-1)),
    ("temporal filter", dict(kt=3, pt=1)),
])
def test_slice_conv_refusals(case, kw):
    a = _args(2, 64, 28, 96, 3, 3, 1, 1, 1, ldy=256)
    a.x, a.w, a.scale, a.shift, a.y = (ctypes.c_void_p(v) for v in (0x10000, 0x20000, 0x30000, 0x40000, 0x50000))
    for k, v in kw.items():
        setattr(a, k, v)
    rc = _lib.load().b2_conv_ndhwc_fprop_slice(ctypes.byref(a), ctypes.c_void_p(0))
    assert rc == B2_ERR_INVALID, (case, rc, _lib.last_error())


@pytest.mark.parametrize("case,args", [
    ("pitch below channels", dict(ldx=32)),
    ("unaligned output", dict(y=0x50008)),
    ("window outside the input", dict(Ho=30)),
    ("padding over half the window", dict(ph=2, pw=2)),
    ("channels not a multiple of 8", dict(C=60)),
    ("empty output", dict(Wo=0)),
])
def test_exclude_pad_pool_refusals(case, args):
    a = dict(x=0x10000, ldx=64, y=0x50000, ldy=128, N=2, T=1, H=28, W=28, C=64, kt=1, kh=3, kw=3, st=1, sh=1, sw=1, pt=0, ph=1, pw=1,
             To=1, Ho=28, Wo=28)
    a.update(args)
    vals = list(a.values())
    rc = _lib.load().b2_avgpool_ndhwc_slice_exclude_pad(ctypes.c_void_p(vals[0]), vals[1], ctypes.c_void_p(vals[2]), *vals[3:],
                                                        ctypes.c_void_p(0))
    assert rc == B2_ERR_INVALID, (case, rc, _lib.last_error())
