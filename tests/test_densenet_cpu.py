"""CPU: the DenseNets against the reference, as recorded in the fixtures (tests/golden/densenet{121,161}_b2_224.pt,
trn_densenet121_MSTRN.pt and trn_densenet_optim_policies.pt, written by oracle/make_golden_densenet.py from the unmodified
reference): state_dict keys, shapes and order, a seeded init bit-identical to the reference's, the registry rows, legacy-key
checkpoints through the factories, the oracle restatement against the reference's features and logits, TRN on densenet121 (its
policies, the fine_tune refusal), the slab slice plans of the dense layers' 3x3 convolutions, and the refusals of the new C entries
(no GPU needed)."""
import ctypes
import os

import pytest
import torch

import pretorched_x_b200 as P
from pretorched_x_b200 import _lib
from oracle import densenet as OD
from oracle import functional as OF
from oracle.make_golden import sample_of

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
B2_ERR_INVALID = -1
# (arch, state_dict entries, parameters, final features)
ARCHS = [("densenet121", 727, 7978856, 1024), ("densenet161", 967, 28681000, 2208), ("densenet169", 1015, 14149480, 1664),
         ("densenet201", 1207, 20013928, 1920)]
FIXTURES = ["densenet121", "densenet161"]


def _load(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


@pytest.mark.parametrize("arch", FIXTURES)
def test_state_dict_layout_and_seeded_init_match_reference(arch):
    fx = _load("%s_b2_224.pt" % arch)
    n_state, n_params = [a[1:3] for a in ARCHS if a[0] == arch][0]
    torch.manual_seed(fx["seeds"]["init"])
    model = P.__dict__[arch](pretrained=None, **fx["kwargs"])
    sd = model.state_dict()
    assert len(sd) == n_state == fx["n_state"] and sum(p.numel() for p in model.parameters()) == n_params
    assert [(k, tuple(v.shape)) for k, v in sd.items()] == [tuple(kv) for kv in fx["keys"]]
    assert OF.digests_match(OF.state_digest(sd), fx["init_digest"])


@pytest.mark.parametrize("arch,n_state,n_params,C", ARCHS)
def test_every_densenet_builds_with_the_reference_layout(arch, n_state, n_params, C):
    model = P.__dict__[arch](pretrained=None)
    sd = model.state_dict()
    assert len(sd) == n_state and sum(p.numel() for p in model.parameters()) == n_params
    assert model.last_linear.in_features == C and not hasattr(model, "classifier")
    assert list(sd)[-2:] == ["last_linear.weight", "last_linear.bias"]
    assert arch in P.model_names and P.pretrained_settings[arch]["imagenet"]["num_classes"] == 1000


@pytest.mark.parametrize("arch", FIXTURES)
def test_pretrained_settings_rows_match_reference(arch):
    fx = _load("%s_b2_224.pt" % arch)
    assert P.pretrained_settings[arch] == fx["settings"][arch]
    assert arch in P.model_names
    if arch == "densenet161":
        assert P.pretrained_settings[arch]["places365"]["num_classes"] == 365


def _legacy(sd):
    """A state dict in the checkpoints' old naming: 'norm.1' ... for the dense layers, 'classifier' for the head, and no
    num_batches_tracked entries (the checkpoints predate them)."""
    out = {}
    for k, v in sd.items():
        if k.endswith("num_batches_tracked"):
            continue
        for old, new in (("norm1", "norm.1"), ("norm2", "norm.2"), ("conv1", "conv.1"), ("conv2", "conv.2")):
            if ".denselayer" in k and ("." + old + ".") in k:
                k = k.replace("." + old + ".", "." + new + ".")
        out[k.replace("last_linear.", "classifier.")] = v.clone()
    return out


@pytest.mark.parametrize("arch,row,classes", [("densenet121", "imagenet", 1000), ("densenet161", "places365", 365)])
def test_legacy_checkpoint_loads_through_the_factory(monkeypatch, arch, row, classes):
    torch.manual_seed(5)
    src = P.__dict__[arch](num_classes=classes, pretrained=None)
    OF.randomize_bn_(src, 6)
    ckpt = _legacy(src.state_dict())
    assert any(".norm.1." in k for k in ckpt) and "classifier.weight" in ckpt
    import torch.utils.model_zoo as model_zoo
    seen = []
    monkeypatch.setattr(model_zoo, "load_url", lambda url: seen.append(url) or dict(ckpt))
    torch.manual_seed(7)
    m = P.__dict__[arch](num_classes=classes, pretrained=row)
    assert seen == [P.pretrained_settings[arch][row]["url"]]
    got, want = m.state_dict(), src.state_dict()
    assert list(got) == list(want) and all(torch.equal(got[k], want[k]) for k in want)
    # preprocessing attributes are attached after a checkpoint load (the reference's DenseNet factories attach none)
    assert (m.input_space, m.input_range, m.mean, m.std, list(m.input_size)) == \
        ("RGB", [0, 1], [0.485, 0.456, 0.406], [0.229, 0.224, 0.225], [3, 224, 224])


@pytest.mark.parametrize("arch", FIXTURES)
def test_oracle_reproduces_reference_features_and_logits(arch):
    fx = _load("%s_b2_224.pt" % arch)
    model = OD.build_package_model(P, fx)
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    assert OF.digests_match(OF.state_digest(sd), fx["weight_digest"])
    x = OF.seeded_input(fx["input_shape"], fx["seeds"]["input"])
    stages = {}
    with torch.no_grad():
        feats = OD.features(x, sd, stages)
        logits = OD.logits(feats, sd)
    assert tuple(feats.shape) == tuple(fx["features"]["shape"])
    s, step = sample_of(feats)
    assert step == fx["features"]["step"] and torch.equal(s, fx["features"]["sample"])
    for name, summ in fx["stages"].items():
        s, step = sample_of(stages[name])
        assert tuple(stages[name].shape) == tuple(summ["shape"]) and step == summ["step"] and torch.equal(s, summ["sample"]), name
    assert torch.equal(logits, fx["logits"])


@pytest.mark.parametrize("arch,C", [(a[0], a[3]) for a in ARCHS])
def test_trn_builds_and_refuses_fine_tune(arch, C):
    m = P.TRN(10, num_segments=4, arch=arch, consensus="MSTRN", pretrained=None, frame_bottleneck_dim=128, video_feature_dim=64)
    assert m.frame_feature_dim == C
    assert isinstance(m.base_model.last_linear, torch.nn.Dropout)
    with pytest.raises(NotImplementedError, match="has none"):
        m.fine_tune(4)
    mod = P.trn(num_classes=10, arch=arch, pretrained=None)
    assert mod.frame_feature_dim == C


def _named(model, groups):
    names = {id(p): n for n, p in model.named_parameters()}
    return [dict(name=g['name'], lr_mult=g['lr_mult'], decay_mult=g['decay_mult'], params=[names[id(p)] for p in g['params']])
            for g in groups]


@pytest.mark.parametrize("pbn", [True, False])
def test_trn_optim_policies_match_reference(pbn):
    fx = _load("trn_densenet_optim_policies.pt")["cases"]["densenet121_MSTRN"]
    model = P.TRN(10, num_segments=fx["segments"], arch=fx["arch"], consensus=fx["consensus"], pretrained=None, **fx["kwargs"])
    model.partialBN(pbn)
    got = _named(model, model.get_optim_policies())
    assert got == fx["policies"][pbn]
    if pbn:
        assert got[4]["params"] == ["base_model.features.norm0.weight", "base_model.features.norm0.bias"]


def test_partial_features_refuse_to_run():
    m = P.densenet121(pretrained=None).eval()
    part = m.features[4:6]
    assert type(part) is type(m.features) and len(part) == 2
    with pytest.raises(NotImplementedError, match="whole trunk"):
        part(torch.zeros(1, 64, 56, 56))


def _conv_args(N, C, H, K, ldy):
    a = _lib.ConvArgs()
    a.N, a.T, a.H, a.W, a.C, a.K, a.ldy = N, 1, H, H, C, K, ldy
    a.kt, a.kh, a.kw, a.st, a.sh, a.sw, a.pt, a.ph, a.pw = 1, 3, 3, 1, 1, 1, 0, 1, 1
    a.mode = _lib.B2_CONV_AUTO
    return a


# the growth-rate 3x3 convolutions of every DenseNet: 4k -> k at the four block resolutions
GROWTH = [(C, H, K) for C, K in ((128, 32), (192, 48)) for H in (56, 28, 14, 7)]


@pytest.mark.parametrize("C,H,K", GROWTH)
@pytest.mark.parametrize("N", [2, 256])
def test_growth_convolutions_have_a_slice_plan(C, H, K, N):
    out = (ctypes.c_int * 10)()
    fn = _lib.load().b2_debug_slab_slice_plan
    fn.argtypes = [ctypes.POINTER(_lib.ConvArgs), ctypes.POINTER(ctypes.c_int)]
    assert fn(ctypes.byref(_conv_args(N, C, H, K, K)), out) == 0
    assert out[0] == 1 and out[1] >= K, tuple(out)


def _plan_view(entry, a):
    out = (ctypes.c_int * 10)()
    fn = getattr(_lib.load(), entry)
    fn.argtypes = [ctypes.POINTER(_lib.ConvArgs), ctypes.POINTER(ctypes.c_int)]
    assert fn(ctypes.byref(a), out) == 0
    return tuple(out)


@pytest.mark.parametrize("C,H,K", GROWTH)
@pytest.mark.parametrize("N", [2, 32, 256])
def test_growth_convolutions_have_a_narrow_plan(C, H, K, N):
    """b2_conv_ndhwc_fprop_slice_narrow plans one N tile exactly K wide (the runtime-N instance), within the register budget."""
    plan = _plan_view("b2_debug_slab_slice_narrow_plan", _conv_args(N, C, H, K, K))
    assert plan[0] == 1 and plan[1] == K and plan[8] == 1 and plan[1] * plan[2] <= 192, plan


@pytest.mark.parametrize("C,H,K", GROWTH + [(32, 149, 32), (8, 299, 32), (48, 35, 64)])
def test_slice_entry_keeps_the_64_wide_tile(C, H, K):
    """The plain slice entry's planner is unchanged: outputs of at most 64 channels (the growth convolutions, Inception-v4's
    32-channel stem convolutions) keep the 64-wide tile; only the narrow entry takes the k-wide one."""
    plan = _plan_view("b2_debug_slab_slice_plan", _conv_args(128, C, H, K, K))
    assert plan[0] == 1 and plan[1] == 64 and plan[8] == 0, plan


def test_narrow_slice_refuses_other_widths():
    a = _conv_args(2, 128, 28, 64, 64)
    a.x, a.w, a.scale, a.shift, a.y = (ctypes.c_void_p(v) for v in (0x10000, 0x20000, 0x30000, 0x40000, 0x50000))
    rc = _lib.load().b2_conv_ndhwc_fprop_slice_narrow(ctypes.byref(a), None)
    assert rc == B2_ERR_INVALID and "32 or 48" in _lib.last_error()


def _gemm_args(**kw):
    g = _lib.GemmArgs()
    g.a, g.b, g.scale, g.shift, g.d = (ctypes.c_void_p(v) for v in (0x10000, 0x20000, 0x30000, 0x40000, 0x50000))
    g.M, g.N, g.Kd, g.lda, g.ldb, g.ldd = 1000, 128, 96, 256, 96, 128
    for k, v in kw.items():
        setattr(g, k, v)
    return g


@pytest.mark.parametrize("case,kw,aff", [
    ("null A", dict(a=None), (0x60000, 0x70000)),
    ("null input affine", dict(), (0, 0x70000)),
    ("unaligned input affine", dict(), (0x60004, 0x70000)),
    ("Kd not a multiple of 8", dict(Kd=100, ldb=104), (0x60000, 0x70000)),
    ("lda < Kd", dict(lda=64), (0x60000, 0x70000)),
    ("residual", dict(residual=ctypes.c_void_p(0x80000), ldr=128), (0x60000, 0x70000)),
    ("fp32 output", dict(out_f32=1), (0x60000, 0x70000)),
    ("per-sample affine", dict(aff_ld=128, aff_rows=128), (0x60000, 0x70000)),
    ("mask", dict(mask=ctypes.c_void_p(0x80000), ldm=128), (0x60000, 0x70000)),
    ("ldd < N", dict(ldd=64), (0x60000, 0x70000)),
])
def test_preact_gemm_refusals(case, kw, aff):
    g = _gemm_args(**kw)
    rc = _lib.load().b2_gemm_preact_f16(ctypes.byref(g), ctypes.c_void_p(aff[0]), ctypes.c_void_p(aff[1]), None)
    assert rc == B2_ERR_INVALID, (case, rc, _lib.last_error())


@pytest.mark.parametrize("case,args", [
    ("null input", (0, 256, 0x20000, 256, 2, 56, 56, 256, 0x30000, 0x40000)),
    ("null affine", (0x10000, 256, 0x20000, 256, 2, 56, 56, 256, 0, 0x40000)),
    ("C not a multiple of 8", (0x10000, 256, 0x20000, 256, 2, 56, 56, 252, 0x30000, 0x40000)),
    ("pitch below C", (0x10000, 128, 0x20000, 256, 2, 56, 56, 256, 0x30000, 0x40000)),
    ("unaligned output", (0x10000, 256, 0x20008, 256, 2, 56, 56, 256, 0x30000, 0x40000)),
    ("1-row map", (0x10000, 256, 0x20000, 256, 2, 1, 56, 256, 0x30000, 0x40000)),
])
def test_transition_pool_refusals(case, args):
    a = [ctypes.c_void_p(v) if i in (0, 2, 8, 9) else v for i, v in enumerate(args)]
    rc = _lib.load().b2_bn_relu_avgpool2_ndhwc(*a, None)
    assert rc == B2_ERR_INVALID, (case, rc, _lib.last_error())


@pytest.mark.parametrize("case,args", [
    ("null output", (0x10000, 0, 2, 49, 1024, 0x30000, 0x40000)),
    ("null affine", (0x10000, 0x20000, 2, 49, 1024, 0x30000, 0)),
    ("C not a multiple of 8", (0x10000, 0x20000, 2, 49, 1020, 0x30000, 0x40000)),
    ("no positions", (0x10000, 0x20000, 2, 0, 1024, 0x30000, 0x40000)),
])
def test_head_pool_refusals(case, args):
    a = [ctypes.c_void_p(v) if i in (0, 1, 5, 6) else v for i, v in enumerate(args)]
    rc = _lib.load().b2_avgpool_global_affine_ndhwc(*a, None)
    assert rc == B2_ERR_INVALID, (case, rc, _lib.last_error())
