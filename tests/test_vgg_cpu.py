"""CPU: VGG and AlexNet against the reference, as recorded in the fixtures (tests/golden/{vgg16,vgg16_bn,vgg11,alexnet}_b2_224.pt
and trn_{vgg16,alexnet}_MSTRN.pt, written by oracle/make_golden_vgg.py from the unmodified reference): state_dict keys, shapes and
order, a seeded init bit-identical to the reference's, the registry rows, both checkpoint layouts through the factories, the oracle
against the reference's features and logits, the space-to-depth form of AlexNet's conv1 and the (h, w, c) form of fc6 in fp64, the
split-K planner, TRN on both families, the refusals, the new C entries' declarations and compiled instances, and the ``ops_vgg``
audit registration (no GPU needed)."""
import ast
import inspect
import os
import re

import pytest
import torch
import torch.nn.functional as F

import pretorched_x_b200 as P
from pretorched_x_b200 import _lib, ops, ops_vgg
from pretorched_x_b200.models import vgg as MV
from oracle import functional as OF
from oracle import vgg as OV
from tests import model_audit as MA
from tests import vgg_audit as VA

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURES = ("vgg16", "vgg16_bn", "vgg11", "alexnet")
ARCHS = ("vgg11", "vgg11_bn", "vgg13", "vgg13_bn", "vgg16", "vgg16_bn", "vgg19", "vgg19_bn", "alexnet")


def _load(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


def _build(fx):
    torch.manual_seed(fx["seeds"]["init"])
    return getattr(P, fx["arch"])(pretrained=None, **fx["kwargs"])


@pytest.mark.parametrize("arch", FIXTURES)
def test_state_dict_layout_and_seeded_init_match_reference(arch):
    fx = _load("%s_b2_224.pt" % arch)
    sd = _build(fx).state_dict()
    assert len(sd) == fx["n_state"]
    assert [(k, tuple(v.shape)) for k, v in sd.items()] == [tuple(kv) for kv in fx["keys"]]
    assert OF.digests_match(OF.state_digest(sd), fx["init_digest"])
    assert list(sd)[0] == "_features.0.weight" and list(sd)[-1] == "last_linear.bias"


def test_module_names_follow_the_reference():
    assert list(dict(P.vgg16(pretrained=None).named_children())) == \
        ["avgpool", "_features", "linear0", "relu0", "dropout0", "linear1", "relu1", "dropout1", "last_linear"]
    assert list(dict(P.alexnet(pretrained=None).named_children())) == \
        ["avgpool", "_features", "dropout0", "linear0", "relu0", "dropout1", "linear1", "relu1", "last_linear"]


def test_pretrained_settings_rows_match_reference():
    for arch in FIXTURES:
        fx = _load("%s_b2_224.pt" % arch)
        assert P.pretrained_settings[arch] == fx["settings"][arch]
    row = P.pretrained_settings["alexnet"]["places365"]
    assert row["num_classes"] == 365 and row["url"] == "http://pretorched-x.csail.mit.edu/models/alexnet_places365-0c3a7b83.pth"
    for arch in ARCHS:
        assert arch in P.model_names and callable(P.__dict__[arch]) and P.pretrained_settings[arch]["imagenet"]["num_classes"] == 1000


@pytest.mark.parametrize("arch,keys", [("vgg11_bn", {"0": "linear0", "3": "linear1", "6": "last_linear"}),
                                       ("alexnet", {"1": "linear0", "4": "linear1", "6": "last_linear"})])
def test_both_checkpoint_layouts_load_through_the_factory(monkeypatch, arch, keys):
    import torch.utils.model_zoo as model_zoo
    torch.manual_seed(5)
    src = getattr(P, arch)(pretrained=None)
    OF.randomize_bn_(src, 6)
    want = src.state_dict()
    inv = {v: k for k, v in keys.items()}
    tv = {}
    for k, v in want.items():               # torchvision's layout: features.*, classifier.<i>.*
        head = k.split(".")[0]
        tv[k[1:] if k.startswith("_features.") else "classifier.%s.%s" % (inv[head], k.split(".", 1)[1])] = v.clone()
    for layout in (tv, want):
        seen = []
        monkeypatch.setattr(model_zoo, "load_url", lambda url, layout=layout: seen.append(url) or {k: v.clone() for k, v in layout.items()})
        torch.manual_seed(7)
        m = getattr(P, arch)()
        assert seen == [P.pretrained_settings[arch]["imagenet"]["url"]]
        got = m.state_dict()
        assert list(got) == list(want) and all(torch.equal(got[k], want[k]) for k in want)
        assert (m.input_space, m.input_range, m.mean, m.std, list(m.input_size)) == \
            ("RGB", [0, 1], [0.485, 0.456, 0.406], [0.229, 0.224, 0.225], [3, 224, 224])
    with pytest.raises(AssertionError, match="num_classes should be 1000"):
        getattr(P, arch)(num_classes=10)


def test_places365_alexnet_and_num_classes():
    import torch.utils.model_zoo as model_zoo
    src = P.alexnet(num_classes=365, pretrained=None)
    assert src.last_linear.out_features == 365
    # the reference's VGG factories ignore num_classes without a checkpoint; here it is honoured
    assert P.vgg16(num_classes=10, pretrained=None).last_linear.out_features == 10
    sd = src.state_dict()
    orig = model_zoo.load_url
    model_zoo.load_url = lambda url: {k: v.clone() for k, v in sd.items()}
    try:
        m = P.alexnet(num_classes=365, pretrained="places365")
    finally:
        model_zoo.load_url = orig
    assert m.last_linear.out_features == 365 and torch.equal(m.last_linear.weight, src.last_linear.weight)


@pytest.mark.parametrize("arch", FIXTURES)
def test_oracle_reproduces_reference_features_and_logits(arch):
    fx = _load("%s_b2_224.pt" % arch)
    model = _build(fx)
    OF.randomize_bn_(model, fx["seeds"]["bn"])
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    assert OF.digests_match(OF.state_digest(sd), fx["weight_digest"])
    x = OF.seeded_input(fx["input_shape"], fx["seeds"]["input"])
    stages = {}
    with torch.no_grad():
        feats = OV.features(x, sd, arch, stages)
        logits = OV.logits(feats, sd)
    assert torch.equal(feats, fx["features"]) and torch.equal(logits, fx["logits"])
    assert list(stages) == list(fx["stages"])
    # every stage far inside fp16's range at the seeded init (no rescaling needed)
    assert all(1e-2 < s["absmax"] < 1024 for s in fx["stages"].values())


@pytest.mark.parametrize("H,W", [(224, 224), (227, 227), (35, 41), (199, 241)])
def test_conv1_equals_valid_3x3_over_space_to_depth_fp64(H, W):
    g = torch.Generator().manual_seed(H * W)
    x = torch.randn((2, 3, H, W), generator=g, dtype=torch.float64)
    w = torch.randn((8, 3, 11, 11), generator=g, dtype=torch.float64)
    want = F.conv2d(x, w, stride=4, padding=2)
    Ho, Wo, Hs, Ws = ops_vgg.s2d_extent(H, W)
    s = _s2d64(x)
    got = F.conv2d(s.reshape(2, Hs, Ws, 48).permute(0, 3, 1, 2), ops_vgg.s2d_filter(w))
    assert got.shape == want.shape == (2, 8, Ho, Wo)
    assert torch.allclose(got, want, rtol=1e-12, atol=1e-10)


def _s2d64(x):
    """s2d_ref's rearrangement without its fp16 rounding."""
    N, C, H, W = x.shape
    _, _, Hs, Ws = ops_vgg.s2d_extent(H, W)
    xp = x.new_zeros((N, C, 4 * Hs, 4 * Ws))
    h1, w1 = min(H, 4 * Hs - 2), min(W, 4 * Ws - 2)
    xp[:, :, 2:2 + h1, 2:2 + w1] = x[:, :, :h1, :w1]
    return xp.reshape(N, C, Hs, 4, Ws, 4).permute(0, 2, 4, 3, 5, 1).reshape(N * Hs * Ws, 16 * C)


@pytest.mark.parametrize("C,H", [(512, 7), (256, 6)])
def test_fc6_on_hwc_flatten_with_permuted_weight_fp64(C, H):
    g = torch.Generator().manual_seed(C)
    fmap = torch.randn((3, C, H, H), generator=g, dtype=torch.float64)
    lin = torch.nn.Linear(C * H * H, 64).double()
    want = lin(fmap.view(3, -1))
    wp = lin.weight.detach().reshape(64, C, H, H).permute(0, 2, 3, 1).reshape(64, H * H * C)
    rows = fmap.permute(0, 2, 3, 1).reshape(3 * H * H, C)         # the engine's [N*H*W][C] map
    got = rows.view(3, H * H * C) @ wp.t() + lin.bias.detach()
    assert torch.allclose(got, want, rtol=1e-12, atol=1e-10)


def test_splitk_planner():
    plan = lambda M, N, K: _lib.load().b2_gemm_splitk_plan(M, N, K, 132)   # noqa: E731
    # fc6 (VGG 25088, AlexNet 9216), fc7 and the 1000 / 365-class heads at the batches the classifier runs at
    assert [plan(M, 4096, 25088) for M in (2, 16, 128, 256)] == [4, 4, 4, 2]
    assert [plan(M, 4096, 9216) for M in (2, 16, 128, 256)] == [4, 4, 4, 2]
    assert [plan(M, 4096, 4096) for M in (2, 16, 128, 256)] == [4, 4, 4, 2]
    assert [plan(M, 1000, 4096) for M in (2, 16, 128, 256)] == [8, 8, 8, 8]
    assert [plan(M, 365, 4096) for M in (2, 16, 128, 256)] == [8, 8, 8, 8]
    # no split: the output tiles fill the SMs, or K is too short to keep 8 K blocks per split
    assert plan(4096, 4096, 4096) == 1 and plan(256 * 49, 512, 4608) == 1 and plan(2, 4096, 960) == 1 and plan(2, 64, 64) == 1
    assert plan(0, 4096, 4096) < 0


def trn_as_reference(arch, fx):
    """The fixture's TRN with the reference's seeded weights.  TRN builds its backbone with 339 classes when ``pretrained=None``;
    the reference's VGG factories ignore that and draw a 1000-class ``last_linear`` (which TRN then replaces by Dropout), so the
    weights drawn after it differ unless the backbone is built the same way here."""
    orig = P.__dict__[arch]
    if arch.startswith("vgg"):
        P.__dict__[arch] = lambda num_classes=1000, pretrained='imagenet': orig(1000, pretrained)
    try:
        torch.manual_seed(fx["seeds"]["init"])
        return P.TRN(10, num_segments=fx["segments"], arch=arch, consensus="MSTRN", pretrained=None, **fx["kwargs"])
    finally:
        P.__dict__[arch] = orig


def test_trn_builds_with_4096d_frame_features_and_refuses_fine_tune():
    for arch in ("vgg16", "alexnet"):
        fx = _load("trn_%s_MSTRN.pt" % arch)
        m = trn_as_reference(arch, fx)
        OF.randomize_bn_(m, fx["seeds"]["bn"])
        assert OF.digests_match(OF.state_digest(m.state_dict()), fx["weight_digest"])
        assert m.frame_feature_dim == 4096 and list(m.input_size) == [224, 224]
        assert isinstance(m.base_model.last_linear, torch.nn.Dropout)
        with pytest.raises(NotImplementedError, match="has none"):
            m.fine_tune(4)


@pytest.mark.parametrize("arch", ("vgg16", "alexnet"))
@pytest.mark.parametrize("pbn", [True, False])
def test_trn_optim_policies_match_reference(arch, pbn):
    fx = _load("trn_%s_MSTRN.pt" % arch)
    model = P.TRN(10, num_segments=fx["segments"], arch=arch, consensus="MSTRN", pretrained=None, **fx["kwargs"])
    model.partialBN(pbn)
    names = {id(p): n for n, p in model.named_parameters()}
    got = [dict(name=g['name'], lr_mult=g['lr_mult'], decay_mult=g['decay_mult'], params=[names[id(p)] for p in g['params']])
           for g in model.get_optim_policies()]
    assert got == fx["policies"][pbn]


@pytest.mark.parametrize("arch", ("vgg16_bn", "alexnet"))
def test_training_mode_partial_trunk_and_other_input_sizes_are_refused(arch):
    m = getattr(P, arch)(pretrained=None)
    with pytest.raises(RuntimeError, match="inference-only"):
        m.features(torch.zeros(1, 3, 224, 224))
    m.eval()
    for hw in ((256, 256), (224, 192), (227, 227)):
        with pytest.raises(ValueError, match="224x224"):
            m(torch.zeros(1, 3, *hw))
    with pytest.raises(NotImplementedError, match=r"features\[a:b\]"):
        m._features[0:3](torch.zeros(1, 3, 224, 224))


# ---------------------------------------------------------------------------------------------
# the C entries and their audit
# ---------------------------------------------------------------------------------------------
def test_entries_are_declared_and_bound():
    with open(os.path.join(ROOT, "include", "b2_pretorched.h")) as f:
        header = f.read()
    assert re.search(r"int b2_space_to_depth4_nchw\(const float\* x, void\* y, int N, int H, int W, void\* stream\);", header)
    assert re.search(r"int b2_gemm_splitk_f16\(const b2_gemm_args\* g, int splits, float\* ws, size_t ws_elems, void\* stream\);", header)
    assert re.search(r"int b2_gemm_splitk_plan\(int M, int N, int Kd, int sm_count\);", header)
    assert re.search(r"size_t b2_gemm_splitk_workspace_elems\(int M, int N, int splits\);", header)
    for sym in ("b2_space_to_depth4_nchw", "b2_gemm_splitk_f16", "b2_gemm_splitk_plan", "b2_gemm_splitk_workspace_elems"):
        assert sym in _lib.SYMBOLS


def test_new_kernels_compile_for_sm90a_without_spills():
    from pretorched_x_b200.csrc import build
    build.build()
    with open(os.path.join(os.path.dirname(build.LIB), "build.log")) as f:
        log = f.read()
    names = [r"_ZN2b212pgemm_kernelILi64ELi0ELi5EE[^']*", r"_ZN2b212pgemm_kernelILi128ELi0ELi5EE[^']*",
             r"_ZN2b220splitk_reduce_kernel[^']*", r"space_to_depth4_kernel"]
    for name in names:
        m = re.search(r"Compiling entry function '%s' for 'sm_90a'\n[^\n]*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                      r"(\d+) bytes spill loads" % name, log)
        assert m, "%s not in the build log" % name
        assert m.groups() == ("0", "0", "0"), (name, m.groups())


def test_every_launching_entry_of_ops_vgg_is_audited():
    """Every function of pretorched_x_b200/ops_vgg.py whose body calls ``_lib.check(`` is in tests/vgg_audit.py's table, with a
    check and exactly the parameters of its signature; nothing of it is also an entry of ``ops``."""
    with open(ops_vgg.__file__) as f:
        tree = ast.parse(f.read())
    launching = {node.name for node in ast.walk(tree) if isinstance(node, ast.FunctionDef)
                 and any(isinstance(c, ast.Call) and isinstance(c.func, ast.Attribute) and c.func.attr == "check"
                         and isinstance(c.func.value, ast.Name) and c.func.value.id == "_lib" for c in ast.walk(node))}
    assert launching == set(VA.ENTRIES) == set(VA.CHECKS) == {"space_to_depth4", "gemm_splitk"}
    for name, params in VA.ENTRIES.items():
        assert tuple(inspect.signature(getattr(ops_vgg, name)).parameters) == params
        assert not hasattr(ops, name) and name not in MA.KNOWN


def test_splitk_check_catches_one_corrupted_element_and_passes_the_rounded_reference():
    g = torch.Generator().manual_seed(0)
    M, N, K = 6, 20, 640
    a = torch.rand((M, K), generator=g).half()
    b = (torch.randn((N, K), generator=g) / 25).half()
    sc, sh = torch.rand(N, generator=g) + 0.5, torch.randn(N, generator=g) * 0.1
    v = torch.relu(sc.double() * (a.double() @ b.double().t()) + sh.double())
    d = torch.zeros((M, 24), dtype=torch.float16)
    d[:, :N] = v.half()
    assert VA.check_gemm_splitk(a, b, sc, sh, M, N, K, d, relu=True)[0] <= 1.0
    d32 = v.float()
    assert VA.check_gemm_splitk(a, b, sc, sh, M, N, K, d32, relu=True, out_f32=True)[0] <= 1.0
    bad = d.clone()
    bad[3, 7] = float(bad[3, 7]) * 1.01 + 0.01      # one split's partial lost or doubled moves one element like this
    r, where = VA.check_gemm_splitk(a, b, sc, sh, M, N, K, bad, relu=True)
    assert r > 1.0 and "row 3 col 7" in where
    pad = d.clone()
    pad[0, N] = 1.0
    assert VA.check_gemm_splitk(a, b, sc, sh, M, N, K, pad, relu=True)[0] == float("inf")


def test_space_to_depth_check_is_bit_exact():
    x = torch.randn((1, 3, 31, 29), generator=torch.Generator().manual_seed(2))
    y = VA.s2d_ref(x)
    assert VA.check_space_to_depth4(x, y)[0] == 0.0
    y2 = y.clone()
    y2[5, 11] = y2[5, 11] + 1
    assert VA.check_space_to_depth4(x, y2)[0] == float("inf")
    assert MV.pretrained_settings["alexnet"]["imagenet"]["url"].endswith("alexnet-owt-4df8aa71.pth")
