"""CPU: Xception against the reference, as recorded in the fixtures (tests/golden/xception_b2_299.pt, xception_b2_224.pt and
trn_xception_MSTRN.pt, written by oracle/make_golden_xception.py from the unmodified reference): state_dict keys, shapes and order,
a seeded init bit-identical to the reference's, the ``rep`` layout, the registry row, both checkpoint layouts through the factory,
the oracle against the reference's stages, features and logits, TRN on Xception (2048-d frame features, policies, the fine_tune
refusal), the refusals, the new C entry's declaration and compiled instance, the wrapper's argument checks and the
``ops_xception`` audit registration (no GPU needed)."""
import ast
import inspect
import os
import re

import pytest
import torch

import pretorched_x_b200 as P
from pretorched_x_b200 import _lib, engine, ops, ops_xception
from pretorched_x_b200.models import xception as MX
from oracle import functional as OF
from oracle import xception as OXc
from oracle.make_golden import sample_of
from tests import model_audit as MA
from tests import xception_audit as XA

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_STATE, N_PARAMS = 276, 22855952
SIZES = (299, 224)


def _load(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


@pytest.mark.parametrize("hw", SIZES)
def test_state_dict_layout_and_seeded_init_match_reference(hw):
    fx = _load("xception_b2_%d.pt" % hw)
    torch.manual_seed(fx["seeds"]["init"])
    model = P.xception(pretrained=None, **fx["kwargs"])
    sd = model.state_dict()
    assert len(sd) == N_STATE == fx["n_state"] and sum(p.numel() for p in model.parameters()) == N_PARAMS
    assert [(k, tuple(v.shape)) for k, v in sd.items()] == [tuple(kv) for kv in fx["keys"]]
    assert OF.digests_match(OF.state_digest(sd), fx["init_digest"])
    assert list(sd)[-2:] == ["last_linear.weight", "last_linear.bias"] and not hasattr(model, "fc")


def test_rep_indices_and_skips_follow_the_reference():
    """The parameter-free slots keep their indices: block1 (start_with_relu=False) starts with its separable convolution, the
    other blocks with a ReLU that is not in place, and the strided blocks end with MaxPool2d(3, 2, 1)."""
    m = P.xception(pretrained=None)
    kinds = lambda b: [type(x).__name__ for x in b.rep]
    assert kinds(m.block1) == ["SeparableConv2d", "BatchNorm2d", "ReLU", "SeparableConv2d", "BatchNorm2d", "MaxPool2d"]
    assert kinds(m.block4) == ["ReLU", "SeparableConv2d", "BatchNorm2d"] * 3
    assert kinds(m.block12) == ["ReLU", "SeparableConv2d", "BatchNorm2d"] * 2 + ["MaxPool2d"]
    assert not m.block2.rep[0].inplace and m.block2.rep[3] is m.block2.relu and m.block2.relu.inplace
    assert [m.block12.rep[i].pointwise.out_channels for i in (1, 4)] == [728, 1024]
    for i in range(1, 13):
        blk = getattr(m, "block%d" % i)
        assert (blk.skip is not None) == (i in (1, 2, 3, 12))
        seps, pool = engine._xception_rep(blk)
        assert len(seps) == (3 if 4 <= i <= 11 else 2) and (pool is not None) == (blk.skip is not None)
        # a ReLU opens every separable convolution except block1's first (start_with_relu=False)
        assert [relu for _, _, relu in seps] == [i != 1] + [True] * (len(seps) - 1)
    assert list(dict(m.named_children())) == ["conv1", "bn1", "relu", "conv2", "bn2"] + ["block%d" % i for i in range(1, 13)] + \
        ["conv3", "bn3", "conv4", "bn4", "last_linear"]


def test_a_rep_layout_the_engine_does_not_run_is_refused():
    blk = MX.Block(64, 64, 2, 1)
    blk.rep = torch.nn.Sequential(*list(blk.rep)[:-1])          # a repetition without its BatchNorm
    with pytest.raises(NotImplementedError, match="as the reference builds them"):
        engine._xception_rep(blk)
    blk = MX.Block(64, 128, 2, 1)                                 # a projection skip without the pool
    with pytest.raises(NotImplementedError, match="as the reference builds them"):
        engine._xception_rep(blk)


def test_pretrained_settings_row_and_registry():
    fx = _load("xception_b2_299.pt")
    assert P.pretrained_settings["xception"] == fx["settings"]["xception"]
    assert "xception" in P.model_names and P.__dict__["xception"] is P.xception
    assert P.models.settings.model_names.count("xception") == 1
    assert inspect.signature(P.xception).parameters["pretrained"].default == "imagenet"
    assert P.xception(num_classes=10, pretrained=None).last_linear.out_features == 10


def _source():
    torch.manual_seed(5)
    src = P.xception(pretrained=None)
    OF.randomize_bn_(src, 6)
    return src


@pytest.mark.parametrize("layout", ["zoo", "reference"])
def test_checkpoint_loads_through_the_factory(monkeypatch, layout):
    """The zoo file names the head ``fc`` (xception.py:223-233 loads it before the rename); the reference's own state_dict names it
    ``last_linear``.  Both load."""
    import torch.utils.model_zoo as model_zoo
    want = _source().state_dict()
    if layout == "zoo":
        ckpt = {("fc." + k[len("last_linear."):] if k.startswith("last_linear.") else k): v.clone() for k, v in want.items()}
        assert "fc.weight" in ckpt and "last_linear.weight" not in ckpt
    else:
        ckpt = {k: v.clone() for k, v in want.items()}
    seen = []
    monkeypatch.setattr(model_zoo, "load_url", lambda url: seen.append(url) or dict(ckpt))
    m = P.xception()
    assert seen == ["http://pretorched-x.csail.mit.edu/models/xception-b429252d.pth"]
    got = m.state_dict()
    assert list(got) == list(want) and all(torch.equal(got[k], want[k]) for k in want)
    assert (m.input_space, m.input_range, m.mean, m.std, list(m.input_size)) == \
        ("RGB", [0, 1], [0.5, 0.5, 0.5], [0.5, 0.5, 0.5], [3, 299, 299])
    with pytest.raises(AssertionError, match="num_classes should be 1000"):
        P.xception(num_classes=10)


@pytest.mark.parametrize("hw", SIZES)
def test_oracle_reproduces_reference_stages_features_and_logits(hw):
    fx = _load("xception_b2_%d.pt" % hw)
    model = OXc.build_package_model(P, fx)
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    assert OF.digests_match(OF.state_digest(sd), fx["weight_digest"])
    x = OF.seeded_input(fx["input_shape"], fx["seeds"]["input"])
    stages = {}
    with torch.no_grad():
        feats = OXc.features(x, sd, stages)
        logits = OXc.logits(feats, sd)
    final = (hw - 3) // 2 - 1                           # conv1 (3x3 stride 2) and conv2 (3x3), both valid
    for _ in range(4):                                   # the MaxPool2d(3, 2, 1) of blocks 1-3 and 12
        final = (final - 1) // 2 + 1
    assert tuple(feats.shape) == tuple(fx["features"]["shape"]) == (2, 2048, final, final)
    s, step = sample_of(feats)
    assert step == fx["features"]["step"] and torch.equal(s, fx["features"]["sample"])
    assert list(fx["stages"]) == ["stem"] + OXc.BLOCKS
    for name, summ in fx["stages"].items():
        s, step = sample_of(stages[name])
        assert tuple(stages[name].shape) == tuple(summ["shape"]) and step == summ["step"] and torch.equal(s, summ["sample"]), name
    assert torch.equal(logits, fx["logits"])


def _named(model, groups):
    names = {id(p): n for n, p in model.named_parameters()}
    return [dict(name=g['name'], lr_mult=g['lr_mult'], decay_mult=g['decay_mult'], params=[names[id(p)] for p in g['params']])
            for g in groups]


def test_trn_builds_with_2048d_frame_features_and_refuses_fine_tune():
    fx = _load("trn_xception_MSTRN.pt")
    m = OXc.build_package_model(P, fx)
    assert OF.digests_match(OF.state_digest(m.state_dict()), fx["weight_digest"])
    assert m.frame_feature_dim == fx["frame_feature_dim"] == 2048
    assert list(m.input_size) == fx["input_size"] == [299, 299] and m.crop_size == [299, 299]
    assert isinstance(m.base_model.last_linear, torch.nn.Dropout)
    with pytest.raises(NotImplementedError, match="has none"):
        m.fine_tune(4)
    assert P.trn(num_classes=10, arch="xception", pretrained=None).frame_feature_dim == 2048


@pytest.mark.parametrize("pbn", [True, False])
def test_trn_optim_policies_match_reference(pbn):
    fx = _load("trn_xception_MSTRN.pt")
    model = P.TRN(10, num_segments=fx["segments"], arch="xception", consensus="MSTRN", pretrained=None, **fx["kwargs"])
    model.partialBN(pbn)
    got = _named(model, model.get_optim_policies())
    assert got == fx["policies"][pbn]
    if pbn:
        assert got[0]["params"] == ["base_model.conv1.weight"] and got[4]["params"] == ["base_model.bn1.weight", "base_model.bn1.bias"]


def test_training_mode_and_small_inputs_are_refused():
    m = P.xception(pretrained=None)
    with pytest.raises(RuntimeError, match="inference-only"):
        m.features(torch.zeros(1, 3, 299, 299))
    m.eval()
    a = ops.Act(torch.zeros((6 * 9, 8), dtype=torch.float16), 1, 1, 6, 9, 3)
    with pytest.raises(ValueError, match="at least 7x7"):
        m.features_act(a)
    with pytest.raises(NotImplementedError, match="inside its Xception block"):
        m.conv3(torch.zeros(1, 1024, 3, 3))


# ---------------------------------------------------------------------------------------------
# the C entry, its wrapper and its audit
# ---------------------------------------------------------------------------------------------
def test_entry_is_declared_and_bound():
    with open(os.path.join(ROOT, "include", "b2_pretorched.h")) as f:
        header = f.read()
    assert re.search(r"int b2_dwconv3x3_relu_in_ndhwc\(const void\* x, const float\* w, void\* y, int N, int H, int W, int C, int ld, "
                     r"void\* stream\);", header)
    assert re.search(r"int b2_dwconv3x3_ndhwc\(const void\* x, const float\* w, const float\* scale, const float\* shift, void\* y, "
                     r"int N, int H, int W, int C,\s+int ld, int stride, int clamp_in, int relu6, void\* stream\);", header)
    assert "b2_dwconv3x3_relu_in_ndhwc" in _lib.SYMBOLS


def test_depthwise_instances_compile_for_sm90a_without_spills():
    from pretorched_x_b200.csrc import build
    build.build()
    with open(os.path.join(os.path.dirname(build.LIB), "build.log")) as f:
        log = f.read()
    for inst in ("ILi1ELi4ELb1EE", "ILi1ELi4ELb0EE", "ILi2ELi2ELb0EE"):
        m = re.search(r"Compiling entry function '_ZN2b216dwconv3x3_kernel%s[^']*' for 'sm_90a'\n[^\n]*\n\s*(\d+) bytes stack frame, "
                      r"(\d+) bytes spill stores, (\d+) bytes spill loads" % inst, log)
        assert m, "dwconv3x3_kernel %s not in the build log" % inst
        assert m.groups() == ("0", "0", "0"), (inst, m.groups())


def test_c_entry_refuses_bad_arguments():
    lib = _lib.load()
    buf = torch.zeros(64, dtype=torch.float32)
    p = buf.data_ptr()
    assert lib.b2_dwconv3x3_relu_in_ndhwc(None, p, p, 1, 4, 4, 8, 8, None) == -1
    assert "null" in _lib.last_error()
    assert lib.b2_dwconv3x3_relu_in_ndhwc(p, p, p, 1, 4, 4, 12, 16, None) == -1        # C % 8 != 0
    assert lib.b2_dwconv3x3_relu_in_ndhwc(p, p, p, 1, 4, 4, 16, 8, None) == -1         # ld < C
    assert lib.b2_dwconv3x3_relu_in_ndhwc(p, p, p, 1, 0, 4, 8, 8, None) == -1          # empty
    assert lib.b2_dwconv3x3_relu_in_ndhwc(p + 4, p, p, 1, 4, 4, 8, 8, None) == -1      # misaligned


def test_wrapper_validates_its_arguments():
    w = torch.zeros((9, 728), dtype=torch.float32)
    a = ops.Act(torch.zeros((2 * 5 * 5, 728), dtype=torch.float16), 2, 1, 5, 5, 728)
    with pytest.raises(RuntimeError, match="CUDA"):
        ops_xception.dwconv3x3_relu_in(a, w)
    bad = ops.Act(torch.zeros((50, 736), dtype=torch.float16), 2, 1, 5, 5, 730)
    with pytest.raises(ValueError, match="C % 8 == 0"):
        ops_xception.dwconv3x3_relu_in(bad, torch.zeros((9, 730)))
    clip = ops.Act(torch.zeros((100, 728), dtype=torch.float16), 2, 2, 5, 5, 728)
    with pytest.raises(ValueError, match="images"):
        ops_xception.dwconv3x3_relu_in(clip, w)
    for w_bad in (torch.zeros((728, 9)), torch.zeros((9, 728), dtype=torch.float64), torch.zeros((9, 1456))[:, ::2]):
        with pytest.raises(ValueError, match=r"fp32 \[9\]\[728\]"):
            ops_xception.dwconv3x3_relu_in(a, w_bad)


def test_every_launching_entry_of_ops_xception_is_audited():
    """Every function of pretorched_x_b200/ops_xception.py whose body calls ``_lib.check(`` is in tests/xception_audit.py's table,
    with a check and exactly the parameters of its signature; nothing of it is also an entry of ``ops``."""
    with open(ops_xception.__file__) as f:
        tree = ast.parse(f.read())
    launching = {node.name for node in ast.walk(tree) if isinstance(node, ast.FunctionDef)
                 and any(isinstance(c, ast.Call) and isinstance(c.func, ast.Attribute) and c.func.attr == "check"
                         and isinstance(c.func.value, ast.Name) and c.func.value.id == "_lib" for c in ast.walk(node))}
    assert launching == set(XA.ENTRIES) == set(XA.CHECKS) == {"dwconv3x3_relu_in"}
    for name, params in XA.ENTRIES.items():
        assert tuple(inspect.signature(getattr(ops_xception, name)).parameters) == params
        assert not hasattr(ops, name) and name not in MA.KNOWN


def test_depthwise_check_catches_one_corrupted_element_and_passes_the_rounded_reference():
    g = torch.Generator().manual_seed(0)
    B, H, W, C, ld = 2, 5, 7, 16, 24
    x = (torch.randn(B, H, W, C, generator=g) * 3).half()
    w9 = torch.randn(9, C, generator=g) * 0.3
    ref, _ = XA.dw_relu_in_ref(x, w9)
    y = torch.zeros((B * H * W, ld), dtype=torch.float16)
    y[:, :C] = ref.half()
    x2d = torch.zeros((B * H * W, ld), dtype=torch.float16)
    x2d[:, :C] = x.reshape(-1, C)
    assert XA.check_dwconv_relu_in(x2d, B, H, W, C, w9, y)[0] <= 1.0
    signed = y.clone()                                   # the signed input read without the ReLU
    one, zero = torch.ones(C), torch.zeros(C)
    from tests import kernel_ref as KR
    signed[:, :C] = KR.dw_ref(x, w9, one, zero, 1, False, False)[0].half()
    assert XA.check_dwconv_relu_in(x2d, B, H, W, C, w9, signed)[0] > 1.0
    bad = y.clone()
    bad[11, 5] = float(bad[11, 5]) * 1.01 + 0.01
    r, where = XA.check_dwconv_relu_in(x2d, B, H, W, C, w9, bad)
    assert r > 1.0 and "row 11 col 5" in where
    pad = y.clone()
    pad[3, C] = 1.0
    assert XA.check_dwconv_relu_in(x2d, B, H, W, C, w9, pad)[0] == float("inf")
