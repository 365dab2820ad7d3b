"""CPU: PolyNet against the reference, as recorded in the fixtures (tests/golden/polynet_b2_331.pt and trn_polynet_MSTRN.pt,
written by oracle/make_golden_polynet.py from the unmodified reference): state_dict keys, shapes and order, a seeded init
bit-identical to the reference's, the registry row, the checkpoint through the factory, the oracle restatement against the
reference's features, module outputs and logits, the rescaled fixture init, TRN on PolyNet (its dims, policies, the fine_tune
refusal), the block table against the reference's modules, the 2-way and poly-3 closes restated as the engine computes them, the
new C entry's declarations, and its compiled instances (no GPU needed)."""
import os
import re

import pytest
import torch

import pretorched_x_b200 as P
from pretorched_x_b200 import _lib, ops, ops_dual
from pretorched_x_b200.models import polynet as PN
from oracle import functional as OF
from oracle import polynet as OP
from oracle.make_golden import sample_of
from tests import dual_audit as DA

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
N_STATE, N_PARAMS = 3104, 95366600


def _load(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


def test_state_dict_layout_and_seeded_init_match_reference():
    fx = _load("polynet_b2_331.pt")
    torch.manual_seed(fx["seeds"]["init"])
    model = P.polynet(pretrained=None, **fx["kwargs"])
    sd = model.state_dict()
    assert len(sd) == N_STATE == fx["n_state"] and sum(p.numel() for p in model.parameters()) == N_PARAMS == fx["n_params"]
    assert [(k, tuple(v.shape)) for k, v in sd.items()] == [tuple(kv) for kv in fx["keys"]]
    assert OF.digests_match(OF.state_digest(sd), fx["init_digest"])
    assert "stage_b.0.path0_1x7.bn_blocks.2.running_var" in sd and "stage_b.0.conv2d_blocks.2.bn.weight" in sd
    assert "stage_b.0.path0_1x7.conv.weight" in sd and "stage_b.0.path0_1x7.bn_blocks.3.weight" not in sd


def test_pretrained_settings_row_matches_reference():
    fx = _load("polynet_b2_331.pt")
    assert P.pretrained_settings["polynet"] == fx["settings"]["polynet"]
    assert "polynet" in P.model_names and P.__dict__["polynet"] is P.polynet


def test_checkpoint_loads_through_the_factory(monkeypatch):
    import torch.utils.model_zoo as model_zoo
    torch.manual_seed(5)
    src = P.polynet(pretrained=None)
    OF.randomize_bn_(src, 6)
    want = src.state_dict()
    seen = []
    monkeypatch.setattr(model_zoo, "load_url", lambda url: seen.append(url) or {k: v.clone() for k, v in want.items()})
    torch.manual_seed(7)
    m = P.polynet()
    assert seen == ["http://data.lip6.fr/cadene/pretrainedmodels/polynet-f71d82a5.pth"]
    got = m.state_dict()
    assert list(got) == list(want) and all(torch.equal(got[k], want[k]) for k in want)
    assert (m.input_space, m.input_range, m.mean, m.std, list(m.input_size)) == \
        ("RGB", [0, 1], [0.485, 0.456, 0.406], [0.229, 0.224, 0.225], [3, 331, 331])
    with pytest.raises(AssertionError, match="num_classes should be 1000"):
        P.polynet(num_classes=10)


def test_oracle_reproduces_reference_features_and_logits():
    fx = _load("polynet_b2_331.pt")
    model = OP.build_package_model(P, fx)
    sd = {k: v.detach().clone() for k, v in model.state_dict().items()}
    assert OF.digests_match(OF.state_digest(sd), fx["weight_digest"])
    x = OF.seeded_input(fx["input_shape"], fx["seeds"]["input"])
    stages = {}
    with torch.no_grad():
        feats = OP.features(x, sd, model, stages)
        logits = OP.logits(feats, sd)
    assert tuple(feats.shape) == tuple(fx["features"]["shape"]) == (2, 2048, 9, 9)
    s, step = sample_of(feats)
    assert step == fx["features"]["step"] and torch.equal(s, fx["features"]["sample"])
    assert list(fx["stages"]) == OP.module_names(model) and len(fx["stages"]) == 43
    for name, summ in fx["stages"].items():
        flat = stages[name].reshape(-1)
        assert tuple(stages[name].shape) == tuple(summ["shape"]), name
        assert torch.equal(flat[::summ["step"]][:summ["sample"].numel()], summ["sample"]), name
    assert torch.equal(logits, fx["logits"])


def test_fixture_init_moves_the_trunk_and_stays_in_fp16_range():
    """At the seeded default init the residual branches barely move the trunk; the fixtures' rescaled init
    (oracle.polynet.rescale_) makes every module's scaled branch sum a sizeable fraction of its input, with every activation far
    inside fp16's range (measured on the reference by oracle/make_golden_polynet.py)."""
    fx = _load("polynet_b2_331.pt")
    names = [r[0] for r in fx["report"]]
    assert len(names) == 40 and names[0] == "stage_a.0" and names[-1] == "stage_c.9"
    assert min(r[1] for r in fx["report"]) >= 0.15 and fx["peak"] < 1024
    assert max(s["absmax"] for s in fx["stages"].values()) < 1024


def test_trn_builds_and_refuses_fine_tune():
    fx = _load("trn_polynet_MSTRN.pt")
    m = OP.build_package_model(P, fx)
    assert OF.digests_match(OF.state_digest(m.state_dict()), fx["weight_digest"])
    assert m.frame_feature_dim == fx["frame_feature_dim"] == 2048
    assert list(m.input_size) == fx["input_size"] == [331, 331]
    assert isinstance(m.base_model.last_linear, torch.nn.Dropout)
    with pytest.raises(NotImplementedError, match="has none"):
        m.fine_tune(4)
    assert P.trn(num_classes=10, arch="polynet", pretrained=None).frame_feature_dim == 2048


@pytest.mark.parametrize("pbn", [True, False])
def test_trn_optim_policies_match_reference(pbn):
    fx = _load("trn_polynet_MSTRN.pt")
    model = P.TRN(10, num_segments=fx["segments"], arch=fx["arch"], consensus=fx["consensus"], pretrained=None, **fx["kwargs"])
    model.partialBN(pbn)
    names = {id(p): n for n, p in model.named_parameters()}
    got = [dict(name=g['name'], lr_mult=g['lr_mult'], decay_mult=g['decay_mult'], params=[names[id(p)] for p in g['params']])
           for g in model.get_optim_policies()]
    assert got == fx["policies"][pbn]


def test_training_mode_and_other_input_sizes_are_refused():
    m = P.polynet(pretrained=None)
    with pytest.raises(RuntimeError, match="inference-only"):
        m.features(torch.zeros(1, 3, 331, 331))
    m.eval()
    for hw in (299, 320):
        with pytest.raises(ValueError, match="331x331"):
            m(torch.zeros(1, 3, hw, hw))
    with pytest.raises(ValueError, match="AvgPool2d\\(9\\)"):
        m.logits(torch.zeros(1, 2048, 8, 8))


# ---------------------------------------------------------------------------------------------
# the block table against the reference's modules, and the closes as the engine computes them (fp64)
# ---------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def pair():
    """(package model, reference model) in fp64 holding the same rescaled weights and random BatchNorm statistics."""
    from oracle import reference_loader as RL
    torch.manual_seed(0)
    m = OP.rescale_(P.polynet(pretrained=None), 0.15)
    OF.randomize_bn_(m, 2)
    ref = RL.build("polynet", num_classes=1000)
    ref.load_state_dict(m.state_dict())
    return m.eval().double(), ref.eval().double()


def _x(C, H, seed=1):
    return torch.rand((1, C, H, H), generator=torch.Generator().manual_seed(seed), dtype=torch.float64) * 3


def _row_units(row):
    return [p for br in row if br[0] != "max" for p in br[1]]


def test_rows_name_every_unit_of_their_modules_once(pair):
    m, _ = pair
    for kind, mod in (("BlockA", m.stage_a[0].blocks[0]), ("BlockB", m.stage_b[1].blocks[0]), ("BlockC", m.stage_c[1].blocks[0]),
                      ("ReductionA", m.reduction_a), ("ReductionB", m.reduction_b)):
        units = _row_units(PN.BRANCHES[kind])
        convs = sorted(n[:-len(".conv")] for n, c in mod.named_modules() if isinstance(c, torch.nn.Conv2d))
        assert sorted(units + (["conv2d"] if kind.startswith("Block") else [])) == convs, kind
    stem = sorted(_row_units(PN.BRANCHES["Stem1"]) + _row_units(PN.BRANCHES["Stem2"]) + _row_units(PN.BRANCHES["Stem3"])
                  + ["conv1.%d" % i for i in range(3)])
    assert stem == sorted(n[:-len(".conv")] for n, c in m.stem.named_modules() if isinstance(c, torch.nn.Conv2d))
    # the reference's order, not Inception-v4's: (7, 1) before (1, 7) in conv2_long, the pool branch first in both stride-2 stages
    assert m.stem.conv2_long[1].conv.kernel_size == (7, 1) and m.stem.conv2_long[2].conv.kernel_size == (1, 7)
    assert PN.BRANCHES["Stem1"][0][0] == PN.BRANCHES["Stem3"][0][0] == "max"


@pytest.mark.parametrize("name,C,H", [("stem", 3, 75), ("reduction_a", 384, 15), ("reduction_b", 1152, 11)])
def test_rows_walked_by_the_oracle_equal_the_reference(pair, name, C, H):
    m, ref = pair
    sd = m.state_dict()
    x = _x(C, H)
    with torch.no_grad():
        want = ref.get_submodule(name)(x)
        got = OP.module(x, sd, m.get_submodule(name), name + ".")
    assert torch.equal(got, want)


@pytest.mark.parametrize("name,C,H", [("stage_a.3", 384, 9), ("stage_b.1", 1152, 7), ("stage_c.1", 2048, 5)])
def test_block_rows_and_2way_close_as_the_engine_computes_it(pair, name, C, H):
    """Each block's row walked by the oracle is the reference block's concatenation; the 2-way module restated as the engine runs
    it -- both concatenations into ONE two-operand product with s * (closing BatchNorm scale) folded into each filter, the shifts
    summed, x as residual, ReLU -- equals the reference module."""
    m, ref = pair
    sd = m.state_dict()
    mod, rmod = m.get_submodule(name), ref.get_submodule(name)
    x = _x(C, H)
    kind = type(mod.blocks[0]).__name__
    with torch.no_grad():
        cats = []
        for i, (b, rb) in enumerate(zip(mod.blocks, rmod.blocks)):
            cat = OP.branches(x, sd, b, "%s.blocks.%d." % (name, i), PN.BRANCHES[kind])
            paths = [rb.path0(x), rb.path1(x)] + ([rb.path2(x)] if hasattr(rb, "path2") else [])
            assert torch.equal(cat, torch.cat(paths, 1)), kind
            cats.append(cat)
        s, acc, shift = float(mod.scale), 0, 0
        for b, cat in zip(mod.blocks, cats):
            sb = (b.conv2d.bn.weight / torch.sqrt(b.conv2d.bn.running_var + b.conv2d.bn.eps)).double()
            tb = b.conv2d.bn.bias - b.conv2d.bn.running_mean * sb
            w = b.conv2d.conv.weight[:, :, 0, 0] * (s * sb)[:, None]
            acc = acc + torch.einsum("nchw,kc->nkhw", cat, w)
            shift = shift + s * tb
        got = torch.relu(acc + shift[None, :, None, None] + x)
        want = rmod(x)
    assert torch.allclose(got, want, rtol=1e-10, atol=1e-10 * float(want.abs().max()))


@pytest.mark.parametrize("name,C,H", [("stage_b.0", 1152, 7), ("stage_c.0", 2048, 5)])
def test_poly3_restated_with_the_dual_close_equals_the_reference(pair, name, C, H):
    """Poly-3 as the engine runs it: per application the branches, then from one accumulator d = (s sb) acc + s tb + running sum
    (the new running sum) and d2 = relu(sb acc + tb) (the next input); the last application d with ReLU."""
    m, ref = pair
    sd = m.state_dict()
    mod = m.get_submodule(name)
    x = _x(C, H)
    s = float(mod.scale)
    with torch.no_grad():
        total, xi = x, x
        for i in range(mod.num_blocks):
            rows = PN.BRANCHES[mod.kind]
            outs = []
            for br in rows:
                h = xi
                for p in br[1]:
                    h = OP.unit(h, sd, "%s.%s." % (name, p), mod.get_submodule(p).conv, bn="%s.%s.bn_blocks.%d." % (name, p, i))
                outs.append(h)
            cat = torch.cat(outs, 1)
            bn = mod.conv2d_blocks[i].bn
            sb = bn.weight / torch.sqrt(bn.running_var + bn.eps)
            tb = bn.bias - bn.running_mean * sb
            acc = torch.einsum("nchw,kc->nkhw", cat, mod.conv2d_blocks[i].conv.weight[:, :, 0, 0])
            d = (s * sb)[None, :, None, None] * acc + (s * tb)[None, :, None, None] + total
            d2 = torch.relu(sb[None, :, None, None] * acc + tb[None, :, None, None])
            total, xi = (d, d2) if i < mod.num_blocks - 1 else (torch.relu(d), None)
        want = ref.get_submodule(name)(x)
    assert torch.allclose(total, want, rtol=1e-10, atol=1e-10 * float(want.abs().max()))


# ---------------------------------------------------------------------------------------------
# the C entry
# ---------------------------------------------------------------------------------------------
def test_dual_gemm_entry_is_declared_bound_and_wrapped():
    with open(os.path.join(ROOT, "include", "b2_pretorched.h")) as f:
        header = f.read()
    assert re.search(r"int b2_gemm_dual_f16\(const b2_gemm_args\* a, const float\* scale2, const float\* shift2, void\* d2, int ldd2, "
                     r"void\* stream\);", header)
    assert "b2_gemm_dual_f16" in _lib.SYMBOLS and callable(ops_dual.gemm_dual)
    with open(os.path.join(ROOT, "pretorched_x_b200", "csrc", "b2_conv_api.cu")) as f:
        assert "int b2_gemm_dual_f16(" in f.read()


def test_dual_gemm_instances_compile_for_sm90a_without_spills():
    from pretorched_x_b200.csrc import build
    build.build()
    with open(os.path.join(os.path.dirname(build.LIB), "build.log")) as f:
        log = f.read()
    found = 0
    for bn in (64, 128):
        m = re.search(r"Compiling entry function '_ZN2b212pgemm_kernelILi%dELi0ELi4EE[^']*' for 'sm_90a'\n[^\n]*\n\s*(\d+) bytes stack "
                      r"frame, (\d+) bytes spill stores, (\d+) bytes spill loads" % bn, log)
        assert m, "pgemm_kernel<%d, 0, 4> not in the build log" % bn
        assert m.groups() == ("0", "0", "0"), m.groups()
        found += 1
    assert found == 2


def test_every_launching_entry_of_ops_dual_is_audited():
    """Every function of pretorched_x_b200/ops_dual.py whose body calls ``_lib.check(`` is in tests/dual_audit.py's table, with
    a check and exactly the parameters of its signature; nothing of it is also an entry of ``ops``."""
    import ast
    import inspect
    from tests import model_audit as MA
    with open(ops_dual.__file__) as f:
        tree = ast.parse(f.read())
    launching = {node.name for node in ast.walk(tree) if isinstance(node, ast.FunctionDef)
                 and any(isinstance(c, ast.Call) and isinstance(c.func, ast.Attribute) and c.func.attr == "check"
                         and isinstance(c.func.value, ast.Name) and c.func.value.id == "_lib" for c in ast.walk(node))}
    assert launching == set(DA.ENTRIES) == set(DA.CHECKS) == {"gemm_dual"}
    for name, params in DA.ENTRIES.items():
        assert tuple(inspect.signature(getattr(ops_dual, name)).parameters) == params
        assert not hasattr(ops, name) and name not in MA.ENTRIES


def test_dual_check_catches_a_wrong_second_output_and_passes_the_rounded_reference():
    g = torch.Generator().manual_seed(0)
    M, N, K = 40, 24, 16
    a = torch.rand((M, K), generator=g).half()
    b = torch.randn((N, K), generator=g).half()
    sb, tb = torch.rand(N, generator=g) + 0.5, torch.randn(N, generator=g) * 0.1
    sc, sh = 0.9 * sb, 0.9 * tb
    res = torch.randn((M, N), generator=g).half()
    acc = a.double() @ b.double().t()
    d = (sc.double() * acc + sh.double() + res.double()).half()
    d2 = torch.relu(sb.double() * acc + tb.double()).half()
    assert DA.check_gemm_dual(a, b, sc, sh, sb, tb, M, N, K, d, d2, residual=res)[0] <= 1.0
    wrong = torch.relu(d.double() * sb.double() + tb.double()).half()      # the generator's second output: of d, not of acc
    r, where = DA.check_gemm_dual(a, b, sc, sh, sb, tb, M, N, K, d, wrong, residual=res)
    assert r > 1.0 and "d2" in where
