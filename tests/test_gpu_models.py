"""GPU (-m gpu): whole-network parity against the reference's outputs (tests/golden, produced by the unmodified
reference) and against the CPU oracle, plus size-independent properties at the BASELINE clip size.

Stated tolerances (fp16 activations, fp32 accumulation; relative to max|reference| of the tensor):
  * per-stage samples <= 1e-2, logits <= 5e-3, arg-max must agree            (BASELINE.md section 4)
  * non-local net at raw random init: the reference's unscaled softmax sees logits of 1e4..1e8, i.e. an arg-max
    whose top-2 gaps fall below fp16 resolution for some rows; one flipped row is then amplified by every later
    non-local block, so whole-network max-norm parity past layer2 is chaotic (DESIGN.md "non-local numerics").
    That fixture is therefore checked end-to-end up to layer2 and block-by-block (teacher-forced: each block gets
    OUR input, the oracle recomputes it in fp32) for the rest; the "tamed" fixture (theta/phi scaled into a
    trained-like regime, same transform on the reference) is checked end-to-end at the normal tolerances.
"""
import glob
import os

import numpy as np
import pytest
import torch

from oracle import functional as OF
import pretorched_x_b200 as P

pytestmark = pytest.mark.gpu

GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "*.pt")))
MODEL_FIX = [g for g in GOLDEN if torch.load(g, weights_only=False)["kind"] == "model"]


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need an H100"
    return torch.device("cuda:0")


def build(fx, dev):
    return OF.build_package_model(P, fx).to(dev)


def stage_errors(m, x, fx):
    from pretorched_x_b200 import engine, ops
    errs = {}
    with torch.no_grad():
        a = engine.run_stem(m, x)
        outs = {"maxpool": a}
        for ln in ("layer1", "layer2", "layer3", "layer4"):
            for blk in getattr(m, ln):
                a = engine.run_block(blk, a)
            outs[ln] = a
        logits = m.logits(a)
    for name, ref in fx["stages"].items():
        if name == "logits":
            continue
        t = ops.to_ncdhw(outs[name]).reshape(-1)[::ref["step"]][:ref["sample"].numel()].cpu().double()
        d = (t - ref["sample"].double()).abs() / max(ref["absmax"], 1e-12)
        errs[name] = (d.max().item(), d.median().item())
    d = (logits.cpu().double() - fx["logits"].double()).abs() / fx["logits"].abs().max().item()
    errs["logits"] = (d.max().item(), d.median().item())
    return errs, logits


@pytest.mark.parametrize("path", MODEL_FIX, ids=[os.path.basename(p)[:-3] for p in MODEL_FIX])
def test_forward_matches_reference_golden(dev, path):
    fx = torch.load(path, weights_only=False)
    m = build(fx, dev)
    assert OF.digests_match(OF.state_digest({k: v.cpu() for k, v in m.state_dict().items()}), fx["weight_digest"])
    x = OF.seeded_input(fx["input_shape"], fx["seeds"]["input"]).to(dev)
    errs, logits = stage_errors(m, x, fx)
    chaotic = "nonlocal" in fx["arch"] and not fx.get("nl_factors")
    for name, (emax, emed) in errs.items():
        if chaotic and name in ("layer3", "layer4", "logits"):
            continue      # arg-max regime: see module docstring; covered block-by-block by the teacher-forced test below
        assert emax <= (5e-3 if name == "logits" else 1e-2), (name, emax, emed)
    if not chaotic:
        assert torch.equal(logits.argmax(1).cpu(), fx["logits"].argmax(1))
    # public API path gives the same numbers as the staged walk
    with torch.no_grad():
        assert torch.equal(m(x), logits)


def test_nonlocal_net_block_by_block_teacher_forced(dev):
    """Every residual / non-local block of the raw random-init non-local net against the CPU oracle on the SAME
    (our) block input: isolates each block's arithmetic from upstream drift."""
    from pretorched_x_b200 import engine, ops
    fx = torch.load([p for p in MODEL_FIX if p.endswith("nonlocalresnet3d50_b1_t16_96.pt")][0], weights_only=False)
    m = build(fx, torch.device("cpu"))
    sd = {k: v.clone() for k, v in m.state_dict().items()}
    m = m.to(dev)
    x = OF.seeded_input(fx["input_shape"], fx["seeds"]["input"]).to(dev)
    nlpos = OF.nonlocal_positions([3, 4, 6, 3], [0, 2, 3, 0])
    with torch.no_grad():
        a = engine.run_stem(m, x)
        inplanes = 64
        for li, ln in enumerate(("layer1", "layer2", "layer3", "layer4")):
            planes = (64, 128, 256, 512)[li]
            for bi, blk in enumerate(getattr(m, ln)):
                stride = 2 if (li > 0 and bi == 0) else 1
                has_ds = bi == 0 and (stride != 1 or inplanes != planes * 4)
                pfx = "%s.%d" % (ln, bi)
                want = OF.bottleneck(ops.to_ncdhw(a).cpu(), sd, pfx, "resnet3d", "A", planes, stride, has_ds)
                a = engine.run_bottleneck(blk, a)
                got = ops.to_ncdhw(a).cpu()
                assert (got - want).abs().max().item() <= 3e-3 * want.abs().max().item(), pfx
                if bi in nlpos[li]:
                    want = OF.nonlocal_block(got, sd, pfx + ".nonlocalblock")
                    a = engine.run_nonlocal(blk.nonlocalblock, a)
                    d = (ops.to_ncdhw(a).cpu() - want).abs() / want.abs().max().item()
                    per_position = d.amax(dim=1).reshape(-1)
                    # near-tied arg-max rows may legitimately flip under fp16 theta/phi; they must stay rare
                    assert float((per_position > 1e-2).double().mean()) <= 0.02, pfx
                    assert d.median().item() <= 1e-3, pfx
                inplanes = planes * 4


def test_features_logits_api_and_identity_head(dev):
    fx = torch.load([p for p in MODEL_FIX if "resnet3d50" in p and "nonlocal" not in p][0], weights_only=False)
    m = build(fx, dev)
    x = OF.seeded_input(fx["input_shape"], fx["seeds"]["input"]).to(dev)
    with torch.no_grad():
        feat = m.features(x)
        assert feat.dtype == torch.float32 and tuple(feat.shape) == fx["stages"]["layer4"]["shape"]
        lg = m.logits(feat)
        assert (lg - m(x)).abs().max().item() <= 2e-3 * lg.abs().max().item()
        m.last_linear = P.Identity()
        pooled = m(x)
        assert tuple(pooled.shape) == (x.shape[0], 2048)
        want = feat.mean(dim=(2, 3, 4))
        assert (pooled - want).abs().max().item() <= 2e-3 * want.abs().max().item()


def test_nonlocal_block_teacher_forced(dev):
    """One non-local block in a benign logit regime (scaled-down theta/phi, as after training) against the oracle."""
    from pretorched_x_b200.models.nonlocalnet import NonLocalBlock3D
    torch.manual_seed(0)
    blk = NonLocalBlock3D(256)
    with torch.no_grad():
        blk.theta.weight.mul_(0.05); blk.phi.weight.mul_(0.05)
        blk.W[1].weight.fill_(1.0)
    OF.randomize_bn_(blk, 3)
    blk.eval()
    x = OF.seeded_input((2, 256, 2, 7, 7), 4).half().float()
    with torch.no_grad():
        want = OF.nonlocal_block(x, {"nl." + k: v for k, v in blk.state_dict().items()}, "nl")
    with torch.no_grad():
        got = blk.to(dev)(x.to(dev))
    assert (got.cpu() - want).abs().max().item() <= 5e-3 * want.abs().max().item()


def test_trn_relations_match_golden(dev):
    gd = os.path.join(os.path.dirname(__file__), "golden")
    for name in ("relation_small", "relation_htrn"):
        fx = torch.load(os.path.join(gd, name + ".pt"), weights_only=False)
        torch.manual_seed(fx["seeds"]["init"])
        r = P.Relation(fx["T"], fx["F"], fx["out"], bottleneck_dim=fx["bottleneck"]).to(dev).eval()
        x = OF.seeded_input((fx["B"], fx["T"], fx["F"]), fx["seeds"]["input"]).to(dev)
        with torch.no_grad():
            y = r(x)
        assert tuple(y.shape) == tuple(fx["output"].shape)
        assert (y.cpu() - fx["output"]).abs().max().item() <= 5e-3 * fx["output"].abs().max().item()
    fx = torch.load(os.path.join(gd, "msrelation_small.pt"), weights_only=False)
    torch.manual_seed(fx["seeds"]["init"])
    r = P.MultiScaleRelation(fx["T"], fx["F"], fx["out"], bottleneck_dim=fx["bottleneck"]).to(dev).eval()
    x = OF.seeded_input((fx["B"], fx["T"], fx["F"]), fx["seeds"]["input"]).to(dev)
    np.random.seed(fx["np_seed"])
    with torch.no_grad():
        y = r(x)
    assert (y.cpu() - fx["output"]).abs().max().item() <= 5e-3 * fx["output"].abs().max().item()


def test_full_size_clips_are_independent_and_graph_replay_is_exact(dev):
    """BASELINE clip size (16x224x224): a clip's logits do not depend on its batch-mates (eval BN, no cross-sample
    coupling), and the CUDA-graph replay reproduces the eager forward bit for bit."""
    from pretorched_x_b200.graph import GraphedForward
    torch.manual_seed(0)
    m = OF.randomize_bn_(P.resnet3d50(num_classes=400, pretrained=None), 1).eval().to(dev)
    x = OF.seeded_input((3, 3, 16, 224, 224), 9).to(dev)
    with torch.no_grad():
        full = m(x)
        solo = torch.cat([m(x[i:i + 1]) for i in range(3)])
    assert torch.isfinite(full).all()
    assert (full - solo).abs().max().item() <= 1e-3 * full.abs().max().item()
    g = GraphedForward(m, x)
    assert torch.equal(g(x), full)
    assert torch.equal(g(), full)


DFS_CASES = [("resnet3d50_b2_t8_64", 5, ["4:2", "5:1,3:2", "1:3", "17:2"]),
             ("r2plus1d34_b1_t8_64", 4, ["4:1", "2:3,3:2"]),
             ("resnet18_b2_64", 6, ["3:4", "1:2,4:3"]),
             ("nonlocalresnet3d50_tamed_b1_t16_96", 3, ["4:1", "8:2", "5:1,4:2"]),
             ("preact_resnet3d50_b2_t8_64", 4, ["3:1,2:2"])]


@pytest.mark.parametrize("name,batch,specs", DFS_CASES, ids=[c[0] for c in DFS_CASES])
def test_depth_first_trunk_schedule_matches_breadth_first(dev, name, batch, specs):
    """engine.run_trunk walked depth-first in clip chunks (the L2-resident schedule of the BASELINE batch sizes, forced here on
    small shapes, ragged last chunk included) gives the breadth-first result: the same kernels compute every output element, so the
    features are equal bit for bit unless a chunk's size moves a layer across a kernel-dispatch boundary (dense-M split-K vs slab),
    where the fp32 accumulation order differs and an output may land on the neighbouring fp16 value (one ulp = 1e-3 of the range
    at the top binade) -- bounded at 3e-3 of the tensor's range, inside the parity tolerance."""
    from pretorched_x_b200 import engine
    from pretorched_x_b200.graph import GraphedForward
    fx = torch.load([p for p in MODEL_FIX if os.path.basename(p) == name + ".pt"][0], weights_only=False)
    m = build(fx, dev)
    shape = (batch,) + tuple(fx["input_shape"][1:])
    x = OF.seeded_input(shape, 77).to(dev)
    try:
        engine.set_dfs("off")
        with torch.no_grad():
            want_f = m.features_act(x)
            want = m.logits(want_f)
        for spec in specs:
            engine.set_dfs(spec)
            with torch.no_grad():
                got_f = m.features_act(x)
                got = m.logits(got_f)
            assert (got_f.N, got_f.T, got_f.H, got_f.W, got_f.C) == (want_f.N, want_f.T, want_f.H, want_f.W, want_f.C), spec
            scale = want_f.data.float().abs().max().item()
            assert (got_f.data.float() - want_f.data.float()).abs().max().item() <= 3e-3 * scale, spec
            assert (got - want).abs().max().item() <= 2e-3 * want.abs().max().item(), spec
            assert torch.equal(got_f.data[:, got_f.C:], torch.zeros_like(got_f.data[:, got_f.C:])), spec   # pad columns stay zero
        # capture-safe: the chunked walk replays from a CUDA graph
        engine.set_dfs(specs[0])
        g = GraphedForward(m, x)
        with torch.no_grad():
            eager = m(x)
        assert torch.equal(g(x), eager)
    finally:
        engine.set_dfs("off")


def test_depth_first_schedule_at_baseline_clip_size(dev):
    """A chunked forward of 5 full-size clips (16x224x224: W chunking, 112/56-wide TMA boxes, the pooled stem) equals the
    breadth-first one; the default schedule is breadth-first (the measured optimum, engine.set_dfs)."""
    from pretorched_x_b200 import engine
    torch.manual_seed(0)
    m = OF.randomize_bn_(P.resnet3d50(num_classes=400, pretrained=None), 1).eval().to(dev)
    assert engine.dfs_plan() == []
    x = OF.seeded_input((5, 3, 16, 224, 224), 11).to(dev)
    try:
        engine.set_dfs("off")
        with torch.no_grad():
            want = m(x)
        engine.set_dfs("5:2,4:4")
        with torch.no_grad():
            got = m(x)
    finally:
        engine.set_dfs("off")
    assert (got - want).abs().max().item() <= 2e-3 * want.abs().max().item()


def test_model_on_a_second_device_with_device_0_current():
    """ADVICE r1: `model.to('cuda:1')` in a process whose current device is 0 -- every operator switches to its tensors' device for
    the launch (ops._on_device), kernel attributes / SM counts are cached per device ordinal.  Needs two GPUs (skipped otherwise)."""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    fx = torch.load([p for p in MODEL_FIX if os.path.basename(p) == "resnet3d50_b2_t8_64.pt"][0], weights_only=False)
    x = OF.seeded_input(fx["input_shape"], fx["seeds"]["input"])
    torch.cuda.set_device(0)
    m0 = build(fx, torch.device("cuda:0"))
    m1 = build(fx, torch.device("cuda:1"))
    with torch.no_grad():
        y0 = m0(x.to("cuda:0"))
        y1 = m1(x.to("cuda:1"))            # current device is still 0
    assert torch.cuda.current_device() == 0 and y1.device.index == 1
    assert torch.equal(y0.cpu(), y1.cpu())


SF_FIX = [g for g in GOLDEN if torch.load(g, weights_only=False)["kind"] == "slowfast"]


@pytest.mark.parametrize("path", SF_FIX, ids=[os.path.basename(p)[:-3] for p in SF_FIX])
def test_slowfast_matches_reference_golden(dev, path):
    """SlowFast / SlowOnly / FastOnly (slowfast.py) end to end against the reference's own logits."""
    fx = torch.load(path, weights_only=False)
    torch.manual_seed(fx["seeds"]["init"])
    m = getattr(P.slowfast, fx["factory"])(mode=fx["mode"], **fx["kwargs"])
    OF.randomize_bn_(m, fx["seeds"]["bn"])
    m = m.eval().to(dev)
    x = OF.seeded_input(fx["input_shape"], fx["seeds"]["input"]).to(dev)
    with torch.no_grad():
        y = m(x)
    assert tuple(y.shape) == tuple(fx["logits"].shape)
    err = (y.cpu().double() - fx["logits"].double()).abs().max().item() / fx["logits"].abs().max().item()
    assert err <= 5e-3, err
    assert torch.equal(y.argmax(1).cpu(), fx["logits"].argmax(1))


NL_FIX = [g for g in GOLDEN if torch.load(g, weights_only=False)["kind"] == "nlblock"]


@pytest.mark.parametrize("path", NL_FIX, ids=[os.path.basename(p)[:-3] for p in NL_FIX])
def test_nonlocal_block_modes_match_reference_golden(dev, path):
    """NonLocalBlock{1,2,3}D in gaussian / dot_product / embedded_gaussian mode, with and without sub-sampling and
    the output BatchNorm (nonlocalnet.py:143-211), against outputs of the reference's own modules."""
    from tests.test_oracle_golden import build_nlblock
    fx = torch.load(path, weights_only=False)
    blk = build_nlblock(fx).to(dev)
    x = (OF.seeded_input(fx["input_shape"], fx["seeds"]["input"]) * fx["input_scale"]).to(dev)
    with torch.no_grad():
        y = blk(x)
    assert tuple(y.shape) == tuple(fx["output"].shape)
    err = (y.cpu().double() - fx["output"].double()).abs().max().item() / fx["output"].abs().max().item()
    assert err <= 5e-3, err


TRN_FIX = [g for g in GOLDEN if torch.load(g, weights_only=False)["kind"] == "trn"]


@pytest.mark.parametrize("path", TRN_FIX, ids=[os.path.basename(p)[:-3] for p in TRN_FIX])
def test_trn_wrapper_matches_reference_golden(dev, path):
    """Full TRN (frames -> 2-D backbone -> relation -> Linear, trn.py:246-263) against the reference's own outputs."""
    from tests.test_oracle_golden import build_trn
    fx = torch.load(path, weights_only=False)
    m = build_trn(fx).to(dev)
    x = OF.seeded_input(fx["input_shape"], fx["seeds"]["input"]).to(dev)
    if fx["np_seed"] is not None:
        np.random.seed(fx["np_seed"])
    with torch.no_grad():
        feats = m.features(x)
        y = m.logits(feats)
    assert tuple(y.shape) == tuple(fx["logits"].shape)
    ef = (feats.cpu().double() - fx["features"].double()).abs().max().item() / fx["features"].abs().max().item()
    el = (y.cpu().double() - fx["logits"].double()).abs().max().item() / fx["logits"].abs().max().item()
    assert ef <= 1e-2 and el <= 1e-2, (ef, el)


def test_multiscale_relation_is_graph_capturable(dev):
    """The tuple table lives in one persistent device buffer: a CUDA graph over forward_tuples replays with NEW tuples after
    a single host->device copy (no per-tuple copies, no host work inside the graph)."""
    from pretorched_x_b200 import ops
    torch.manual_seed(0)
    r = P.MultiScaleRelation(8, 256, 64, bottleneck_dim=128).to(dev).eval()
    x = OF.seeded_input((4, 8, 256), 5).to(dev)
    with torch.no_grad():
        x16 = ops.cast_rows(x.view(4, -1), relu=True).view(4, 8, -1)
        np.random.seed(7)
        picks_a = r.sample_tuples()
        picks_b = r.sample_tuples()
        table = r.upload_tuples(picks_a, dev)
        total = torch.empty((4, 64), dtype=torch.float32, device=dev)
        r.forward_tuples(x16, table, total)                      # warm-up (packs weights)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            r.forward_tuples(x16, table, total)
        g.replay()
        torch.cuda.synchronize()
        got_a = total.clone()
        r.upload_tuples(picks_b, dev)
        g.replay()
        torch.cuda.synchronize()
        got_b = total.clone()
        sd = {k: v.cpu() for k, v in r.state_dict().items()}
        want_a = OF.multiscale_relation(x.cpu(), sd, 8, 256, tuples=picks_a).view(4, 64)
        want_b = OF.multiscale_relation(x.cpu(), sd, 8, 256, tuples=picks_b).view(4, 64)
    assert (got_a.cpu() - want_a).abs().max().item() <= 5e-3 * want_a.abs().max().item()
    assert (got_b.cpu() - want_b).abs().max().item() <= 5e-3 * want_b.abs().max().item()
    assert not torch.equal(got_a, got_b)


def test_trainable_head_on_frozen_engine_features(dev):
    """torch.autograd.Function boundary: the trunk is a frozen feature extractor (non-differentiable outputs), the dense head has
    a real backward on the wgmma GEMM.  Gradients of last_linear match torch's fp32 autograd on the same pooled features."""
    torch.manual_seed(0)
    m = OF.randomize_bn_(P.resnet3d18(num_classes=7, pretrained=None), 1).eval().to(dev)
    x = OF.seeded_input((3, 3, 8, 64, 64), 4).to(dev).requires_grad_(True)
    target = torch.tensor([1, 5, 2], device=dev)
    logits = m(x)                                                   # grad mode on, head parameters require grad
    assert logits.requires_grad
    loss = torch.nn.functional.cross_entropy(logits, target)
    loss.backward()
    assert x.grad is None                                           # frozen trunk: nothing flows to the input
    assert all(p.grad is None for n, p in m.named_parameters() if not n.startswith("last_linear"))
    gw, gb = m.last_linear.weight.grad.clone(), m.last_linear.bias.grad.clone()
    with torch.no_grad():
        from pretorched_x_b200 import ops
        pooled = ops.avgpool_global(m.features_act(x))[:, :512].float()
    w = m.last_linear.weight.detach().clone().requires_grad_(True)
    b = m.last_linear.bias.detach().clone().requires_grad_(True)
    ref_loss = torch.nn.functional.cross_entropy(pooled @ w.t() + b, target)
    ref_loss.backward()
    assert abs(loss.item() - ref_loss.item()) <= 2e-3 * max(1.0, abs(ref_loss.item()))
    assert (gw - w.grad).abs().max().item() <= 5e-3 * w.grad.abs().max().item()
    assert (gb - b.grad).abs().max().item() <= 5e-3 * b.grad.abs().max().item()
    # an optimiser step changes the head's output (the packed copy follows the parameter's version counter)
    opt = torch.optim.SGD(m.last_linear.parameters(), lr=0.5)
    opt.step()
    with torch.no_grad():
        assert not torch.equal(m(x), logits.detach())


def test_relation_mlp_backward_matches_torch(dev):
    torch.manual_seed(0)
    r = P.Relation(4, 64, 16, bottleneck_dim=32).to(dev)
    x = OF.seeded_input((5, 4, 64), 3).to(dev).requires_grad_(True)
    y = r(x)
    y.square().mean().backward()
    got = {n: p.grad.clone() for n, p in r.named_parameters()}
    gx = x.grad.clone()
    ref = torch.nn.Sequential(torch.nn.ReLU(), torch.nn.Linear(256, 32), torch.nn.ReLU(), torch.nn.Linear(32, 16)).to(dev)
    ref.load_state_dict({k.replace("relate.", ""): v for k, v in r.state_dict().items()})
    x2 = x.detach().clone().requires_grad_(True)
    ref(x2.view(5, -1)).square().mean().backward()
    for n, p in ref.named_parameters():
        assert (got["relate." + n] - p.grad).abs().max().item() <= 1e-2 * p.grad.abs().max().item() + 1e-6, n
    assert (gx - x2.grad).abs().max().item() <= 1e-2 * x2.grad.abs().max().item() + 1e-6
