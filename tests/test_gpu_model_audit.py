"""GPU (-m gpu): every library launch of each benchmarked forward, at the per-GPU batch bench.py times, held element by element to
the fp64 bound of tests/kernel_ref.py (tests/model_audit.py), and the audited eager output equal bit for bit to the CUDA-graph
replay bench.py times.

The hand-picked shapes of the kernel-matrix files run at small batch; the dispatch rules pick kernels and tile plans from batch
and item counts, so at the benchmarked shapes other plans run.  Models and inputs are built as bench.py's run_ours / run_biggan
build them (imported from bench.py, so the audit follows the benchmark configurations), with the default schedules.  A per-launch
table is printed (pytest -s)."""
import functools
import os
import time

import pytest
import torch

import bench
from tests.conftest import has_h100
from tests import kernel_ref as KR
from tests.kernel_ref import att_bound, att_ref, conv_ref, gemm_acc
from tests.model_audit import audit
from tests.test_gpu_kernel_matrix import KNOB_ENV as MATRIX_KNOBS

# the kernel-choice knobs of the matrix files, and every other variable that changes what a forward launches: the depth-first
# trunk / generator schedules and the stem, slab and launch options the library reads.  The audit is of the default choices.
KNOB_ENV = MATRIX_KNOBS + ("B2_DFS", "B2_GAN_DFS", "B2_STEM_POOLW", "B2_STEM_PAIR", "B2_STEM_ROWS", "B2_SLAB_MP", "B2_SLAB_MT",
                           "B2_PDL")

pytestmark = [
    pytest.mark.gpu,
    pytest.mark.skipif(not has_h100(), reason="needs an H100"),
    pytest.mark.skipif(any(os.environ.get(e) for e in KNOB_ENV),
                       reason="a dispatch override is set in the environment (%s)" % ", ".join(KNOB_ENV)),
]

# (workload, per-GPU batch): r2plus1d34's 16 clips shard over 1 / 2 / 4 / 8 GPUs (strong scaling), so each GPU runs 16 .. 2
CASES = [("resnet3d50", 32), ("r2plus1d34", 16), ("r2plus1d34", 8), ("r2plus1d34", 4), ("r2plus1d34", 2), ("nonlocal50", 8),
         ("resnet18", 256), ("trn", 32)]


def _report(name, rep, seconds):
    """The per-launch table, the worst ratio per (entry, kernel), every distinct (kernel, plan) pair with its launch count and worst
    ratio, and one summary line with the wall time of the audit and the fp64 rate of its reference products."""
    print(rep.table(name))
    by_kernel, by_plan = {}, {}
    for r in rep.rows:
        if r["ratio"] is not None:
            key = (r["entry"], r["kernel"])
            by_kernel[key] = max(by_kernel.get(key, 0.0), r["ratio"])
            if r["kernel"] != "-":
                n, w = by_plan.get((r["kernel"], r["info"]), (0, 0.0))
                by_plan[(r["kernel"], r["info"])] = (n + 1, max(w, r["ratio"]))
    for (entry, kernel), worst in sorted(by_kernel.items()):
        print("[model-audit] %s worst %-15s %-12s %.4f" % (name, entry, kernel, worst))
    for (kernel, info), (n, worst) in sorted(by_plan.items()):
        print("[model-audit] %s plan %-12s %-24s launches %3d worst %.4f" % (name, kernel, info, n, worst))
    print("[model-audit] %s launches %d (wrapped entries %d), audited %d, worst err/bound %.4f, %.1f s, fp64 references %.2f TFLOP "
          "(%.2f TFLOP/s)" % (name, rep.launches, rep.counted, sum(r["ratio"] is not None for r in rep.rows), rep.worst, seconds,
                              rep.ref_flops / 1e12, rep.ref_flops / 1e12 / max(seconds, 1e-9)))


def _assert_clean(name, rep):
    bad = rep.failures()
    assert not bad, "%s: %d launches over their bound, first: #%d %s %s %s %s: %s" % (
        name, len(bad), bad[0]["index"], bad[0]["entry"], bad[0]["geometry"], bad[0]["kernel"], bad[0]["info"], bad[0]["where"])


@pytest.mark.timeout(1800, method="thread")
@pytest.mark.parametrize("workload,B", CASES, ids=["%s_B%d" % c for c in CASES])
def test_benchmarked_forward_every_launch_against_fp64(workload, B):
    from pretorched_x_b200.graph import GraphedForward
    spec = bench.WORKLOADS[workload]
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    model = bench.build_ours(spec).to(dev)
    g = torch.Generator().manual_seed(1000)                      # rank 0's input, as run_ours draws it
    x = torch.randn((B,) + spec["sample"], generator=g).to(dev)
    t0 = time.time()
    rep = audit(lambda: model(x))
    seconds = time.time() - t0
    _report("%s_B%d" % (workload, B), rep, seconds)
    _assert_clean(workload, rep)
    want = rep.output.clone()
    rep = None
    graphed = GraphedForward(model, x, warmup=2)
    got = graphed()
    torch.cuda.synchronize()
    assert torch.equal(got.view(-1).view(torch.int32 if got.dtype == torch.float32 else torch.int16),
                       want.view(-1).view(torch.int32 if want.dtype == torch.float32 else torch.int16)), \
        "the CUDA-graph replay differs from the audited eager forward"


@pytest.mark.timeout(1800, method="thread")
def test_biggan_forward_every_launch_against_fp64():
    import pretorched_x_b200 as P
    from pretorched_x_b200.graph import GraphedForward
    from oracle import biggan as OB
    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    model, _, _, _ = OB.build_case(P.biggan_deep, bench.BIGGAN_RES, bench.BIGGAN_CH, bench.BIGGAN_CLASSES, 4, init="ortho")
    model = model.to(dev)
    z, lab = OB.seeded_inputs(bench.BIGGAN_BATCH, bench.BIGGAN_CLASSES, 1000)
    z, lab = z.to(dev), lab.to(dev)
    t0 = time.time()
    rep = audit(lambda: model(z, lab, out_dtype=torch.float16))
    seconds = time.time() - t0
    _report("biggan256_B%d" % bench.BIGGAN_BATCH, rep, seconds)
    _assert_clean("biggan256", rep)
    want = rep.output.clone()
    rep = None
    graphed = GraphedForward(model, (z, lab), warmup=1, out_dtype=torch.float16)
    got = graphed()
    torch.cuda.synchronize()
    assert torch.equal(got.view(torch.int16), want.view(torch.int16)), "the CUDA-graph replay differs from the audited eager forward"


@pytest.mark.timeout(900, method="thread")
def test_audit_catches_a_fault_in_one_launch_of_a_benchmarked_forward():
    """The audit's references are live at the benchmark's shapes: one output element of the last image in resnet18's tenth
    convolution, at B = 256, moved by 1/8 makes that launch, and only that launch, fail its bound."""
    from pretorched_x_b200 import ops
    spec = bench.WORKLOADS["resnet18"]
    dev = torch.device("cuda:0")
    model = bench.build_ours(spec).to(dev)
    x = torch.randn((256,) + spec["sample"], generator=torch.Generator().manual_seed(1000)).to(dev)
    real, calls = ops.conv, []

    @functools.wraps(real)
    def faulty(*args, **kwargs):
        y = real(*args, **kwargs)
        calls.append(1)
        if len(calls) == 10:
            t = y.data[-3, 5]
            y.data[-3, 5] = t + 0.125 * torch.sign(t) + 0.125 * (t == 0)
        return y
    ops.conv = faulty
    try:
        rep = audit(lambda: model(x))
    finally:
        ops.conv = real
    bad = rep.failures()
    print("[model-audit] injected fault: %s" % ["#%d %s %s: %s" % (r["index"], r["entry"], r["geometry"], r["where"]) for r in bad])
    conv_rows = [r for r in rep.rows if r["entry"] == "conv"]
    assert [r["index"] for r in bad] == [conv_rows[9]["index"]]
    assert "col 5" in bad[0]["where"]


def test_gpu_fp64_references_equal_cpu_ones():
    """The device switch of the kernel_ref builders: the same references on the GPU and the CPU, to 1e-12 relative."""
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(7)

    def close(a, b):
        a, b = a.cpu(), b.cpu()
        return float((a - b).abs().max() / b.abs().max().clamp_min(1e-300)) <= 1e-12

    for N, T, H, W, C, K, k, s, p in [(2, 4, 9, 11, 16, 24, (3, 3, 3), (1, 2, 2), (1, 1, 1)), (1, 1, 14, 14, 8, 64, (1, 7, 7), (1, 2, 2),
                                                                                                (0, 3, 3)),
                                      (3, 5, 6, 6, 32, 40, (3, 1, 1), (1, 1, 1), (1, 0, 0))]:
        x = torch.randn(N, T, H, W, C, generator=g).half()
        w = torch.randn(K, k[0] * k[1] * k[2], C, generator=g).half()
        sc, sh = torch.rand(K, generator=g) + 0.5, torch.randn(K, generator=g)
        r = torch.randn(N * ((T + 2 * p[0] - k[0]) // s[0] + 1) * ((H + 2 * p[1] - k[1]) // s[1] + 1)
                        * ((W + 2 * p[2] - k[2]) // s[2] + 1), K, generator=g).half()
        cpu = conv_ref(x, w, sc, sh, k, s, p, residual=r, relu=True)
        gpu = conv_ref(x.to(dev), w.to(dev), sc.to(dev), sh.to(dev), k, s, p, residual=r.to(dev), relu=True, device=dev)
        assert close(gpu[0], cpu[0]) and close(gpu[1], cpu[1])
    for M, N, Kd in [(300, 72, 520), (1, 400, 2048), (129, 8, 64)]:
        a, b = torch.randn(M, Kd, generator=g).half(), torch.randn(N, Kd, generator=g).half()
        cpu, gpu = gemm_acc(a, b), gemm_acc(a.to(dev), b.to(dev), device=dev)
        assert close(gpu[0], cpu[0]) and close(gpu[1], cpu[1])
    # the generator epilogues and the depthwise reference
    N, H, W, C, K = 2, 5, 6, 16, 24
    xl = torch.randn(N, H, W, C, generator=g).half()
    wph = torch.randn(K, 16, C, generator=g).half()
    cpu, gpu = KR.upconv_acc(xl, wph), KR.upconv_acc(xl.to(dev), wph.to(dev), device=dev)
    assert close(gpu[0], cpu[0]) and close(gpu[1], cpu[1])
    rows = H * W
    isc, ish = torch.rand(N, C + 8, generator=g) + 0.5, torch.randn(N, C + 8, generator=g)
    wk = torch.randn(K, C, generator=g).half()
    xr = xl.reshape(-1, C)
    cpu = KR.in_affine_acc(xr, wk, isc, ish, rows)
    gpu = KR.in_affine_acc(xr.to(dev), wk.to(dev), isc.to(dev), ish.to(dev), rows, device=dev)
    assert close(gpu[0], cpu[0]) and close(gpu[1], cpu[1])
    skip = torch.randn(N * rows, K + 8, generator=g).half()
    cpu, gpu = KR.nearest_up2(skip, N, 2 * H, 2 * W, K), KR.nearest_up2(skip.to(dev), N, 2 * H, 2 * W, K, device=dev)
    assert close(gpu, cpu)
    acc, mag = KR.gemm_acc(xr, wk)
    ssc, ssh = torch.rand(N, K + 8, generator=g) + 0.5, torch.randn(N, K + 8, generator=g)
    res = torch.randn(N * rows, K, generator=g).half()
    cpu = KR.epilogue(acc, mag, KR.per_row(ssc, rows, N * rows, K), KR.per_row(ssh, rows, N * rows, K), res, pre=True)
    gpu = KR.epilogue(acc.to(dev), mag.to(dev), KR.per_row(ssc.to(dev), rows, N * rows, K, device=dev),
                      KR.per_row(ssh.to(dev), rows, N * rows, K, device=dev), res.to(dev), pre=True, device=dev)
    assert close(gpu[0], cpu[0]) and close(gpu[1], cpu[1])
    s2, t2 = KR.per_row(ssc, rows, N * rows, K), KR.per_row(ssh, rows, N * rows, K)
    cpu2 = KR.second_output(cpu[0], cpu[1], s2, t2)
    gpu2 = KR.second_output(gpu[0], gpu[1], s2.to(dev), t2.to(dev), device=dev)
    assert close(gpu2[0], cpu2[0]) and close(gpu2[1], cpu2[1])
    w9, dsc, dsh = torch.randn(9, C, generator=g), torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g)
    for stride, clamp_in in ((1, False), (2, True)):
        cpu = KR.dw_ref(xl, w9, dsc, dsh, stride, clamp_in, True)
        gpu = KR.dw_ref(xl.to(dev), w9.to(dev), dsc.to(dev), dsh.to(dev), stride, clamp_in, True, device=dev)
        assert close(gpu[0], cpu[0]) and close(gpu[1], cpu[1])
    for mode in (0, 1, 2):
        B, Nq, Nk, d, dv = 2, 130, 70, 64, 128
        q, k_, v = (torch.randn(B * n, c, generator=g).half() for n, c in ((Nq, d), (Nk, d), (Nk, dv)))
        cpu = att_ref(q, k_, v, B, Nq, Nk, mode)
        gpu = att_ref(q.to(dev), k_.to(dev), v.to(dev), B, Nq, Nk, mode)
        assert close(gpu[0], cpu[0]) and close(gpu[1], cpu[1])
        assert close(att_bound(gpu[0], gpu[1], v.to(dev), B, Nq, Nk, mode), att_bound(cpu[0], cpu[1], v, B, Nq, Nk, mode))
