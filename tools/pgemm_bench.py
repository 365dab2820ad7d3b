"""GPU time of the persistent GEMM (pgemm_kernel) at the 1x1x1 convolutions of resnet3d50 (B = 32 clips of 16 x 224^2, shortcut B:
conv1 / conv3 of every bottleneck, conv3 with the type-B projection fused as a second operand pair), each issued the way the engine
issues it (fp16 NDHWC rows, folded BN, residual + ReLU where the block closes) and timed as CUDA-graph replays between CUDA events
after a warm-up.

Per shape: us per call, algorithmic TFLOP/s and GB/s (each operand and output byte once), and the ratio of the least time the
card could take -- max(FLOP / 989 TFLOP/s, bytes / 3.35 TB/s), the H100 SXM data-sheet dense fp16 and HBM3 figures -- to the
measured time, naming the side that bounds it.  The card's name, power limit and the SM clock sampled after each shape are printed.
usage: pgemm_bench.py [shape ...]   (default: all shapes below)"""
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pretorched_x_b200 import ops  # noqa: E402

PEAK_TFLOPS, PEAK_TBS = 989.0, 3.35
# layer1 runs at 8 x 56^2, layer2 at 4 x 28^2, layer3 at 2 x 14^2, layer4 at 1 x 7^2 (x 32 clips); a stage's first conv1 runs at the
# previous stage's resolution (the stride sits in conv2)
M1, M2, M3, M4 = 32 * 8 * 56 * 56, 32 * 4 * 28 * 28, 32 * 2 * 14 * 14, 32 * 1 * 7 * 7
# name: M, N (output channels), K, K2 of the fused projection (0: none), residual, launches per forward
SHAPES = {
    "l1.0-conv1-64-64": (M1, 64, 64, 0, False, 1),
    "l1-conv1-256-64": (M1, 64, 256, 0, False, 2),
    "l1.0-conv3+proj-64-256": (M1, 256, 64, 64, False, 1),
    "l1-conv3-64-256+res": (M1, 256, 64, 0, True, 2),
    "l2.0-conv1-256-128": (M1, 128, 256, 0, False, 1),
    "l2.0-conv3+proj-128-512": (M2, 512, 128, 256, False, 1),
    "l2-conv1-512-128": (M2, 128, 512, 0, False, 3),
    "l2-conv3-128-512+res": (M2, 512, 128, 0, True, 3),
    "l3.0-conv1-512-256": (M2, 256, 512, 0, False, 1),
    "l3.0-conv3+proj-256-1024": (M3, 1024, 256, 512, False, 1),
    "l3-conv1-1024-256": (M3, 256, 1024, 0, False, 5),
    "l3-conv3-256-1024+res": (M3, 1024, 256, 0, True, 5),
    "l4.0-conv1-1024-512": (M3, 512, 1024, 0, False, 1),
    "l4.0-conv3+proj-512-2048": (M4, 2048, 512, 1024, False, 1),
    "l4-conv1-2048-512": (M4, 512, 2048, 0, False, 2),
    "l4-conv3-512-2048+res": (M4, 2048, 512, 0, True, 2),
}
REP = 20
ROUNDS = 10


def smi(query):
    try:
        return subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + query, "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        return "unknown"


def time_graph(fn):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(REP):
            fn()
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(ROUNDS):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    del g
    return e0.elapsed_time(e1) * 1e3 / (ROUNDS * REP)


def main(names):
    dev = torch.device("cuda:0")
    print("card: %s (power limit, max SM clock: %s)" % (torch.cuda.get_device_name(0), smi("power.limit,clocks.max.sm")), flush=True)
    print("%-26s %8s %5s %5s %5s %9s %8s %8s %7s %6s  %s" % ("shape", "M", "N", "K", "K2", "us", "TFLOP/s", "GB/s", "bound", "side",
                                                         "SM clock"), flush=True)
    tot_us = tot_bound = 0.0
    for name in names:
        M, N, K, K2, res, n = SHAPES[name]
        g = torch.Generator(device=dev).manual_seed(0)
        with torch.no_grad():
            A = torch.randn(M, K, device=dev, generator=g).half()
            B = (torch.randn(N, K, device=dev, generator=g) / K ** 0.5).half()
            sc, sh = torch.rand(N, device=dev, generator=g) + 0.5, torch.randn(N, device=dev, generator=g)
            R = torch.randn(M, N, device=dev, generator=g).half() if res else None
            second = None
            if K2:
                second = (torch.randn(M, K2, device=dev, generator=g).half(),
                          (torch.randn(N, K2, device=dev, generator=g) / K2 ** 0.5).half(), K2)
            out = torch.empty(M, N, device=dev, dtype=torch.float16)
            fn = lambda: ops.gemm(A, B, sc, sh, M, N, K, residual=R, relu=True, out=out, second=second)
            us = time_graph(fn)
        clock = smi("clocks.sm")
        flop = 2.0 * M * N * (K + K2)
        nbytes = 2.0 * (M * (K + K2) + N * (K + K2) + M * N * (2 if res else 1))
        t_flop, t_byte = flop / (PEAK_TFLOPS * 1e12) * 1e6, nbytes / (PEAK_TBS * 1e12) * 1e6
        bound = max(t_flop, t_byte)
        tot_us += n * us
        tot_bound += n * bound
        print("%-26s %8d %5d %5d %5d %9.1f %8.1f %8.0f %7.2f %6s  %s" % (name, M, N, K, K2, us, flop / us / 1e6, nbytes / us / 1e3,
                                                                     bound / us, "tensor" if t_flop > t_byte else "hbm", clock), flush=True)
        del A, B, R, second, out
    print("1x1 family of one forward (launch counts as listed): %.0f us measured, %.0f us bound (%.2f)" % (tot_us, tot_bound, tot_bound / tot_us),
          flush=True)


if __name__ == "__main__":
    main(sys.argv[1:] or list(SHAPES))
