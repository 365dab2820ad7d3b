"""GPU time of the stem convolution at the stem shapes of the benchmarked networks, issued the way engine.run_stem issues it:
the Toeplitz stem kernel with BN + ReLU (and, where the network's max-pool follows, the W direction of that pool) in its
epilogue, then the remaining (T, H) pool pass.  Each is timed as CUDA-graph replays between CUDA events after a warm-up.

Per shape: the instance the kernel ran with (G output rows per work item, "G=4t" for the transposed four-row one), conv ms and
stem ms (conv + pool pass), the conv's algorithmic TFLOP/s (3 input channels, every tap) and executed TFLOP/s (what the kernel
issues: K padded from 21 to 32 per (dt, dh), 128-row M tiles or 112-wide N tiles for the transposed instance, output channels
rounded up to the N tile, temporal taps outside the clip skipped), and the card's name and power limit.
usage: stem_bench.py [--rows 2|4|4t] [shape ...]   (default: all shapes below; --rows forces the two-row, the four-row or the
transposed four-row instance of the BN = 64 stems where it applies, as B2_STEM_ROWS does)"""
import ctypes
import os
import subprocess
import sys

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pretorched_x_b200 import _lib, engine, ops  # noqa: E402

# name: clips N, T, H, W, output channels, conv kernel, conv padding, max-pool (kernel, stride, padding) of the (T, H) pass or None
SHAPES = {
    "resnet3d50": (32, 16, 224, 224, 64, (7, 7, 7), (3, 3, 3), ((3, 3, 1), (2, 2, 1), (1, 1, 0))),
    "nonlocal50": (8, 32, 224, 224, 64, (7, 7, 7), (3, 3, 3), ((3, 3, 1), (2, 2, 1), (1, 1, 0))),
    "r2plus1d34": (16, 32, 112, 112, 110, (1, 7, 7), (0, 3, 3), None),       # spatial half of the (2+1)D stem, pair-of-planes mode
    "resnet18": (256, 1, 224, 224, 64, (1, 7, 7), (0, 3, 3), ((1, 3, 1), (1, 2, 1), (0, 1, 0))),
}
REP = 10
ROUNDS = 5


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        q = "power limit unknown"
    return "%s (%s)" % (name, q)


def executed_flops(N, T, Ho, Wo, K, kt, kh, pt, transposed):
    bn = 64 if K <= 64 else 128
    ncols = -(-((K + 7) // 8 * 8) // bn) * bn
    pair = kt == 1 and pt == 0 and Wo <= 60
    taps = sum(min(kt - 1, T - 1 - t + pt) - max(0, pt - t) + 1 for t in range(T + 2 * pt - kt + 1))
    tiles = Ho * -(-Wo // 120) * (N * taps if not pair else -(-N * T // 2) * kt)   # (plane, temporal tap) pairs x row x column tiles
    return 2.0 * tiles * (112 if transposed else 128) * ncols * kh * 32


def time_graph(fn):
    for _ in range(2):
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
    return e0.elapsed_time(e1) / (ROUNDS * REP)


def main(names):
    dev = torch.device("cuda:0")
    lib = _lib.load()
    if "--rows" in names:
        i = names.index("--rows")
        lib.b2_debug_set_stem_rows({"2": 2, "4": 4, "4t": 4 | 16}[names[i + 1]])
        names = names[:i] + names[i + 2:]
    names = names or list(SHAPES)
    print("card: %s" % card(), flush=True)
    for name in names:
        N, T, H, W, K, k, p, pool = SHAPES[name]
        torch.manual_seed(0)
        conv = nn.Conv3d(3, K, k, stride=(1, 2, 2), padding=p, bias=False).to(dev)
        bn = nn.BatchNorm3d(K).eval().to(dev)
        with torch.no_grad():
            bn.running_mean.normal_(0, 0.1); bn.running_var.uniform_(0.5, 1.5); bn.weight.uniform_(0.5, 1.5); bn.bias.normal_(0, 0.1)
            a = ops.from_ncdhw(torch.randn(N, 3, T, H, W, device=dev))
            To, Ho, Wo = T + 2 * p[0] - k[0] + 1, (H + 2 * p[1] - k[1]) // 2 + 1, (W - 1) // 2 + 1
            conv_fn = lambda: engine.conv_bn_act(conv, bn, a, relu=True, pool_w=pool is not None)
            stem_fn = (lambda: ops.maxpool3d(conv_fn(), *pool)) if pool is not None else conv_fn
            ms_conv = time_graph(conv_fn)
            ms_stem = time_graph(stem_fn) if pool is not None else ms_conv
            conv_fn()
            torch.cuda.synchronize()
            G = lib.b2_debug_last_stem_rows()
            info = (ctypes.c_int * 5)()
            lib.b2_debug_last_kernel(info)
            transposed = bool(info[1]) and G == 4
        alg = 2.0 * N * To * Ho * Wo * K * 3 * k[0] * k[1] * 7
        exe = executed_flops(N, T, Ho, Wo, K, k[0], k[1], p[0], transposed)
        print("%-11s N=%-3d T=%-2d %dx%d %s->%d  G=%-2s  conv %7.3f ms  stem %7.3f ms  algorithmic %6.1f TFLOP/s  executed %6.1f TFLOP/s"
              % (name, N, T, H, W, "x".join(map(str, k)), K, "%d%s" % (G, "t" if transposed else ""), ms_conv, ms_stem,
                 alg / ms_conv / 1e9, exe / ms_conv / 1e9), flush=True)


if __name__ == "__main__":
    main(sys.argv[1:])
