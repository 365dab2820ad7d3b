"""DenseNet-121 / -161 on the engine against torchvision's model on cuDNN, with a per-kernel breakdown.

    python tools/bench_densenet.py [--batch 256] [--iters 20] [--rounds 5]

Engine: ``GraphedForward`` replays of B images at 224^2.  cuDNN: torchvision's DenseNet with the same parameters in fp16,
channels_last, cudnn.benchmark on, CUDA-graph captured (its forward re-concatenates every layer's input).  The two are alternated
``rounds`` times (CUDA events around ``iters`` replays each) and the medians reported.  A profiled eager pass (ops.profile)
splits the engine's time by launch kind and by launch shape.  Also timed, CUDA-graph captured: the growth-rate 3x3 convolutions
(4k -> k through the slice entry) at the four block resolutions on the 64-wide and on the k-wide N tile, and the pre-activated GEMM at N = 128, 192 and 256 on one
densenet161 layer shape (N = 192 runs as two 128-wide tiles).  Prints one JSON object with the card name and power limit read in
the same run; needs an H100.
"""
import argparse
import json
import os
import statistics
import sys
from collections import defaultdict

import torch
import torchvision.models as tvm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import pretorched_x_b200 as P                   # noqa: E402
from pretorched_x_b200 import ops               # noqa: E402
from pretorched_x_b200.graph import GraphedForward   # noqa: E402
from pretorched_x_b200.ops import Act           # noqa: E402
from oracle import functional as OF             # noqa: E402
from tools.bench_bninception import _card, _graphed, _time   # noqa: E402


def _profile(model, x, top=12):
    with torch.no_grad(), ops.profile() as prof:
        model(x)
    kinds, descs = defaultdict(float), defaultdict(lambda: [0, 0.0])
    for r in prof.rows:
        kinds[r["kind"]] += r["ms"]
        descs[r["desc"]][0] += 1
        descs[r["desc"]][1] += r["ms"]
    rows = sorted(descs.items(), key=lambda kv: -kv[1][1])[:top]
    return dict(kinds), [dict(desc=d, launches=n, ms=ms) for d, (n, ms) in rows]


def _growth_convs(B, iters):
    dev = torch.device("cuda:0")
    out = []
    for C, K in ((128, 32), (192, 48)):
        for H in (56, 28, 14, 7):
            w = torch.randn(K, C, 3, 3, device=dev) * (9 * C) ** -0.5
            pc = ops.PackedConv(w, None, None, (1, 1, 1), (0, 1, 1), in_pitch=C)
            a = Act(torch.rand((B * H * H, C), device=dev).half(), B, 1, H, H, C)
            y = torch.empty((B * H * H, 4 * K), dtype=torch.float16, device=dev)
            row = dict(shape="%d->%d 3x3 %d^2" % (C, K, H))
            for name, narrow in (("tile64", False), ("tile%d" % K, True)):
                ms = _time(_graphed(lambda: ops.conv_slice(a, pc, y[:, K:2 * K], relu=False, narrow=narrow)), iters)
                row[name + "_ms"], row[name + "_tflops"] = ms, 2.0 * B * H * H * K * C * 9 / ms / 1e9
            out.append(row)
    return out


def _preact_widths(B, iters, C_L=1056, H=14):
    dev = torch.device("cuda:0")
    M = B * H * H
    blk = torch.rand((M, 2208), device=dev).half()
    kpad = ops._round_up(C_L, 64)
    s1 = torch.zeros(kpad, device=dev)
    t1 = torch.zeros(kpad, device=dev)
    s1[:C_L], t1[:C_L] = 1.0, 0.0
    out = {}
    for N in (128, 192, 256):
        w = (torch.randn(N, C_L, device=dev) * C_L ** -0.5).half()
        s, t = torch.ones(N, device=dev), torch.zeros(N, device=dev)
        out["N=%d" % N] = _time(_graphed(lambda: ops.gemm_preact(blk, w, s, t, s1, t1, M, N, C_L)), iters)
    return dict(shape="M=%d K=%d" % (M, C_L), ms=out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    torch.backends.cudnn.benchmark = True
    out = {"card": _card(), "batch": args.batch}
    for arch in ("densenet121", "densenet161"):
        torch.manual_seed(0)
        m = P.__dict__[arch](pretrained=None)
        OF.randomize_bn_(m, 1)
        m = m.eval().to(dev)
        tv = getattr(tvm, arch)(weights=None)
        sd = dict(m.state_dict())
        sd["classifier.weight"], sd["classifier.bias"] = sd.pop("last_linear.weight"), sd.pop("last_linear.bias")
        tv.load_state_dict(sd)
        tv = tv.eval().to(dev).half().to(memory_format=torch.channels_last)
        x = torch.rand((args.batch, 3, 224, 224), device=dev)
        xc = x.half().contiguous(memory_format=torch.channels_last)
        g = GraphedForward(m, x)
        ref = _graphed(lambda: tv(xc))
        eng_ms, ref_ms = [], []
        for _ in range(args.rounds):
            eng_ms.append(_time(lambda: g(x), args.iters))
            ref_ms.append(_time(ref, args.iters))
        with torch.no_grad():
            want = tv(xc).float()
        got = g(x).clone()
        kinds, top = _profile(m, x)
        out[arch] = dict(engine_ms=statistics.median(eng_ms), cudnn_fp16_ms=statistics.median(ref_ms), engine_rounds_ms=eng_ms,
                         cudnn_rounds_ms=ref_ms, images_per_s=args.batch / statistics.median(eng_ms) * 1e3,
                         logits_rel_diff_vs_cudnn=float((got - want).abs().max() / want.abs().max()),
                         profile_ms_by_kind=kinds, profile_top_launches=top)
        del m, g, tv, ref
        torch.cuda.empty_cache()
    out["growth_convs"] = _growth_convs(args.batch, args.iters)
    out["preact_gemm_widths"] = _preact_widths(args.batch, args.iters)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
