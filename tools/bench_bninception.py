"""BNInception and TRN-MSTRN on BNInception: engine vs the same network on cuDNN, and the split GEMM vs the GEMMs it replaces.

    python tools/bench_bninception.py [--batch 256] [--videos 16] [--segments 8] [--iters 20] [--out DIR]

Engine: ``GraphedForward`` replays of bninception (B images, 224^2) and of TRN(arch='bninception', consensus='MSTRN') (videos x
segments frames), CUDA events around ``iters`` replays after warm-up.  cuDNN: oracle/bninception.py's functional restatement in fp16
channels_last (cudnn.benchmark on), CUDA-graph captured for bninception and eager for the TRN (its relation indexes frames with host
lists).  A separate profiled eager pass (ops.profile, CUDA events per launch)
attributes the engine's time to its launch kinds: split GEMMs (``gemm_split``), slice convolutions (``conv_slice``), pools
(``pool``).  Per block, the split GEMM of the three 1x1 heads is timed at the ops level against the three stand-alone b2_gemm_f16
launches it replaces (same operands, CUDA-graph captured).  Prints one JSON object; needs an H100.
"""
import argparse
import json
import os
import subprocess
import sys
from collections import defaultdict

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import pretorched_x_b200 as P                   # noqa: E402
from pretorched_x_b200 import engine, ops       # noqa: E402
from pretorched_x_b200.graph import GraphedForward   # noqa: E402
from pretorched_x_b200.models import bninception as PB   # noqa: E402
from oracle import bninception as OB            # noqa: E402
from oracle import functional as OF             # noqa: E402


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception:           # noqa: BLE001 - the card description is informational
        return "unknown"


def _time(fn, iters):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def _graphed(fn, *xs):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.no_grad():
        for _ in range(2):
            fn(*xs)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g), torch.no_grad():
        fn(*xs)
    return g.replay


def _profile(model, x):
    with torch.no_grad(), ops.profile() as prof:
        model(x)
    kinds = defaultdict(float)
    for r in prof.rows:
        kinds[r["kind"]] += r["ms"]
    return dict(kinds), sum(kinds.values())


def _split_vs_three(model, B, iters):
    """Per block: the split GEMM over the block input against the three stand-alone GEMMs (1x1 head, 3x3 reduce, double reduce)."""
    rows = {}
    dev = next(model.parameters()).device
    for spec in PB.BLOCKS:
        n, cin, c1, (c3r, _), (cdr, _), _ = spec
        hw = {'3': 28, '4': 14, '5': 7}[n[0]]
        M = B * hw * hw
        a = torch.rand((M, cin), device=dev).to(torch.float16)
        heads = ([('inception_%s_1x1' % n, c1)] if c1 is not None else []) + [('inception_%s_3x3_reduce' % n, c3r),
                                                                              ('inception_%s_double_3x3_reduce' % n, cdr)]
        w, sc, sh = engine._split_pack(model, [h for h, _ in heads], cin)
        npad, box0 = ops.split_plan([k for _, k in heads])
        dests = [torch.empty((M, k), dtype=torch.float16, device=dev) for _, k in heads]
        parts = [(w[64 * b:64 * b + k], sc[64 * b:64 * b + k].contiguous(), sh[64 * b:64 * b + k].contiguous(), k)
                 for b, (_, k) in zip(box0, heads)]
        split = _graphed(lambda: ops.gemm_split(a, w, sc, sh, M, cin, dests, relu=True))
        three = _graphed(lambda: [ops.gemm(a, pw, ps, ph, M, k, cin, relu=True, out=d) for (pw, ps, ph, k), d in zip(parts, dests)])
        rows[n] = dict(M=M, K=cin, cols=[k for _, k in heads], packed=npad, split_ms=_time(split, iters), three_ms=_time(three, iters))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--videos", type=int, default=16)
    ap.add_argument("--segments", type=int, default=8)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_bninception needs an H100")
    dev = torch.device("cuda:0")
    torch.backends.cudnn.benchmark = True
    B = args.batch
    result = dict(card=_card(), batch=B, iters=args.iters)

    torch.manual_seed(0)
    model = P.bninception(pretrained=None)
    OF.randomize_bn_(model, 1)
    model = model.eval().to(dev)
    x = OF.seeded_input((B, 3, 224, 224), 2).to(dev)
    g = GraphedForward(model, x)
    ms = _time(lambda: g(), args.iters)
    row = dict(engine_ms=ms, engine_img_s=B / ms * 1e3)
    del g
    row["profiled_ms_by_kind"], row["profiled_ms_total"] = _profile(model, x)
    sd = {k: v.detach().half() if v.is_floating_point() else v for k, v in model.state_dict().items()}
    xh = x.half().contiguous(memory_format=torch.channels_last)
    ref = _graphed(lambda t: OB.forward(t, sd), xh)
    row["cudnn_fp16_ms"] = _time(ref, args.iters)
    row["cudnn_fp16_img_s"] = B / row["cudnn_fp16_ms"] * 1e3
    del ref
    result["bninception"] = row
    result["split_vs_three_gemms"] = _split_vs_three(model, B, args.iters)
    del model
    torch.cuda.empty_cache()

    V, T = args.videos, args.segments
    torch.manual_seed(0)
    trn = P.TRN(339, num_segments=T, arch="bninception", consensus="MSTRN", pretrained=None)
    OF.randomize_bn_(trn, 1)
    trn = trn.eval().to(dev)
    xv = OF.seeded_input((V, T, 3, 224, 224), 2).to(dev)
    np.random.seed(0)
    g = GraphedForward(trn, xv)
    ms = _time(lambda: g(), args.iters)
    trow = dict(videos=V, segments=T, engine_ms=ms, engine_videos_s=V / ms * 1e3)
    del g
    np.random.seed(0)
    trow["profiled_ms_by_kind"], trow["profiled_ms_total"] = _profile(trn, xv)
    sd = {k: v.detach().half() if v.is_floating_point() else v for k, v in trn.state_dict().items()}
    xvh = xv.half()
    np.random.seed(0)
    with torch.no_grad():     # eager: the restatement indexes frames with host lists, which a CUDA graph cannot capture
        trow["cudnn_fp16_eager_ms"] = _time(lambda: OB.trn_forward(xvh, sd, T), args.iters)
    result["trn_bninception_mstrn"] = trow

    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_bninception.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
