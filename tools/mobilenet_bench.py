#!/usr/bin/env python
"""Time MobileNetV2 inference on the engine, per depthwise layer and against torch's fp16 cuDNN, in one process on one card.

    python tools/mobilenet_bench.py [--batch 256] [--size 224] [--steps 50] [--warmup 10] [--no-torch]

* images/s of ``mobilenetv2`` as CUDA-graph replays (``graph.GraphedForward``) after ``--warmup`` replays;
* every depthwise layer's kernel time (CUDA events around each library launch, ``ops.profile``, median over ``--profile-reps``
  eager forwards) and its share of the HBM bound: the input and output bytes from the shapes over 3.35 TB/s (the H100 SXM data
  sheet figure; the measured card's power limit and clock are reported beside it);
* for context, the same network as ``oracle.mobilenet.forward`` on fp16 CUDA copies of the parameters, input and filters in
  ``channels_last``, ``cudnn.benchmark`` on, eager, timed with CUDA events.
Prints one JSON line.  Needs an H100; there is no CPU fallback."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import pretorched_x_b200 as P  # noqa: E402
from pretorched_x_b200 import ops  # noqa: E402
from pretorched_x_b200.graph import GraphedForward  # noqa: E402
from oracle import functional as OF  # noqa: E402
from oracle import mobilenet as OM  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return dict(zip(("gpu", "power_limit", "sm_clock", "max_sm_clock"), [v.strip() for v in out.split(",")]))
    except Exception:
        return dict(gpu=torch.cuda.get_device_name(0), power_limit="unknown", sm_clock="unknown", max_sm_clock="unknown")


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--size", type=int, default=224)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--profile-reps", type=int, default=5)
    ap.add_argument("--no-torch", action="store_true", help="skip the cuDNN comparison")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mobilenet_bench needs an H100 (no GPU found)")
    info = card()
    torch.manual_seed(0)
    model = OF.randomize_bn_(P.mobilenetv2(num_classes=1000, pretrained=None), 1).eval().cuda()
    x = torch.randn((args.batch, 3, args.size, args.size), generator=torch.Generator().manual_seed(1)).cuda()

    g = GraphedForward(model, x)
    ms = timed(g, args.steps, args.warmup)

    per = {}
    with torch.no_grad():
        model(x)
        for _ in range(args.profile_reps):
            with ops.profile() as prof:
                model(x)
            for i, r in enumerate(r for r in prof.rows if r["kind"] == "dwconv"):
                per.setdefault(i, dict(desc=r["desc"], bytes=r["bytes"], ms=[]))["ms"].append(r["ms"])
    layers = []
    for i in sorted(per):
        d = per[i]
        t = statistics.median(d["ms"])
        bound = d["bytes"] / HBM_BYTES_PER_S * 1e3
        layers.append(dict(layer=i, desc=d["desc"], ms=round(t, 4), bytes=int(d["bytes"]), hbm_bound_ms=round(bound, 4),
                           share_of_hbm_bound=round(bound / t, 3), achieved_tb_s=round(d["bytes"] / (t * 1e-3) / 1e12, 3)))
    dw_total = sum(r["ms"] for r in layers)

    ref_ms = None
    if not args.no_torch:
        sd = {}
        for k, v in model.state_dict().items():
            t = v.detach().clone().cuda()
            if t.is_floating_point():
                t = t.half()
                if t.dim() == 4:
                    t = t.contiguous(memory_format=torch.channels_last)
            sd[k] = t
        xh = x.half().contiguous(memory_format=torch.channels_last)
        torch.backends.cudnn.benchmark = True
        with torch.no_grad():
            ref_ms = timed(lambda: OM.forward(xh, sd), args.steps, args.warmup)

    print(json.dumps(dict(metric="mobilenetv2 inference", input=[args.batch, 3, args.size, args.size], steps=args.steps, warmup=args.warmup,
                          engine_graph_ms=round(ms, 3), engine_images_per_s=round(args.batch / ms * 1e3, 1),
                          torch_cudnn_fp16_eager_ms=None if ref_ms is None else round(ref_ms, 3),
                          torch_cudnn_fp16_eager_images_per_s=None if ref_ms is None else round(args.batch / ref_ms * 1e3, 1),
                          depthwise_total_ms=round(dw_total, 3), depthwise_layers=layers, **info)))


if __name__ == "__main__":
    main()
