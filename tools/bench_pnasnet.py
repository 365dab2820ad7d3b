"""PNASNet-5-Large forward throughput on the engine vs the same network on cuDNN, and the share of the engine's forward spent in the
depthwise passes.

    python tools/bench_pnasnet.py [--batch 256] [--iters 20] [--out DIR]

Engine: ``GraphedForward`` replays of pnasnet5large, fp32 NCHW 331^2 input, B images, CUDA events around ``iters`` replays after
warm-up.  Both sides run the fixture's init (oracle.pnasnet.rescale_) with random BatchNorm statistics.
cuDNN: oracle/pnasnet.py's functional restatement of the reference network in fp16 channels_last, input and filters alike
(torch.backends.cudnn.benchmark on), also CUDA-graph captured, timed in the same run.  Depthwise share: one eager forward under
``ops.profile`` (CUDA events around every launch, in a pass of its own after the timed ones): the summed time of the ``dwconv``
launches over the summed time of all launches, with the summed time of the GEMMs (pointwise 1x1 convolutions, ReluConvBn,
FactorizedReduction) beside it, and the depthwise passes' algorithmic bytes (input read once, output written once) over their time.  The card's name, power limit and maximum SM clock are read in the same run.  Prints
one JSON object; needs an H100.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import pretorched_x_b200 as P                   # noqa: E402
from pretorched_x_b200 import ops               # noqa: E402
from pretorched_x_b200.graph import GraphedForward   # noqa: E402
from oracle import functional as OF             # noqa: E402
from oracle import pnasnet as OPn               # noqa: E402


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


def _graphed(fn, x):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s), torch.no_grad():
        for _ in range(2):
            fn(x)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g), torch.no_grad():
        fn(x)
    return g.replay


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_pnasnet needs an H100")
    dev = torch.device("cuda:0")
    torch.backends.cudnn.benchmark = True
    B = args.batch
    x = OF.seeded_input((B, 3, 331, 331), 2).to(dev)
    torch.manual_seed(0)
    model = OPn.rescale_(P.pnasnet5large(pretrained=None))
    OF.randomize_bn_(model, 1)
    model = model.eval().to(dev)
    g = GraphedForward(model, x)
    ms = _time(lambda: g(), args.iters)
    result = dict(card=_card(), batch=B, input=[331, 331], iters=args.iters, engine_ms=ms, engine_img_s=B / ms * 1e3)
    del g
    sd = {k: v.detach().half().to(dev) if v.is_floating_point() else v.to(dev) for k, v in model.state_dict().items()}
    sd = {k: v.contiguous(memory_format=torch.channels_last) if v.dim() == 4 else v for k, v in sd.items()}
    xh = x.half().contiguous(memory_format=torch.channels_last)
    ref = _graphed(lambda t: OPn.forward(t, sd), xh)
    result["cudnn_fp16_ms"] = _time(ref, args.iters)
    result["cudnn_fp16_img_s"] = B / result["cudnn_fp16_ms"] * 1e3
    del ref, sd
    torch.cuda.empty_cache()
    with torch.no_grad():
        model(x)
        torch.cuda.synchronize()
        with ops.profile() as prof:
            model(x)
    total = sum(r["ms"] for r in prof.rows)
    dw = sum(r["ms"] for r in prof.rows if r["kind"] == "dwconv")
    pw = sum(r["ms"] for r in prof.rows if r["kind"] in ("gemm", "gemm_preact"))
    result["profile"] = dict(launches=len(prof.rows), summed_ms=total, dwconv_ms=dw, dwconv_share=dw / total,
                             dwconv_launches=sum(r["kind"] == "dwconv" for r in prof.rows), gemm_ms=pw,
                             dwconv_bytes=sum(r["bytes"] for r in prof.rows if r["kind"] == "dwconv"))
    result["profile"]["dwconv_gb_s"] = result["profile"]["dwconv_bytes"] / (dw * 1e-3) / 1e9
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_pnasnet.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
