"""ResNeXt-101 32x4d / 64x4d forward throughput on the engine vs the same network on cuDNN, and TRN-MSTRN on resnext101_32x4d.

    python tools/bench_resnext101.py [--batch 256] [--iters 20] [--out DIR]

Engine: ``GraphedForward`` replays of resnext101_32x4d and resnext101_64x4d, fp32 NCHW 224^2 input, B images, CUDA events around
``iters`` replays after warm-up.  cuDNN: oracle/resnext.py's functional restatement in fp16 channels_last
(torch.backends.cudnn.benchmark on), also CUDA-graph captured.  TRN-MSTRN: 16 videos x 8 segments on the engine, graph-replayed.
The card's name, power limit and maximum SM clock are printed with the numbers.  Prints one JSON object; needs an H100.
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
from pretorched_x_b200.graph import GraphedForward   # noqa: E402
from oracle import functional as OF             # noqa: E402
from oracle import resnext as OX                # noqa: E402


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
        raise SystemExit("bench_resnext101 needs an H100")
    dev = torch.device("cuda:0")
    torch.backends.cudnn.benchmark = True
    B = args.batch
    x = OF.seeded_input((B, 3, 224, 224), 2).to(dev)
    result = dict(card=_card(), batch=B, iters=args.iters, models={})
    for arch in OX.ARCHS:
        torch.manual_seed(0)
        model = P.__dict__[arch](pretrained=None)
        OF.randomize_bn_(model, 1)
        model = model.eval().to(dev)
        g = GraphedForward(model, x)
        ms = _time(lambda: g(), args.iters)
        row = dict(engine_ms=ms, engine_img_s=B / ms * 1e3)
        del g
        sd = {k: v.detach().half().to(dev) if v.is_floating_point() else v.to(dev) for k, v in model.state_dict().items()}
        xh = x.half().contiguous(memory_format=torch.channels_last)
        ref = _graphed(lambda t: OX.forward(t, sd, arch), xh)
        row["cudnn_fp16_ms"] = _time(ref, args.iters)
        row["cudnn_fp16_img_s"] = B / row["cudnn_fp16_ms"] * 1e3
        result["models"][arch] = row
        del model, ref, sd
        torch.cuda.empty_cache()
    torch.manual_seed(0)
    trn = P.TRN(10, num_segments=8, arch="resnext101_32x4d", consensus="MSTRN", pretrained=None, frame_bottleneck_dim=128,
                video_feature_dim=64)
    OF.randomize_bn_(trn, 1)
    trn = trn.eval().to(dev)
    xv = OF.seeded_input((16, 8, 3, 224, 224), 2).to(dev)
    g = GraphedForward(trn, xv)
    ms = _time(lambda: g(), args.iters)
    result["trn_resnext101_32x4d_MSTRN_16x8"] = dict(engine_ms=ms, videos_s=16 / ms * 1e3)
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bench_resnext101.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
