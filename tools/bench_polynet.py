"""PolyNet: engine vs the reference network on cuDNN, and TRN-MSTRN on PolyNet.

    python tools/bench_polynet.py [--batch 256] [--videos 16] [--segments 8] [--iters 20] [--no-profile]

Engine: ``GraphedForward`` replays (B images, 331^2; TRN(arch='polynet', consensus='MSTRN') on videos x segments frames), CUDA
events around ``iters`` replays after warm-up.  cuDNN: the package's PolyNet parameters loaded into oracle/polynet.py's
functional restatement in fp16 channels_last (cudnn.benchmark on), CUDA-graph captured.  Both run the rescaled init of
oracle.polynet.rescale_ with random BatchNorm statistics.  The multiply-accumulates per image are counted from the convolution
and linear shapes the restatement runs.  A profiled eager pass (ops.profile) splits the engine's forward by launch kind.  Prints
one JSON object with the card name, power limit and maximum SM clock read in the same run; needs an H100.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import pretorched_x_b200 as P                   # noqa: E402
from pretorched_x_b200.graph import GraphedForward   # noqa: E402
from oracle import functional as OF             # noqa: E402
from oracle import polynet as OP                # noqa: E402
from tools.bench_bninception import _card, _graphed, _profile, _time   # noqa: E402


def _macs_per_image(model, sd):
    """Multiply-accumulates of one 331^2 image, counted from every F.conv2d / F.linear the restatement calls."""
    total = [0]
    conv, lin = F.conv2d, F.linear

    def c(x, w, b=None, stride=1, padding=0, *a):
        y = conv(x, w, b, stride, padding, *a)
        total[0] += y[0].numel() * w[0].numel()
        return y

    def li(x, w, b=None):
        total[0] += w.numel()
        return lin(x, w, b)
    F.conv2d, F.linear = c, li
    try:
        with torch.no_grad():
            OP.forward(torch.zeros(1, 3, 331, 331), sd, model)
    finally:
        F.conv2d, F.linear = conv, lin
    return total[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--videos", type=int, default=16)
    ap.add_argument("--segments", type=int, default=8)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--no-profile", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_polynet needs an H100")
    dev = torch.device("cuda:0")
    torch.backends.cudnn.benchmark = True
    out = dict(card=_card(), batch=args.batch)
    torch.manual_seed(0)
    m = OP.rescale_(P.polynet(pretrained=None), 0.15)
    OF.randomize_bn_(m, 1)
    m.eval()
    sd_cpu = {k: v.detach().clone() for k, v in m.state_dict().items()}
    out["gmac_per_image"] = _macs_per_image(m, sd_cpu) / 1e9
    m = m.to(dev)
    x = torch.randn((args.batch, 3, 331, 331), generator=torch.Generator().manual_seed(1)).to(dev)
    g = GraphedForward(m, x)
    out["engine_ms"] = _time(lambda: g(x), args.iters)
    if not args.no_profile:
        kinds, total = _profile(m, x)
        out["engine_profile_ms"] = {k: round(v, 3) for k, v in sorted(kinds.items(), key=lambda kv: -kv[1])}
    # cuDNN: the same weights through the functional restatement, fp16 channels_last
    sd16 = {k: (v.to(dev).half() if v.is_floating_point() else v.to(dev)) for k, v in sd_cpu.items()}
    geom = m
    x16 = x.half().contiguous(memory_format=torch.channels_last)

    def cudnn():
        return OP.forward(x16, sd16, geom)
    with torch.no_grad():
        ref = cudnn()
        eng = m(x)
    out["cudnn_vs_engine_logit_rel_err"] = float((ref.float() - eng).abs().max() / eng.abs().max())
    out["cudnn_fp16_ms"] = _time(_graphed(cudnn), args.iters)
    del g, sd16
    torch.cuda.empty_cache()
    # TRN-MSTRN on PolyNet
    torch.manual_seed(0)
    t = OP.rescale_(P.TRN(10, num_segments=args.segments, arch="polynet", consensus="MSTRN", pretrained=None,
                          frame_bottleneck_dim=128, video_feature_dim=64), 0.15)
    OF.randomize_bn_(t, 1)
    t = t.eval().to(dev)
    xv = torch.randn((args.videos, args.segments, 3, 331, 331), generator=torch.Generator().manual_seed(2)).to(dev)
    np.random.seed(0)
    gt = GraphedForward(t, xv, warmup=1)
    out["trn_mstrn_ms"] = _time(lambda: gt(xv), args.iters)
    out["trn_shape"] = [args.videos, args.segments]
    out["tflops_engine"] = 2 * out["gmac_per_image"] * args.batch / out["engine_ms"]
    out["tflops_cudnn"] = 2 * out["gmac_per_image"] * args.batch / out["cudnn_fp16_ms"]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
