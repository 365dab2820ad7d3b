"""Inception-v4, Inception-ResNet-v2 and Inception-v3: engine vs the same network on cuDNN, TRN-MSTRN on each, and the slab kernel
vs the gather kernel on every valid-padded convolution.

    python tools/bench_inception.py [--batch 256] [--videos 16] [--segments 8] [--iters 20] [--archs inceptionv3 ...] [--no-convs]

Engine: ``GraphedForward`` replays (B images, 299^2; TRN(arch, consensus='MSTRN') on videos x segments frames), CUDA events around
``iters`` replays after warm-up.  cuDNN: oracle/inception.py's functional restatement in fp16 channels_last (cudnn.benchmark on),
CUDA-graph captured; for Inception-v3, torchvision's own Inception3 with the same weights in fp16 channels_last (cudnn.benchmark
on), CUDA-graph captured, and its multiply-accumulates per image counted from the convolution and linear shapes (forward hooks).
Inception-v3's weights are rescaled to their fan-in (oracle.inceptionv3.fan_in_scale_) so that neither arm overflows fp16.  A
profiled eager pass (ops.profile) splits the engine's time by launch kind (for Inception-v3 also TRN's).  Unless --no-convs, per
valid-padded shape (oracle/inception.VALID) at B, the slice entry (slab kernel) against the plain entry with the gather kernel
forced (b2_debug_set_conv_algo(1)), each CUDA-graph captured.  Prints one JSON object with the card name and power limit read in
the same run; needs an H100.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import pretorched_x_b200 as P                   # noqa: E402
from pretorched_x_b200 import _lib, ops         # noqa: E402
from pretorched_x_b200.graph import GraphedForward   # noqa: E402
from pretorched_x_b200.ops import Act           # noqa: E402
from oracle import functional as OF             # noqa: E402
from oracle import inception as OI              # noqa: E402
from oracle import inceptionv3 as OV3           # noqa: E402
from oracle.inception import VALID              # noqa: E402
from tools.bench_bninception import _card, _graphed, _profile, _time   # noqa: E402


def _conv_pair(N, C, H, K, kh, kw, s, ph, pw, iters):
    dev = torch.device("cuda:0")
    conv = torch.nn.Conv2d(C, K, (kh, kw), stride=s, padding=(ph, pw)).to(dev)
    pc = ops.PackedConv(conv.weight.detach(), conv.bias, None, (1, s, s), (0, ph, pw), in_pitch=C)
    a = Act(torch.rand((N * H * H, C), device=dev).half(), N, 1, H, H, C)
    Ho = (H - kh) // s + 1
    y = torch.empty((N * Ho * Ho, K), dtype=torch.float16, device=dev)
    slab = _time(_graphed(lambda: ops.conv_slice(a, pc, y)), iters)
    lib = _lib.load()
    lib.b2_debug_set_conv_algo(1)
    try:
        gather = _time(_graphed(lambda: ops.conv(a, pc, relu=True)), iters)
    finally:
        lib.b2_debug_set_conv_algo(0)
    mac = N * Ho * Ho * K * C * kh * kw
    return dict(shape="%d->%d %dx%d s%d valid %d^2" % (C, K, kh, kw, s, H), slab_ms=slab, gather_ms=gather, gmac=mac / 1e9)


def _torchvision_v3(m):
    """torchvision's Inception3 (eval, fp16, channels_last) holding ``m``'s weights: ``last_linear`` back under ``fc``."""
    import torchvision.models.inception as tvinception
    tv = tvinception.Inception3(init_weights=False)
    sd = m.state_dict()
    tv.load_state_dict({('fc.' + k[len('last_linear.'):] if k.startswith('last_linear.') else k): v for k, v in sd.items()})
    return tv.eval().half().to(memory_format=torch.channels_last).to(next(m.parameters()).device)


def _macs_per_image(tv, hw):
    """Multiply-accumulates of one image through ``tv``'s convolutions and linear layers, from their output shapes."""
    macs = []

    def hook(mod, inp, out):
        if isinstance(mod, torch.nn.Conv2d):
            macs.append(out[0].numel() * mod.in_channels // mod.groups * mod.kernel_size[0] * mod.kernel_size[1])
        else:
            macs.append(mod.in_features * mod.out_features)
    hs = [mod.register_forward_hook(hook) for mod in tv.modules() if isinstance(mod, (torch.nn.Conv2d, torch.nn.Linear))]
    with torch.no_grad():
        tv(torch.zeros((1, 3, hw, hw), dtype=torch.float16, device=next(tv.parameters()).device))
    for h in hs:
        h.remove()
    return sum(macs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--videos", type=int, default=16)
    ap.add_argument("--segments", type=int, default=8)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--archs", nargs="+", default=["inceptionv4", "inceptionresnetv2", "inceptionv3"])
    ap.add_argument("--no-convs", action="store_true", help="skip the slab vs gather comparison of the valid-padded convolutions")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    torch.backends.cudnn.benchmark = True
    out = {"card": _card(), "batch": args.batch}
    for arch in args.archs:
        torch.manual_seed(0)
        m = P.__dict__[arch](pretrained=None)
        if arch == "inceptionv3":
            OV3.fan_in_scale_(m)
        OF.randomize_bn_(m, 1)
        m = m.eval().to(dev)
        x = torch.rand((args.batch, 3, 299, 299), device=dev)
        g = GraphedForward(m, x)
        eng = _time(lambda: g(x), args.iters)
        xc = x.half().contiguous(memory_format=torch.channels_last)
        extra = {}
        if arch == "inceptionv3":
            tv = _torchvision_v3(m)
            ref = _time(_graphed(lambda: tv(xc)), args.iters)
            extra["gmac_per_image"] = _macs_per_image(tv, 299) / 1e9
            del tv
        else:
            sd = {k: v.half() if v.is_floating_point() else v for k, v in m.state_dict().items()}
            ref = _time(_graphed(lambda: OI.forward(xc, sd, m)), args.iters)
        trn = P.TRN(10, num_segments=args.segments, arch=arch, consensus="MSTRN", pretrained=None)
        if arch == "inceptionv3":
            OV3.fan_in_scale_(trn)
            OF.randomize_bn_(trn, 1)
        trn = trn.eval().to(dev)
        v = torch.rand((args.videos, args.segments, 3, 299, 299), device=dev)
        np.random.seed(0)
        with torch.no_grad():
            trn(v)
        gt = GraphedForward(trn, v, warmup=1)
        out[arch] = dict(engine_ms=eng, cudnn_fp16_ms=ref, trn_mstrn_ms=_time(lambda: gt(v), args.iters),
                         profile_ms_by_kind=_profile(m, x)[0], **extra)
        if arch == "inceptionv3":
            np.random.seed(0)
            out[arch]["trn_profile_ms_by_kind"] = _profile(trn, v)[0]
        del m, g, trn, gt
        torch.cuda.empty_cache()
    if not args.no_convs:
        out["valid_convs"] = [_conv_pair(args.batch, *s, args.iters) for s in VALID]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
