"""VGG-16, VGG-16-BN, VGG-19 and AlexNet on the engine against torchvision's models on cuDNN, TRN-MSTRN on VGG-16, and the
classifier GEMMs split-K against the unsplit persistent GEMM.

    python tools/bench_vgg.py [--batch 256] [--iters 20] [--rounds 5]

Engine: ``GraphedForward`` replays of B images at 224^2.  cuDNN: torchvision's model with the same parameters in fp16,
channels_last, cudnn.benchmark on, CUDA-graph captured.  The two are alternated ``rounds`` times (CUDA events around ``iters``
replays each) and the medians reported.  A profiled eager pass (ops.profile) splits the engine's time by launch kind.  The three
classifier GEMMs (fc6 25088 / 9216 -> 4096, fc7 4096 -> 4096, last_linear 4096 -> 1000) are timed at B and at 16 rows, split-K with
the planner's splits against the unsplit persistent GEMM, alternated in the same rounds.  Prints one JSON object with the card
name and power limit read in the same run; needs an H100.
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
from pretorched_x_b200 import ops, ops_vgg      # noqa: E402
from pretorched_x_b200.graph import GraphedForward   # noqa: E402
from oracle import functional as OF             # noqa: E402
from tools.bench_bninception import _card, _graphed, _time   # noqa: E402

TRN_KW = dict(frame_bottleneck_dim=128, video_feature_dim=64)


def _profile(model, x):
    with torch.no_grad(), ops.profile() as prof:
        model(x)
    kinds = defaultdict(float)
    for r in prof.rows:
        kinds[r["kind"]] += r["ms"]
    return dict(kinds)


def _torchvision(arch, m):
    """torchvision's model holding ``m``'s parameters (the reference's names mapped back to features.* / classifier.<i>.*)."""
    tv = getattr(tvm, arch)(weights=None)
    idx = {"linear0": 1, "linear1": 4, "last_linear": 6} if arch == "alexnet" else {"linear0": 0, "linear1": 3, "last_linear": 6}
    sd = {}
    for k, v in m.state_dict().items():
        head, leaf = k.split(".", 1)
        sd[k[1:] if head == "_features" else "classifier.%d.%s" % (idx[head], leaf)] = v
    tv.load_state_dict(sd)
    return tv


def _classifier_gemms(rows, iters, rounds, sms):
    dev = torch.device("cuda:0")
    out = []
    for name, N, K in (("fc6 vgg", 4096, 25088), ("fc6 alexnet", 4096, 9216), ("fc7", 4096, 4096), ("last_linear", 1000, 4096)):
        for M in rows:
            a = torch.rand((M, K), device=dev).half()
            w = (torch.randn(N, K, device=dev) * K ** -0.5).half()
            s, t = torch.ones(N, device=dev), torch.zeros(N, device=dev)
            S = ops_vgg.splitk_plan(M, N, K, sms)
            plain = _graphed(lambda: ops.gemm(a, w, s, t, M, N, K, relu=True))
            split = _graphed(lambda: ops_vgg.gemm_splitk(a, w, s, t, M, N, K, max(S, 2), relu=True))
            p_ms, s_ms = [], []
            for _ in range(rounds):
                p_ms.append(_time(plain, iters))
                s_ms.append(_time(split, iters))
            p, q = statistics.median(p_ms), statistics.median(s_ms)
            out.append(dict(gemm=name, M=M, N=N, K=K, splits=max(S, 2), planned_splits=S, unsplit_ms=p, splitk_ms=q,
                            unsplit_weight_GBps=2.0 * N * K / p / 1e6, splitk_weight_GBps=2.0 * N * K / q / 1e6))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    torch.backends.cudnn.benchmark = True
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    out = {"card": _card(), "batch": args.batch}
    for arch in ("vgg16", "vgg16_bn", "vgg19", "alexnet"):
        torch.manual_seed(0)
        m = P.__dict__[arch](pretrained=None)
        OF.randomize_bn_(m, 1)
        m = m.eval().to(dev)
        tv = _torchvision(arch, m).eval().to(dev).half().to(memory_format=torch.channels_last)
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
        out[arch] = dict(engine_ms=statistics.median(eng_ms), cudnn_fp16_ms=statistics.median(ref_ms), engine_rounds_ms=eng_ms,
                         cudnn_rounds_ms=ref_ms, images_per_s=args.batch / statistics.median(eng_ms) * 1e3,
                         logits_rel_diff_vs_cudnn=float((got - want).abs().max() / want.abs().max()),
                         profile_ms_by_kind=_profile(m, x))
        del m, g, tv, ref
        torch.cuda.empty_cache()
    torch.manual_seed(0)
    trn = P.TRN(10, num_segments=8, arch="vgg16", consensus="MSTRN", pretrained=None, **TRN_KW).eval().to(dev)
    xt = torch.rand((16, 8, 3, 224, 224), device=dev)
    gt = GraphedForward(trn, xt)
    out["trn_vgg16_MSTRN_16x8_ms"] = statistics.median([_time(lambda: gt(xt), args.iters) for _ in range(args.rounds)])
    del trn, gt
    torch.cuda.empty_cache()
    out["classifier_gemms"] = _classifier_gemms((args.batch, 16), args.iters, args.rounds, sms)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
