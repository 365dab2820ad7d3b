#!/usr/bin/env python
"""Time one fine-tuning step (forward + backward + SGD step) of TRN-MSTRN on a resnet50 backbone on the engine and on torch's
own fp16 cuDNN autograd, in the same process on the same card.

    python tools/bench_finetune_trn.py [--batch 16] [--segments 8] [--size 224] [--ks 4,3] [--steps 10] [--warmup 3] [--graph]

Engine: ``TRN(339, arch='resnet50', consensus='MSTRN').fine_tune(k)`` + SGD on the trainable parameters (the backbone's
``layer{k}..layer4``, the relation and the final Linear), eval-mode (frozen) BatchNorm.  Baseline:
``oracle.functional.trn_forward`` on fp16 CUDA copies of the same parameters (the same ones trainable), filters in
``channels_last``, ``cudnn.benchmark`` on, SGD on the fp16 trainable parameters.  Both draw the multi-scale frame tuples from
NumPy's global RNG the same way.  Both timed with CUDA events over ``--steps`` steps after ``--warmup`` steps.  A separate
profiled engine step reports the share of the backward time spent in the weight-gradient kernel (CUDA events around every
library launch, ``ops.profile``).  The card name and power limit are read in the same run.  Prints one JSON line.  Needs an
H100; there is no CPU fallback.

``--graph``: instead, the same engine step run eagerly and as a replay of one CUDA graph (``graph.GraphedFineTuneStep``, which
draws the frame tuples of every replay on the host like the eager forward) on the same model and optimizer, timed alternately
(``--rounds`` rounds of ``--steps`` steps each, median reported), and the device time the replayed step spends re-packing the
trainable filters (``bench_finetune.repack_cost``)."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

import pretorched_x_b200 as P  # noqa: E402
from pretorched_x_b200 import ops  # noqa: E402
from oracle import functional as OF  # noqa: E402
from pretorched_x_b200.graph import GraphedFineTuneStep  # noqa: E402
from bench_finetune import alternate, card, repack_cost, timed  # noqa: E402

NUM_CLASSES = 339


def engine_case(x, target, k, segments, steps, warmup):
    torch.manual_seed(0)
    model = P.TRN(NUM_CLASSES, num_segments=segments, arch="resnet50", consensus="MSTRN", pretrained=None)
    model = OF.randomize_bn_(model, 1).eval().cuda().fine_tune(k)
    opt = torch.optim.SGD([p for p in model.parameters() if p.requires_grad], lr=1e-5, momentum=0.9)
    np.random.seed(0)

    def step():
        opt.zero_grad(set_to_none=True)
        F.cross_entropy(model(x), target).backward()
        opt.step()

    ms = timed(step, steps, warmup)
    opt.zero_grad(set_to_none=True)
    loss = F.cross_entropy(model(x), target)
    torch.cuda.synchronize()
    b0, b1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    with ops.profile() as prof:
        b0.record()
        loss.backward()
        b1.record()
    bwd_ms = b0.elapsed_time(b1)
    wgrad_ms = sum(r["ms"] for r in prof.rows if r["kind"] == "wgrad")
    by_kind = {}
    for r in prof.rows:
        by_kind[r["kind"]] = by_kind.get(r["kind"], 0.0) + r["ms"]
    return ms, bwd_ms, wgrad_ms, by_kind, model


def graph_case(x, target, k, segments, steps, warmup, rounds):
    torch.manual_seed(0)
    model = P.TRN(NUM_CLASSES, num_segments=segments, arch="resnet50", consensus="MSTRN", pretrained=None)
    model = OF.randomize_bn_(model, 1).eval().cuda().fine_tune(k)
    opt = torch.optim.SGD([p for p in model.parameters() if p.requires_grad], lr=1e-5, momentum=0.9)
    np.random.seed(0)

    def step():
        opt.zero_grad(set_to_none=True)
        F.cross_entropy(model(x), target).backward()
        opt.step()

    graphed = GraphedFineTuneStep(model, opt, F.cross_entropy, x, target)
    row = dict(k=k, **alternate(step, graphed, steps, warmup, rounds))
    row.update(repack_cost(model, x, steps, warmup))
    row["repack_share_of_replayed_step"] = round(row["repack_ms"] / row["graph_ms_per_step"], 4)
    return row


def torch_case(model, x, target, segments, steps, warmup):
    trainable = {n for n, p in model.named_parameters() if p.requires_grad}
    sd = {}
    for n, v in model.state_dict().items():
        t = v.detach().clone().cuda()
        if t.is_floating_point():
            t = t.half()
            if t.dim() == 4:
                t = t.contiguous(memory_format=torch.channels_last)
        sd[n] = t.requires_grad_(n in trainable)
    opt = torch.optim.SGD([sd[n] for n in trainable], lr=1e-5, momentum=0.9)
    xh = x.half()
    torch.backends.cudnn.benchmark = True
    np.random.seed(0)

    def step():
        opt.zero_grad(set_to_none=True)
        F.cross_entropy(OF.trn_forward(xh, sd, "resnet50", "MSTRN", segments).float(), target).backward()
        opt.step()

    return timed(step, steps, warmup)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--segments", type=int, default=8)
    ap.add_argument("--size", type=int, default=224)
    ap.add_argument("--ks", default="4,3")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-torch", action="store_true", help="skip the cuDNN baseline")
    ap.add_argument("--graph", action="store_true", help="eager steps against CUDA-graph replays of the step")
    ap.add_argument("--rounds", type=int, default=5, help="--graph: alternating rounds")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_finetune_trn needs an H100 (no GPU found)")
    name, power = card()
    shape = (args.batch, args.segments, 3, args.size, args.size)
    x = torch.randn(shape, generator=torch.Generator().manual_seed(1)).cuda()
    target = torch.randint(0, NUM_CLASSES, (args.batch,), generator=torch.Generator().manual_seed(2)).cuda()
    if args.graph:
        rows = []
        for k in [int(v) for v in args.ks.split(",")]:
            rows.append(graph_case(x, target, k, args.segments, args.steps, args.warmup, args.rounds))
            torch.cuda.empty_cache()
        print(json.dumps(dict(metric="ms per fine-tuning step (forward + backward + SGD step), eager vs CUDA-graph replay",
                              model="TRN-MSTRN resnet50", input=list(shape), steps=args.steps, warmup=args.warmup,
                              rounds=args.rounds, gpu=name, power_limit=power, results=rows)))
        return
    rows = []
    for k in [int(v) for v in args.ks.split(",")]:
        ms, bwd_ms, wgrad_ms, by_kind, model = engine_case(x, target, k, args.segments, args.steps, args.warmup)
        ref_ms = None if args.no_torch else torch_case(model, x, target, args.segments, args.steps, args.warmup)
        del model
        torch.cuda.empty_cache()
        rows.append(dict(k=k, engine_ms_per_step=round(ms, 3), torch_cudnn_fp16_ms_per_step=None if ref_ms is None else round(ref_ms, 3),
                         speedup=None if ref_ms is None else round(ref_ms / ms, 3),
                         profiled_backward_ms=round(bwd_ms, 3), wgrad_ms=round(wgrad_ms, 3),
                         wgrad_share_of_backward=round(wgrad_ms / bwd_ms, 3) if bwd_ms > 0 else None,
                         backward_launch_ms_by_kind={kk: round(v, 3) for kk, v in sorted(by_kind.items())}))
    print(json.dumps(dict(metric="ms per fine-tuning step (forward + backward + SGD step)", model="TRN-MSTRN resnet50",
                          input=list(shape), steps=args.steps, warmup=args.warmup, gpu=name, power_limit=power, results=rows)))


if __name__ == "__main__":
    main()
