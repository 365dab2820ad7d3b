#!/usr/bin/env python
"""Time one fine-tuning step (forward + backward + SGD step) of resnet3d50 on the engine and on torch's own fp16 cuDNN
autograd, in the same process on the same card.

    python tools/bench_finetune.py [--batch 32] [--frames 16] [--size 224] [--ks 4,3] [--steps 10] [--warmup 3]

Engine: ``get_fine_tuning_parameters(model, k)`` + SGD, eval-mode (frozen) BatchNorm.  Baseline: ``oracle.functional.forward``
on fp16 CUDA copies of the same parameters (the same ones trainable), input and filters in ``channels_last_3d``,
``cudnn.benchmark`` on, SGD on the fp16 trainable parameters.  Both timed with CUDA events over ``--steps`` steps after
``--warmup`` steps.  A separate profiled engine step reports the share of the backward time spent in the weight-gradient
kernel (CUDA events around every library launch, ``ops.profile``).  The card name and power limit are read in the same run.
Prints one JSON line.  Needs an H100; there is no CPU fallback."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

import pretorched_x_b200 as P  # noqa: E402
from pretorched_x_b200 import ops  # noqa: E402
from oracle import functional as OF  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [v.strip() for v in out.split(",")]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def timed(step, steps, warmup):
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def engine_case(x, target, k, steps, warmup):
    torch.manual_seed(0)
    model = OF.randomize_bn_(P.resnet3d50(num_classes=400, pretrained=None), 1).eval().cuda()
    opt = torch.optim.SGD(P.models.resnet3d.get_fine_tuning_parameters(model, k), lr=1e-5, momentum=0.9)

    def step():
        opt.zero_grad(set_to_none=True)
        F.cross_entropy(model(x), target).backward()
        opt.step()

    ms = timed(step, steps, warmup)
    # one profiled step: library launches inside the backward, and the backward's own wall time on the stream
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


def torch_case(model, x, target, k, steps, warmup):
    trainable = {n for n, p in model.named_parameters() if p.requires_grad}
    sd = {}
    for n, v in model.state_dict().items():
        t = v.detach().clone().cuda()
        if t.is_floating_point():
            t = t.half()
            if t.dim() == 5:
                t = t.contiguous(memory_format=torch.channels_last_3d)
        sd[n] = t.requires_grad_(n in trainable)
    params = [sd[n] for n in trainable]
    opt = torch.optim.SGD(params, lr=1e-5, momentum=0.9)
    xh = x.half().contiguous(memory_format=torch.channels_last_3d)
    torch.backends.cudnn.benchmark = True

    def step():
        opt.zero_grad(set_to_none=True)
        F.cross_entropy(OF.forward(xh, sd, "resnet3d50").float(), target).backward()
        opt.step()

    return timed(step, steps, warmup)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--size", type=int, default=224)
    ap.add_argument("--ks", default="4,3")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--no-torch", action="store_true", help="skip the cuDNN baseline")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_finetune needs an H100 (no GPU found)")
    name, power = card()
    x = torch.randn((args.batch, 3, args.frames, args.size, args.size), generator=torch.Generator().manual_seed(1)).cuda()
    target = torch.randint(0, 400, (args.batch,), generator=torch.Generator().manual_seed(2)).cuda()
    rows = []
    for k in [int(v) for v in args.ks.split(",")]:
        ms, bwd_ms, wgrad_ms, by_kind, model = engine_case(x, target, k, args.steps, args.warmup)
        ref_ms = None if args.no_torch else torch_case(model, x, target, k, args.steps, args.warmup)
        del model
        torch.cuda.empty_cache()
        rows.append(dict(k=k, engine_ms_per_step=round(ms, 3), torch_cudnn_fp16_ms_per_step=None if ref_ms is None else round(ref_ms, 3),
                         speedup=None if ref_ms is None else round(ref_ms / ms, 3),
                         profiled_backward_ms=round(bwd_ms, 3), wgrad_ms=round(wgrad_ms, 3),
                         wgrad_share_of_backward=round(wgrad_ms / bwd_ms, 3) if bwd_ms > 0 else None,
                         backward_launch_ms_by_kind={kk: round(v, 3) for kk, v in sorted(by_kind.items())}))
    print(json.dumps(dict(metric="ms per fine-tuning step (forward + backward + SGD step)", model="resnet3d50",
                          input=[args.batch, 3, args.frames, args.size, args.size], steps=args.steps, warmup=args.warmup,
                          gpu=name, power_limit=power, results=rows)))


if __name__ == "__main__":
    main()
