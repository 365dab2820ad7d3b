#!/usr/bin/env python
"""Time ResNeXt-3D's grouped 3x3x3 convolutions on the group-aware kernel (ops.PackedGroupedConv) and on the block-diagonal dense
filter (ops.PackedConv over ops.dense_from_grouped), in the same process on the same card.

    python tools/bench_groupconv.py [--batch 8] [--frames 16] [--size 224] [--reps 20] [--rounds 5] [--e2e-batch 4] [--out FILE]

Layers: the conv2 shapes of resnext3d50 for a [batch, 3, frames, size, size] clip batch -- widths 128 / 256 / 512 / 1024 with 4 / 8 /
16 / 32 channels per group, the stride-2 instance that opens layer2..4 and the stride-1 instance of every stage.  Each route's
``reps`` calls are one CUDA graph; after a warm-up replay of both, the graphs are replayed alternately ``rounds`` times between
CUDA events and the median per-call time is reported, with the algorithmic FLOP/s (2 * positions * K * C/groups * 27 over time), the
executed FLOP/s (the MMA work the route issues: 4x / 2x / 1x / 1x the algorithmic count on the grouped route, groups x on the dense
one) and the packed-filter bytes.  End to end: clips/s of resnext3d50 and resnext3d101 (graph replays, random weights) with each
route; the dense route is forced from here, by placing a dense PackedConv into every conv2's pack cache -- the library and the
engine have no switch.  The card name and power limit are read in the same run.  Prints one JSON line (and writes it to --out).
Needs an H100; there is no CPU fallback."""
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


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [v.strip() for v in out.split(",")]
        return name, power
    except Exception:
        return torch.cuda.get_device_name(0), "unknown"


def conv2_shapes(batch, frames, size):
    """(name, C, channels per group, stride, input T, H, W) of resnext3d50's conv2 layers: the stem halves H and W, the max-pool
    halves T, H and W, every later stage halves all three in its first block's conv2."""
    T, H = (frames - 1) // 2 + 1, ((size - 1) // 2 + 1 - 1) // 2 + 1
    shapes = []
    for stage, C in enumerate((128, 256, 512, 1024)):
        if stage:
            shapes.append(("layer%d.0 s2" % (stage + 1), C, C // 32, 2, T, H, H))
            T, H = (T - 1) // 2 + 1, (H - 1) // 2 + 1
        shapes.append(("layer%d s1" % (stage + 1), C, C // 32, 1, T, H, H))
    return [(n, C, cg, s, batch, t, h, w) for (n, C, cg, s, t, h, w) in shapes]


def graph_of(fn, reps):
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        fn()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            fn()
    return g


def alternate(graphs, rounds):
    """Median time of one replay of each graph, replayed in turn ``rounds`` times after one warm-up replay each."""
    for g in graphs:
        g.replay()
    torch.cuda.synchronize()
    times = [[] for _ in graphs]
    for _ in range(rounds):
        for i, g in enumerate(graphs):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            g.replay()
            e1.record()
            torch.cuda.synchronize()
            times[i].append(e0.elapsed_time(e1))
    return [statistics.median(t) for t in times]


def bench_layer(dev, name, C, cg, stride, N, T, H, W, reps, rounds):
    g = torch.Generator().manual_seed(C + stride)
    w = (torch.randn((C, cg, 3, 3, 3), generator=g) * 0.05).to(dev)
    x = torch.randn((N * T * H * W, C), generator=g).half().to(dev)
    a = ops.Act(x, N, T, H, W, C)
    s, p = (stride,) * 3, (1, 1, 1)
    grouped = ops.PackedGroupedConv(w, 32, stride=s, padding=p)
    dense = ops.PackedConv(ops.dense_from_grouped(w, 32), stride=s, padding=p)
    yg, yd = ops.conv(a, grouped, relu=True), ops.conv(a, dense, relu=True)
    diff = float((yg.data.float() - yd.data.float()).abs().max()) / max(float(yd.data.float().abs().max()), 1e-12)
    out_g, out_d = torch.empty_like(yg.data), torch.empty_like(yd.data)
    graphs = [graph_of(lambda: ops.conv(a, grouped, relu=True, out=out_g), reps),
              graph_of(lambda: ops.conv(a, dense, relu=True, out=out_d), reps)]
    ms_g, ms_d = (t / reps for t in alternate(graphs, rounds))
    flops = 2.0 * yg.M * C * cg * 27
    executed = {4: 4.0, 8: 2.0, 16: 1.0, 32: 1.0}[cg]
    return dict(layer=name, C=C, per_group=cg, stride=stride, input=[N, T, H, W], positions=yg.M, algorithmic_gflop=flops / 1e9,
                max_rel_diff=diff,
                grouped=dict(ms=ms_g, algorithmic_tflops=flops / ms_g / 1e9, executed_tflops=executed * flops / ms_g / 1e9,
                             weight_bytes=grouped.w.numel() * 2),
                dense=dict(ms=ms_d, algorithmic_tflops=flops / ms_d / 1e9, executed_tflops=32.0 * flops / ms_d / 1e9,
                           weight_bytes=dense.w.numel() * 2),
                speedup=ms_d / ms_g)


def conv2_layers(model):
    return [blk.conv2 for ln in ("layer1", "layer2", "layer3", "layer4") for blk in getattr(model, ln)]


def bench_model(dev, arch, x, steps, rounds):
    torch.manual_seed(0)
    model = OF.randomize_bn_(getattr(P, arch)(num_classes=400), 1).eval().to(dev)
    with torch.no_grad():
        ref = model(x).clone()                                  # packs every filter: conv2 on the grouped route
        g_grouped = GraphedForward(model, x)
        keep = [c.__dict__["_b2_cache"]["pc"][1] for c in conv2_layers(model)]      # the captured graph reads these filters
        grouped_bytes = sum(pc.w.numel() * 2 for pc in keep)
        for c in conv2_layers(model):                           # same cache key, dense pack: the dense route
            sig, pc, _ = c.__dict__["_b2_cache"]["pc"]
            assert type(pc) is ops.PackedGroupedConv
            dpc = ops.PackedConv(ops.dense_from_grouped(c.weight.detach(), c.groups), stride=pc.s, padding=pc.p)
            dpc.scale, dpc.shift = pc.scale, pc.shift
            c.__dict__["_b2_cache"]["pc"] = (sig, dpc, None)
        dense_out = model(x)
        g_dense = GraphedForward(model, x)
        dense_bytes = sum(c.__dict__["_b2_cache"]["pc"][1].w.numel() * 2 for c in conv2_layers(model))
    assert all(type(c.__dict__["_b2_cache"]["pc"][1]) is ops.PackedConv for c in conv2_layers(model)) and len(keep) == len(conv2_layers(model))
    diff = float((dense_out - ref).abs().max()) / float(ref.abs().max())

    class Rep:                                                   # `steps` forwards per timed replay
        def __init__(self, g):
            self.g = g

        def replay(self):
            for _ in range(steps):
                self.g()

    ms_g, ms_d = (t / steps for t in alternate([Rep(g_grouped), Rep(g_dense)], rounds))
    B = x.shape[0]
    return dict(arch=arch, input=list(x.shape), logits_max_rel_diff=diff,
                grouped=dict(ms=ms_g, clips_per_s=B / ms_g * 1e3, conv2_weight_bytes=grouped_bytes),
                dense=dict(ms=ms_d, clips_per_s=B / ms_d * 1e3, conv2_weight_bytes=dense_bytes), speedup=ms_d / ms_g)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--size", type=int, default=224)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--e2e-batch", type=int, default=4)
    ap.add_argument("--e2e-steps", type=int, default=5)
    ap.add_argument("--archs", default="resnext3d50,resnext3d101")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_groupconv.py needs an H100: there is no CPU fallback and no timing without a device")
    dev = torch.device("cuda:0")
    name, power = card()
    layers = [bench_layer(dev, *shape, args.reps, args.rounds) for shape in conv2_shapes(args.batch, args.frames, args.size)]
    x = OF.seeded_input((args.e2e_batch, 3, args.frames, args.size, args.size), 2).to(dev)
    models = [bench_model(dev, arch, x, args.e2e_steps, args.rounds) for arch in args.archs.split(",") if arch]
    result = dict(card=name, power_limit=power, batch=args.batch, frames=args.frames, size=args.size, reps=args.reps,
                  rounds=args.rounds, layers=layers, models=models)
    line = json.dumps(result)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
