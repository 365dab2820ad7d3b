"""GPU time of single convolution layers, measured as CUDA-graph replays (no host launch overhead in the number), for several
kernel-selection settings in ONE process.  Each line of the spec file / stdin:  N Cin T H W K kt kh kw st sh sw [res]
usage: conv_sweep.py specfile "maxm:force_s" ["maxm:force_s" ...]"""
import ctypes, os, sys
import torch, torch.nn as nn
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pretorched_x_b200 import ops, engine, _lib

lib = _lib.load()
lib.b2_debug_set_densem.restype = ctypes.c_int
lib.b2_debug_set_densem.argtypes = [ctypes.c_int, ctypes.c_int]
specs = [l.split() for l in open(sys.argv[1]) if l.strip() and not l.startswith("#")]
# a setting is "maxm:force_s" (dense-M path: -1 = default rule, 0 = off) optionally followed by ":mt" (slab M tiles per item, 0 = cost model)
settings = [tuple(int(v) for v in s.split(":")) for s in sys.argv[2:]] or [(0, 0), (1 << 30, 0)]
lib.b2_debug_set_slab_mt.restype = ctypes.c_int
lib.b2_debug_set_slab_mt.argtypes = [ctypes.c_int]
lib.b2_debug_set_slab_wide.restype = ctypes.c_int
lib.b2_debug_set_slab_wide.argtypes = [ctypes.c_int]          # 4th field of a setting: 256-column N tiles 1 = always, 0 = never, -1 / absent = the library's rule
lib.b2_debug_set_tstack.restype = ctypes.c_int
lib.b2_debug_set_tstack.argtypes = [ctypes.c_int]             # 5th field: temporal stack kernel 1 = whenever eligible, 0 = never, -1 / absent = the library's rule
lib.b2_debug_set_slab_t128.restype = ctypes.c_int
lib.b2_debug_set_slab_t128.argtypes = [ctypes.c_int]          # 6th field: 128-wide transposed slab form 1 = wherever it applies, 0 = never, -1 / absent = the rule
lib.b2_debug_set_slab_t64.restype = ctypes.c_int
lib.b2_debug_set_slab_t64.argtypes = [ctypes.c_int]           # 7th field: 64-wide transposed slab form 1 = wherever it applies, 0 = never, -1 / absent = the rule
# 8th field: -1 / absent = the plain entry; 0 = the slice entry (b2_conv_ndhwc_fprop_slice, its own N tile); 1 = the slice entry with the
# N tile exactly K wide (b2_conv_ndhwc_fprop_slice_narrow, K = 32 or 48).  Slice settings run without BatchNorm or ReLU (DenseNet's
# growth-rate convolutions) and report the largest difference from the first slice setting's output (bits: 0 = bitwise equal).
dev = torch.device("cuda:0")
REP = 20
for sp in specs:
    N, Cin, T, H, W, K, kt, kh, kw, st, sh, sw = [int(v) for v in sp[:12]]
    with_res = len(sp) > 12
    torch.manual_seed(0)
    conv = nn.Conv3d(Cin, K, (kt, kh, kw), stride=(st, sh, sw), padding=(kt // 2, kh // 2, kw // 2), bias=False).to(dev)
    bn = nn.BatchNorm3d(K).eval().to(dev)
    with torch.no_grad():
        bn.running_mean.normal_(0, 0.1); bn.running_var.uniform_(0.5, 1.5); bn.weight.uniform_(0.5, 1.5); bn.bias.normal_(0, 0.1)
        x = ops.from_ncdhw(torch.randn(N, Cin, T, H, W, device=dev))
        lib.b2_debug_set_densem(0, 0)
        want = engine.conv_bn_act(conv, bn, x, relu=True, simt=True)
        res = None
        if with_res:
            res = ops.Act(torch.randn_like(want.data.float()).half(), want.N, want.T, want.H, want.W, want.C)
            res.data[:, want.C:] = 0
            want = engine.conv_bn_act(conv, bn, x, residual=res, relu=True, simt=True)
        M = want.data.shape[0]
        fl = 2.0 * M * K * Cin * kt * kh * kw
        out = ["%-44s M=%-7d" % (" ".join(sp[:12]) + (" +res" if with_res else ""), M)]
        ref_slice = None
        for st in settings:
            maxm, fs = st[0], st[1]
            if len(st) > 7 and st[7] >= 0:
                pc = engine.packed_conv(conv, None, x.ld)
                ys = torch.empty((M, K), dtype=torch.float16, device=dev)
                run = lambda: ops.conv_slice(x, pc, ys, relu=False, narrow=st[7] == 1)
                run(); torch.cuda.synchronize()
                if ref_slice is None:
                    ref_slice = ys.clone()
                diff = int((ys.view(torch.int16) != ref_slice.view(torch.int16)).sum())
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    for _ in range(REP):
                        run()
                g.replay(); torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(3):
                    g.replay()
                e1.record(); torch.cuda.synchronize()
                us = e0.elapsed_time(e1) / (3 * REP) * 1e3
                info = (ctypes.c_int * 5)()
                kid = lib.b2_debug_last_kernel(info)
                out.append("[%s] %7.1f us %6.0f TF/s k%d%s bits!=%d" % (":".join(map(str, st)), us, fl / us / 1e6, kid, tuple(info), diff))
                del g
                continue
            mt = st[2] if len(st) > 2 else 0
            lib.b2_debug_set_densem(maxm, fs)
            lib.b2_debug_set_slab_mt(mt)
            lib.b2_debug_set_slab_wide(st[3] if len(st) > 3 else -1)
            lib.b2_debug_set_tstack(st[4] if len(st) > 4 else -1)
            lib.b2_debug_set_slab_t128(st[5] if len(st) > 5 else -1)
            lib.b2_debug_set_slab_t64(st[6] if len(st) > 6 else -1)
            for _ in range(2):
                y = engine.conv_bn_act(conv, bn, x, residual=res, relu=True)
            torch.cuda.synchronize()
            err = (y.data.float() - want.data.float()).abs().max().item() / max(want.data.float().abs().max().item(), 1e-6)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                for _ in range(REP):
                    y = engine.conv_bn_act(conv, bn, x, residual=res, relu=True)
            g.replay(); torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(3):
                g.replay()
            e1.record(); torch.cuda.synchronize()
            us = e0.elapsed_time(e1) / (3 * REP) * 1e3
            info = (ctypes.c_int * 5)()
            kid = lib.b2_debug_last_kernel(info)
            out.append("[%s] %7.1f us %6.0f TF/s k%d%s %s" % (":".join(map(str, st)), us, fl / us / 1e6, kid, tuple(info),
                                                          "" if err < 2e-3 else "ERR %.1e" % err))
            del g
        print("  ".join(out), flush=True)
