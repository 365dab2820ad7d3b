"""Probe wgmma smem-descriptor semantics on the GPU (see csrc/b2_probe.cu).  Prints which variants are exact."""
import ctypes
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from pretorched_x_b200 import _lib  # noqa: E402

lib = _lib.load()
fn = lib.b2_debug_umma_probe
fn.restype = ctypes.c_int
fn.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
dev = torch.device("cuda:0")
g = torch.Generator().manual_seed(0)


def run(a, b, mode, shift, base_off):
    shape = (64, base_off) if mode == 3 else (64, 112) if mode == 4 else (128, 128 if mode == 2 else 64)
    out = torch.full(shape, float("nan"), dtype=torch.float32, device=dev)
    rc = fn(a.data_ptr(), b.data_ptr(), out.data_ptr(), mode, shift, base_off, None)
    assert rc == 0, _lib.last_error()
    torch.cuda.synchronize()
    return out.cpu()


A = torch.randn(256, 64, generator=g).half()
B = (torch.randn(64, 64, generator=g) / 8).half()
Ad, Bd = A.to(dev), B.to(dev)
print("mode 0: SW128 K-major A with start address shifted by s rows (128 B each)")
for s in range(0, 9):
    want = A[s:s + 128].float() @ B.float().t()
    for bo in sorted({0, s % 8}):
        got = run(Ad, Bd, 0, s, bo)
        err = (got - want).abs().max().item() / want.abs().max().item()
        print("  shift %d base_offset %d: rel err %.3e %s" % (s, bo, err, "EXACT" if err < 1e-5 else "wrong"))

buf = torch.randn(2048, generator=g).half()
B1 = (torch.randn(64, 32, generator=g) / 6).half()
idx = (torch.arange(128).view(-1, 1) * 8 + torch.arange(32).view(1, -1))
want = buf.float()[idx] @ B1.float().t()
got = run(buf.to(dev), B1.to(dev), 1, 0, 0)
err = (got - want).abs().max().item() / want.abs().max().item()
print("mode 1: no-swizzle Toeplitz A (LBO=16, SBO=128): rel err %.3e %s" % (err, "EXACT" if err < 1e-5 else "wrong"))

want = B1.float() @ buf.float()[idx[:112]].t()
got = run(buf.to(dev), B1.to(dev), 4, 0, 0)
err4 = (got - want).abs().max().item() / want.abs().max().item()
print("mode 4: no-swizzle Toeplitz B at N = 112 (LBO=16, SBO=128), A = 64 x 32 no-swizzle: rel err %.3e %s"
      % (err4, "EXACT" if err4 < 1e-5 else "wrong"))

A2 = torch.randn(128, 64, generator=g).half()
V2 = (torch.randn(64, 128, generator=g) / 8).half()
want = A2.float() @ V2.float()
got = run(A2.to(dev), V2.to(dev), 2, 0, 0)
err = (got - want).abs().max().item() / want.abs().max().item()
print("mode 2: MN-major SW128 B (LBO=8192, SBO=1024, K step 2048 B): rel err %.3e %s" % (err, "EXACT" if err < 1e-5 else "wrong"))

print("mode 3: SW128 K-major B (N rows) with start address shifted by s rows (128 B each), A = 64 x 64 K-major tile")
bad = 0
for n in (64, 128, 192):
    for s in (0, 1, 3, 5, 7, 8, 9, 13, 37, 256 - n):
        want = B.float() @ A[s:s + n].float().t()
        got = run(Ad, Bd, 3, s, n)
        err = ((got - want).abs().max() / want.abs().max()).item()
        ok = err < 1e-5
        bad += not ok
        print("  N %3d shift %3d: rel err %.3e %s" % (n, s, err, "EXACT" if ok else "wrong"))
print("mode 3: %s" % ("all EXACT" if bad == 0 else "%d WRONG" % bad))
bad += err4 >= 1e-5
sys.exit(1 if bad else 0)
