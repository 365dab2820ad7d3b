"""The dual-output closing GEMM of PolyNet's poly-3 modules (b2_gemm_dual_f16, pgemm_kernel<BN, 0, 4>).

Kept out of ``ops`` because every launching entry of ``ops`` is held by the whole-forward audit's own tables
(tests/model_audit.py); this module's entries are audited by tests/dual_audit.py, which plugs them into the same auditor, and
tests/test_polynet_cpu.py holds every launching function of this module to that table.  Call sites reach the entry through the
module attribute (``ops_dual.gemm_dual(...)``) so that the audit's patch sees every launch.
"""
import ctypes

import torch

from . import _lib, ops


@ops._on_device
def gemm_dual(a2d, b2d, scale, shift, scale2, shift2, M, N, Kd, residual=None, relu=False, out=None, out2=None):
    """(D, D2) from one accumulator acc = A[M][Kd] . B[N][Kd]^T (b2_gemm_dual_f16): D = act(scale * acc + shift + residual) as
    ``gemm`` writes it, D2 = relu(scale2 * acc + shift2), both fp16 [M][round_up(N, 8)].  The close of one application of a
    PolyNet poly-3 module: D the running sum, D2 the next application's input."""
    dev = a2d.device
    ldd = ops._round_up(N, 8)
    out = torch.empty((M, ldd), dtype=torch.float16, device=dev) if out is None else ops._out_rows(out, M, ldd)
    out2 = torch.empty((M, ldd), dtype=torch.float16, device=dev) if out2 is None else ops._out_rows(out2, M, ldd)
    g = ops.GemmArgs()
    g.a, g.b, g.scale, g.shift = ops._ptr(a2d), ops._ptr(b2d), ops._ptr(scale), ops._ptr(shift)
    g.residual = ops._ptr(residual)
    g.d = ops._ptr(out)
    g.M, g.N, g.Kd = M, N, Kd
    g.lda, g.ldb, g.ldd = a2d.stride(0), b2d.stride(0), ldd
    g.ldr = residual.stride(0) if residual is not None else 0
    g.relu = int(relu)
    with ops._timed("gemm_dual", "gemm dual M=%d N=%d K=%d" % (M, N, Kd), 2.0 * M * N * Kd,
                        2.0 * (M * Kd + N * Kd + 2 * M * ldd + (M * N if residual is not None else 0))):
        _lib.check(_lib.load().b2_gemm_dual_f16(ctypes.byref(g), ops._ptr(scale2), ops._ptr(shift2), ops._ptr(out2), ldd, ops._stream()),
                   "b2_gemm_dual_f16")
    return out, out2
