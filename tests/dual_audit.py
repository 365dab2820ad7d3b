"""The whole-forward audit (tests/model_audit.py) extended to the launching entries of ``pretorched_x_b200.ops_dual``: the
dual-output closing GEMM of PolyNet's poly-3 modules.

tests/model_audit.py wraps the launching entries of ``ops`` from its own tables.  ``ENTRIES`` below is the same kind of table for
``ops_dual``: for the duration of one ``audit``, each of its entries is wrapped by the same auditor (same snapshot, launch count,
kernel record and accounting), with its parameters registered in the auditor's ``KNOWN`` / ``RECORDS_KERNEL`` tables and its
check bound as ``audit_<name>``; the tables are restored afterwards.  The launch count of the whole forward must still equal the
sum over the wrapped entries of both modules, so a launch of ``ops_dual`` that this table missed fails the audit.
tests/test_polynet_cpu.py requires every launching function of ops_dual.py to be in ``ENTRIES``.

``check_gemm_dual`` takes plain tensors and runs on any device, like the ``check_*`` functions of tests/model_audit.py.
"""
import contextlib
import types

import torch

from tests import kernel_ref as KR
from tests import model_audit as MA

# entry -> the parameters its check models
ENTRIES = {
    "gemm_dual": ("a2d", "b2d", "scale", "shift", "scale2", "shift2", "M", "N", "Kd", "residual", "relu", "out", "out2"),
}


def check_gemm_dual(a, b, scale, shift, scale2, shift2, M, N, Kd, d, d2, residual=None, relu=False, pad=True):
    """b2_gemm_dual_f16: D = act(scale * acc + shift + residual), held as tests/model_audit.check_gemm holds it, and
    D2 = relu(scale2 * acc + shift2) from the same accumulator acc = A[:, :Kd] . B[:N, :Kd]^T, each to its own per-element bound.
    ``pad``: columns [N, ldd) of both outputs must be zero."""
    dev = d.device
    chunk = MA._samples_per_chunk(8 * (2 * Kd + 10 * N))
    wst = MA._Worst()
    for m0 in range(0, M, chunk):
        m1 = min(M, m0 + chunk)
        acc, mag = KR.gemm_acc(a[m0:m1, :Kd], b[:N, :Kd], device=dev)
        res = residual[m0:m1, :N].double() if residual is not None else None
        v, A = KR.epilogue(acc, mag, scale[:N].double(), shift[:N].double(), res, relu=relu, device=dev)
        wst.add("d", d[m0:m1, :N], v, KR.bound(v, A, True), m0)
        del v, A, res
        v2, A2 = KR.epilogue(acc, mag, scale2[:N].double(), shift2[:N].double(), None, relu=True, device=dev)
        wst.add("d2", d2[m0:m1, :N], v2, KR.bound(v2, A2, True), m0)
        if pad:
            MA._pad_zero(wst, "d", d[m0:m1], N, m0)
            MA._pad_zero(wst, "d2", d2[m0:m1], N, m0)
        del acc, mag, v2, A2
    return wst.result()


def _audit_gemm_dual(aud, b, out):
    d, d2 = out
    aud.report.ref_flops += 2 * 2.0 * b["M"] * b["N"] * b["Kd"]
    geom = "gemm_dual M%d N%d K%d%s%s" % (b["M"], b["N"], b["Kd"], " res" if b["residual"] is not None else "",
                                         " relu" if b["relu"] else "")
    return geom, check_gemm_dual(b["a2d"], b["b2d"], b["scale"], b["shift"], b["scale2"], b["shift2"], b["M"], b["N"], b["Kd"], d,
                                 d2, residual=b["residual"], relu=b["relu"], pad=b["out"] is None and b["out2"] is None)


CHECKS = {"gemm_dual": _audit_gemm_dual}


@contextlib.contextmanager
def patched(chain_bitwise=True):
    """tests/model_audit.patched, with the entries of ``ops_dual`` wrapped by the same auditor; yields the auditor."""
    from pretorched_x_b200 import ops_dual
    known, records = dict(MA.KNOWN), MA.RECORDS_KERNEL
    saved = {n: getattr(ops_dual, n) for n in ENTRIES}
    try:
        MA.KNOWN.update(ENTRIES)
        MA.RECORDS_KERNEL = records + tuple(ENTRIES)
        with MA.patched(chain_bitwise) as aud:
            for n in ENTRIES:
                setattr(aud, "audit_" + n, types.MethodType(CHECKS[n], aud))
                setattr(ops_dual, n, aud.wrap(n, saved[n]))
            try:
                yield aud
            finally:
                for n, f in saved.items():
                    setattr(ops_dual, n, f)
    finally:
        MA.KNOWN.clear()
        MA.KNOWN.update(known)
        MA.RECORDS_KERNEL = records


def audit(model_fn, chain_bitwise=True):
    """tests/model_audit.audit over the launching entries of ``ops`` and ``ops_dual``."""
    with torch.no_grad(), patched(chain_bitwise) as aud:
        torch.cuda.synchronize()
        c0 = aud.lib.b2_launch_count()
        out = model_fn()
        torch.cuda.synchronize()
        rep = aud.report
        rep.launches = aud.lib.b2_launch_count() - c0 - aud.extra
        rep.output = out
    if rep.launches != rep.counted:
        raise MA.AuditError("the forward made %d library launches, the wrapped entries account for %d" % (rep.launches, rep.counted))
    return rep
