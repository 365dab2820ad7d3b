"""The whole-forward audit (tests/model_audit.py) extended to the launching entries of ``pretorched_x_b200.ops_pnasnet``: the k x k
ReLU-on-input depthwise pass of PNASNet-5's separable branches and FactorizedReduction's offset gather.

Same scheme as tests/xception_audit.py: ``ENTRIES`` is the table of ``ops_pnasnet``'s entries and the parameters their checks model;
for the duration of one ``audit`` each is wrapped by the model audit's auditor (snapshot, launch count, kernel record, accounting),
with its check bound as ``audit_<name>``; the tables are restored afterwards.  The launch count of the whole forward must still
equal the sum over the wrapped entries.  tests/test_pnasnet_cpu.py requires every launching function of ops_pnasnet.py to be in
``ENTRIES``.

``check_*`` take plain tensors and run on any device.
"""
import contextlib
import types

import torch

from tests import kernel_ref as KR
from tests import model_audit as MA
from tests import pnasnet_kernel_ref as PR

# entry -> the parameters its check models
ENTRIES = {
    "dwconv_kxk_relu_in": ("a", "wk", "k", "stride", "pad", "Ho", "Wo", "out"),
    "gather_offset": ("a", "stride", "offset", "relu"),
}
RECORDS = ("dwconv_kxk_relu_in",)
KID_DWCONV_KXK = 20                # csrc/b2_host.h


def check_dwconv_kxk(x2d, N, H, W, C, wk, k, stride, pad, Ho, Wo, y):
    """Every element of the C columns of ``y`` (rows of any pitch) within the per-element bound of tests/kernel_ref.py.  ``x2d``:
    the input rows (any pitch, first C columns used)."""
    S, So = H * W, Ho * Wo
    wst = MA._Worst()
    for n0, n1 in MA._chunks(N, 8 * 10 * S * C):
        x = x2d[n0 * S:n1 * S, :C].reshape(n1 - n0, H, W, C)
        ref, A = PR.dw_kxk_relu_in_ref(x, wk, k, stride, pad, Ho, Wo, device=y.device)
        wst.add("y", y[n0 * So:n1 * So, :C], ref, KR.bound(ref, A, True), n0 * So)
        del ref, A
    return wst.result()


def check_gather(x2d, N, H, W, stride, offset, relu, y):
    """The gather is a copy: every element exact, the pad columns copied from the (zero) input pad columns."""
    x = x2d.reshape(N, H, W, x2d.shape[1])
    ref = PR.gather_offset_ref(x.clamp(min=0) if relu else x, stride, offset)
    wst = MA._Worst()
    wst.exact("y", y, ref, 0)
    return wst.result()


def _audit_dwconv_kxk_relu_in(aud, b, out):
    a = b["a"]
    k, Ho, Wo = b["k"], b["Ho"], b["Wo"]
    aud.report.ref_flops += 2 * 2.0 * k * k * a.N * Ho * Wo * a.C
    geom = "dwconv_kxk K%d s%d p%d N%d %dx%d->%dx%d C%d" % (k, b["stride"], b["pad"], a.N, a.H, a.W, Ho, Wo, a.C)
    return geom, check_dwconv_kxk(a.data, a.N, a.H, a.W, a.C, b["wk"], k, b["stride"], b["pad"], Ho, Wo, out.data)


def _audit_gather_offset(aud, b, out):
    a = b["a"]
    geom = "gather s%d +%d N%d %dx%d C%d%s" % (b["stride"], b["offset"], a.N, a.H, a.W, a.ld, " relu" if b["relu"] else "")
    return geom, check_gather(a.data, a.N, a.H, a.W, b["stride"], b["offset"], b["relu"], out.data)


CHECKS = {"dwconv_kxk_relu_in": _audit_dwconv_kxk_relu_in, "gather_offset": _audit_gather_offset}


@contextlib.contextmanager
def patched(chain_bitwise=True):
    """tests/model_audit.patched, with the entries of ``ops_pnasnet`` wrapped by the same auditor too; yields the auditor."""
    from pretorched_x_b200 import ops_pnasnet
    saved = {n: getattr(ops_pnasnet, n) for n in ENTRIES}
    known, records = dict(MA.KNOWN), MA.RECORDS_KERNEL
    try:
        MA.KNOWN.update(ENTRIES)
        MA.RECORDS_KERNEL = records + RECORDS
        with MA.patched(chain_bitwise) as aud:
            for n in ENTRIES:
                setattr(aud, "audit_" + n, types.MethodType(CHECKS[n], aud))
                setattr(ops_pnasnet, n, aud.wrap(n, saved[n]))
            try:
                yield aud
            finally:
                for n, f in saved.items():
                    setattr(ops_pnasnet, n, f)
    finally:
        MA.KNOWN.clear()
        MA.KNOWN.update(known)
        MA.RECORDS_KERNEL = records


def audit(model_fn, chain_bitwise=True):
    """tests/model_audit.audit over the launching entries of ``ops`` and ``ops_pnasnet``."""
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
