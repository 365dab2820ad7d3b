"""The whole-forward audit (tests/model_audit.py) extended to the launching entry of ``pretorched_x_b200.ops_xception``: the
depthwise pass of Xception's separable convolutions, which reads ReLU(x) and applies no affine.

Same scheme as tests/vgg_audit.py: ``ENTRIES`` is the table of ``ops_xception``'s entries and the parameters their checks model;
for the duration of one ``audit`` each is wrapped by the model audit's auditor (snapshot, launch count, kernel record, accounting),
with its check bound as ``audit_<name>``; the tables are restored afterwards.  The launch count of the whole forward must still
equal the sum over the wrapped entries.  tests/test_xception_cpu.py requires every launching function of ops_xception.py to be in
``ENTRIES``.

``check_*`` take plain tensors and run on any device.
"""
import contextlib
import types

import torch

from tests import kernel_ref as KR
from tests import model_audit as MA

# entry -> the parameters its check models
ENTRIES = {
    "dwconv3x3_relu_in": ("a", "w9", "out"),
}
RECORDS = ("dwconv3x3_relu_in",)
KID_DWCONV_RELU_IN = 19            # csrc/b2_host.h


def dw_relu_in_ref(x, w9, device="cpu"):
    """fp64 reference of b2_dwconv3x3_relu_in_ndhwc from its fp16 input x [B, H, W, C] (the C used channels) and fp32 taps w9 [9][C]:
    the depthwise 3x3 (stride 1, padding 1) of max(x, 0) (exact in fp16), no affine.  Returns (ref, A), fp64 [B * H * W, C]."""
    C = x.shape[-1]
    one = torch.ones(C, dtype=torch.float64)
    zero = torch.zeros(C, dtype=torch.float64)
    return KR.dw_ref(x.double().clamp(min=0.0), w9, one, zero, 1, False, False, device=device)


def check_dwconv_relu_in(x2d, N, H, W, C, w9, y):
    """Every used element within the per-element bound of tests/kernel_ref.py; padding channels [C, ld) zero."""
    S = H * W
    wst = MA._Worst()
    for n0, n1 in MA._chunks(N, 8 * 10 * S * C):
        ref, A = dw_relu_in_ref(x2d[n0 * S:n1 * S, :C].reshape(n1 - n0, H, W, C), w9, device=y.device)
        wst.add("y", y[n0 * S:n1 * S, :C], ref, KR.bound(ref, A, True), n0 * S)
        MA._pad_zero(wst, "y", y[n0 * S:n1 * S], C, n0 * S)
        del ref, A
    return wst.result()


def _audit_dwconv3x3_relu_in(aud, b, out):
    a = b["a"]
    aud.report.ref_flops += 2 * 18.0 * a.M * a.C
    geom = "dwconv_relu_in N%d %dx%d C%d" % (a.N, a.H, a.W, a.C)
    return geom, check_dwconv_relu_in(a.data, a.N, a.H, a.W, a.C, b["w9"], out.data)


CHECKS = {"dwconv3x3_relu_in": _audit_dwconv3x3_relu_in}


@contextlib.contextmanager
def patched(chain_bitwise=True):
    """tests/model_audit.patched, with the entries of ``ops_xception`` wrapped by the same auditor too; yields the auditor."""
    from pretorched_x_b200 import ops_xception
    saved = {n: getattr(ops_xception, n) for n in ENTRIES}
    known, records = dict(MA.KNOWN), MA.RECORDS_KERNEL
    try:
        MA.KNOWN.update(ENTRIES)
        MA.RECORDS_KERNEL = records + RECORDS
        with MA.patched(chain_bitwise) as aud:
            for n in ENTRIES:
                setattr(aud, "audit_" + n, types.MethodType(CHECKS[n], aud))
                setattr(ops_xception, n, aud.wrap(n, saved[n]))
            try:
                yield aud
            finally:
                for n, f in saved.items():
                    setattr(ops_xception, n, f)
    finally:
        MA.KNOWN.clear()
        MA.KNOWN.update(known)
        MA.RECORDS_KERNEL = records


def audit(model_fn, chain_bitwise=True):
    """tests/model_audit.audit over the launching entries of ``ops`` and ``ops_xception``."""
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
