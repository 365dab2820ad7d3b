"""The whole-forward audit (tests/model_audit.py) extended to the launching entries of ``pretorched_x_b200.ops_vgg``: AlexNet's
space-to-depth stem input and the split-K classifier GEMM.

Same scheme as tests/dual_audit.py: ``ENTRIES`` is the table of ``ops_vgg``'s entries and the parameters their checks model; for
the duration of one ``audit`` each is wrapped by the model audit's auditor (snapshot, launch count, kernel record, accounting), with
its check bound as ``audit_<name>``; the tables are restored afterwards.  The launch count of the whole forward must still equal
the sum over the wrapped entries of all three modules.  tests/test_vgg_cpu.py requires every launching function of ops_vgg.py to be
in ``ENTRIES``.

``check_*`` take plain tensors and run on any device.
"""
import contextlib
import types

import torch

from tests import dual_audit as DA
from tests import kernel_ref as KR
from tests import model_audit as MA

# entry -> the parameters its check models
ENTRIES = {
    "space_to_depth4": ("x",),
    "gemm_splitk": ("a2d", "b2d", "scale", "shift", "M", "N", "Kd", "splits", "relu", "out_f32"),
}
RECORDS = ("gemm_splitk",)


def s2d_ref(x):
    """fp16 [N*Hs*Ws][48] space-to-depth image of fp32 images x [N][3][H][W], built with torch (b2_space_to_depth4_nchw's contract)."""
    N, C, H, W = x.shape
    Ho, Wo = (H + 4 - 11) // 4 + 1, (W + 4 - 11) // 4 + 1
    Hs, Ws = Ho + 2, Wo + 2
    xp = x.new_zeros((N, C, 4 * Hs, 4 * Ws))
    h1, w1 = min(H, 4 * Hs - 2), min(W, 4 * Ws - 2)
    xp[:, :, 2:2 + h1, 2:2 + w1] = x[:, :, :h1, :w1]
    return xp.reshape(N, C, Hs, 4, Ws, 4).permute(0, 2, 4, 3, 5, 1).reshape(N * Hs * Ws, 16 * C).half()


def check_space_to_depth4(x, y):
    """Bit-exact against ``s2d_ref``: one rounding of each input value, zeros outside the image."""
    wst = MA._Worst()
    want = s2d_ref(x.float())
    if tuple(y.shape) != tuple(want.shape):
        return float("inf"), "shape %s, want %s" % (tuple(y.shape), tuple(want.shape))
    wst.ratio, wst.where = 0.0, "bit-exact"
    wst.exact("space_to_depth4", y, want)
    return wst.result()


def check_gemm_splitk(a, b, scale, shift, M, N, Kd, d, relu=False, out_f32=False):
    """b2_gemm_splitk_f16: D = act(scale * A[:, :Kd] . B[:N, :Kd]^T + shift) held to the per-element bound of tests/kernel_ref.py (the
    split partial sums are fp32 accumulations of the same terms, summed in fp32); fp16 pad columns [N, ldd) must be zero."""
    dev = d.device
    chunk = MA._samples_per_chunk(8 * (2 * Kd + 6 * N))
    wst = MA._Worst()
    for m0 in range(0, M, chunk):
        m1 = min(M, m0 + chunk)
        acc, mag = KR.gemm_acc(a[m0:m1, :Kd], b[:N, :Kd], device=dev)
        v, A = KR.epilogue(acc, mag, scale[:N].double(), shift[:N].double(), None, relu=relu, device=dev)
        wst.add("d", d[m0:m1, :N], v, KR.bound(v, A, not out_f32), m0)
        if not out_f32:
            MA._pad_zero(wst, "d", d[m0:m1], N, m0)
        del acc, mag, v, A
    return wst.result()


def _audit_space_to_depth4(aud, b, out):
    x = b["x"]
    aud.report.ref_flops += 0.0
    return "space_to_depth4 N%d %dx%d" % (x.shape[0], x.shape[2], x.shape[3]), check_space_to_depth4(x, out.data)


def _audit_gemm_splitk(aud, b, out):
    aud.report.ref_flops += 2 * 2.0 * b["M"] * b["N"] * b["Kd"]
    geom = "gemm_splitk M%d N%d K%d S%d%s%s" % (b["M"], b["N"], b["Kd"], b["splits"], " relu" if b["relu"] else "",
                                                " f32" if b["out_f32"] else "")
    return geom, check_gemm_splitk(b["a2d"], b["b2d"], b["scale"], b["shift"], b["M"], b["N"], b["Kd"], out, relu=b["relu"],
                                   out_f32=b["out_f32"])


CHECKS = {"space_to_depth4": _audit_space_to_depth4, "gemm_splitk": _audit_gemm_splitk}


@contextlib.contextmanager
def patched(chain_bitwise=True):
    """tests/dual_audit.patched, with the entries of ``ops_vgg`` wrapped by the same auditor too; yields the auditor."""
    from pretorched_x_b200 import ops_vgg
    saved = {n: getattr(ops_vgg, n) for n in ENTRIES}
    with DA.patched(chain_bitwise) as aud:
        known, records = dict(MA.KNOWN), MA.RECORDS_KERNEL
        try:
            MA.KNOWN.update(ENTRIES)
            MA.RECORDS_KERNEL = records + RECORDS
            for n in ENTRIES:
                setattr(aud, "audit_" + n, types.MethodType(CHECKS[n], aud))
                setattr(ops_vgg, n, aud.wrap(n, saved[n]))
            yield aud
        finally:
            for n, f in saved.items():
                setattr(ops_vgg, n, f)
            MA.KNOWN.clear()
            MA.KNOWN.update(known)
            MA.RECORDS_KERNEL = records


def audit(model_fn, chain_bitwise=True):
    """tests/model_audit.audit over the launching entries of ``ops``, ``ops_dual`` and ``ops_vgg``."""
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
