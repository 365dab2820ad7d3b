"""Whole-forward audit: every library launch of one model forward, at the batch it runs at, held element by element to the fp64
bound of tests/kernel_ref.py.

``audit(model_fn)`` patches the launching entries of ``pretorched_x_b200.ops`` for the duration of one call of ``model_fn``.  Every
engine call site goes through the module attribute (``ops.conv(...)``), so the patch reaches every launch.  For each call the
wrapper snapshots any operand whose storage the call may overwrite, calls the original, synchronises, records the library launch
count and the kernel the dispatcher chose (``b2_debug_last_kernel``), and checks the output against an fp64 reference built on the
GPU from exactly the operands the kernel read.  Nothing is skipped silently:

  * the launch-count delta of the whole forward must equal the sum of the deltas of the wrapped entries;
  * an entry without a check (``UNAUDITED`` lists the layout helpers and why), or an argument combination the checks below do not
    understand, raises ``AuditError``;
  * an entry that writes column slices of a wider matrix leaves every other column of those rows bit for bit as it was
    (``SliceGuard``), and the pre-activated GEMM's output depends on nothing of A, B or its input affine past Kd
    (``preact_contract``);
  * the composite entries (``PASS_THROUGH``) launch nothing themselves: the inner entry they call is audited, once.

Filters: ordinary packs are read back from ``pc.w`` as [K][taps][C] (as tests/test_gpu_kernel_matrix.py's ``Problem`` does); the
upsampling pack is read back as the [K][16][C] phase bank and itself checked against ``upconv_fold`` of its source weight; the stem
and grouped packs cannot be read back, so the PackedConv / PackedGroupedConv constructors are wrapped to record the source weight
(``stem_operands`` / ``dense_from_grouped``).  An audit therefore runs on a freshly built model, before anything is packed.

The ``check_*`` functions take plain tensors and run on any device (tests/test_model_audit_cpu.py runs them on the CPU).  Each
returns ``(worst err / bound, where)`` over all elements.  The references are built in chunks of samples (or rows) whose estimated
fp64 working set stays under ``CAP_BYTES``; the estimate does not count cuDNN's workspace for the fp64 convolutions or the
snapshot clones, and the embedding check (a [B][D] matrix) is not chunked.
"""
import contextlib
import ctypes
import functools
import inspect

import torch
import torch.nn.functional as F

from tests import kernel_ref as KR

CAP_BYTES = 4 << 30        # estimated extra device memory of one reference chunk (the GPU machines are shared)

# b2_debug_last_kernel ids (KID_* of csrc/b2_host.h)
KIND = {0: "none", 1: "stem", 2: "slab", 4: "tstack", 5: "densem", 6: "pgemm", 7: "igemm", 8: "simt", 9: "attention",
        10: "groupconv", 11: "pgemm_chain", 12: "pgemm_split", 13: "slab_slice", 14: "pool", 15: "slab_t128", 16: "slab_t64"}

UNAUDITED = {
    "from_ncdhw": "layout: fp32 / fp16 NCDHW -> fp16 NDHWC; its one rounding is the input every reference starts from",
    "to_ncdhw": "layout: fp16 NDHWC -> fp32 NCDHW, an exact widening of values the audit has already checked",
    "cast_rows": "fp32 -> fp16 cast of torch-computed rows (TRN's relation MLP input)",
    "gather_frames": "index gather of fp16 rows (TRN)",
    "gather_frame_tuples": "index gather of fp16 rows (TRN)",
    "conv_wgrad": "fine-tuning backward, held by tests/test_gpu_finetune_bounds.py",
    "zero_insert": "fine-tuning backward, held by tests/test_gpu_finetune_bounds.py",
    "colsum": "fine-tuning backward, held by tests/test_gpu_finetune_bounds.py",
    "loss_scale_": "fine-tuning backward, held by tests/test_gpu_finetune_bounds.py",
    "avgpool_global_backward": "fine-tuning backward, held by tests/test_gpu_finetune_bounds.py",
}
# composite entries: they launch only through the named entry, which is audited
PASS_THROUGH = {"linear": "gemm", "nonlocal_attention": "attention", "concat_channels": "concat_rows"}


# the parameters each audited entry's check models: a parameter an entry gains later fails the audit until its check learns it
KNOWN = {
    "conv": ("a", "pc", "residual", "relu", "simt", "sample_affine", "residual_up", "residual_pre", "next_affine", "pool_w",
             "in_affine", "out", "mask"),
    "gemm": ("a2d", "b2d", "scale", "shift", "M", "N", "Kd", "residual", "relu", "per_row", "out", "out_f32", "accumulate",
             "second", "aff_rows", "next_affine", "mask"),
    "gemm_chain": ("a2d", "b2d", "scale", "shift", "M", "N", "Kd", "w1", "scale1", "shift1", "n1", "residual", "relu", "second",
                   "out"),
    "gemm_sample_affine": ("a2d", "b2d", "scale", "shift", "M", "N", "Kd", "aff_rows", "residual", "relu", "out"),
    "attention": ("q2d", "k2d", "v2d", "d", "dv", "B", "Nq", "Nk", "dot_product", "mode"),
    "maxpool3d": ("a", "kernel", "stride", "padding", "out"),
    "maxpool2d_ceil": ("a", "k", "s", "p", "out"),
    "avgpool_global": ("a",),
    "shortcut_a": ("a", "stride", "out_channels"),
    "concat_rows": ("a2d", "Ca", "b2d", "Cb"),
    "relu6_": ("a",),
    "dwconv3x3": ("a", "w9", "scale", "shift", "stride", "clamp_in", "relu6", "out"),
    "ccbn_act": ("a", "scale", "shift", "channels", "up", "relu"),
    "embed_concat": ("z", "labels", "table", "split"),
    "rgb_head": ("partial", "bias", "N", "H", "W", "K", "out_dtype", "out"),
    "tanh_to_nchw": ("a", "out_dtype", "out"),
    "conv_slice": ("a", "pc", "y", "relu", "narrow"),
    "gemm_split": ("a2d", "b2d", "scale", "shift", "M", "Kd", "dests", "relu"),
    "pool_slice": ("a", "k", "s", "p", "avg", "y", "count_include_pad", "ceil_mode"),
    "gemm_preact": ("a2d", "b2d", "scale", "shift", "in_scale", "in_shift", "M", "N", "Kd", "relu"),
    "bn_relu_avgpool2": ("a", "scale", "shift", "y"),
    "avgpool_global_affine": ("a", "scale", "shift"),
    "se_excite": ("h", "w1", "b1", "w2", "b2", "s3", "t3", "out"),
}
# entries whose launch records the kernel and plan it ran (b2_debug_last_kernel)
RECORDS_KERNEL = ("conv", "gemm", "gemm_chain", "gemm_sample_affine", "attention", "conv_slice", "gemm_split", "gemm_preact",
                  "pool_slice", "bn_relu_avgpool2", "avgpool_global_affine")


class AuditError(AssertionError):
    pass


def _samples_per_chunk(per_sample_bytes):
    return max(1, int(CAP_BYTES // max(1, per_sample_bytes)))


def _ratio(got, ref, bnd):
    """(max |got - ref| / bnd, index of the worst element) on the tensors' device; non-finite ``got`` counts as infinite."""
    err = (got.double() - ref).abs()
    err = torch.where(torch.isfinite(err), err, torch.full_like(err, float("inf")))
    r = (err / bnd).reshape(-1)
    i = int(torch.argmax(r))
    return float(r[i]), i


class _Worst:
    """Running maximum of err / bound over chunks, with the element that reached it."""

    def __init__(self):
        self.ratio, self.where = 0.0, "no elements"

    def add(self, what, got, ref, bnd, row0=0):
        r, i = _ratio(got, ref, bnd)
        r = r if r == r else float("inf")
        if r > self.ratio or self.where == "no elements":
            cols = ref.shape[-1] if ref.dim() > 1 else 1
            m, c = divmod(i, cols)
            self.ratio = r
            self.where = "%s row %d col %d: got %r ref %r bound %r" % (what, row0 + m, c, float(got.reshape(-1)[i]),
                                                                     float(ref.reshape(-1)[i]), float(bnd.reshape(-1)[i]))

    def exact(self, what, got, want, row0=0):
        """Bit-exact comparison (an exact reference): any difference is an infinite ratio."""
        diff = got.double() != want.double()
        if bool(diff.any()):
            i = int(torch.nonzero(diff.reshape(-1))[0])
            cols = want.shape[-1] if want.dim() > 1 else 1
            m, c = divmod(i, cols)
            self.ratio = float("inf")
            self.where = "%s row %d col %d: got %r want %r (bit-exact)" % (what, row0 + m, c, float(got.reshape(-1)[i]),
                                                                           float(want.reshape(-1)[i]))

    def merge(self, what, ratio, where):
        """Fold in the (ratio, where) of a sub-check; NaN counts as infinite."""
        if not ratio <= self.ratio or self.where == "no elements":
            self.ratio, self.where = ratio if ratio == ratio else float("inf"), "%s: %s" % (what, where)

    def result(self):
        return self.ratio, self.where


def _pad_zero(w, what, y, K, row0=0):
    """Columns [K, ld) of an fp16 output are written as zero."""
    if y.shape[-1] > K:
        w.exact(what + " pad columns", y[:, K:], torch.zeros_like(y[:, K:]), row0)


def _rows(v, r0, r1, rows, K):
    """Per-sample rows [N][>= K] -> the [r1 - r0][K] rows of output rows [r0, r1) (row m takes sample m // rows); [K] stays."""
    if v.dim() == 1:
        return v[:K].double()
    idx = torch.arange(r0, r1, device=v.device) // rows
    return v[:, :K].double().index_select(0, idx)


# ---------------------------------------------------------------------------------------------
# convolution (ops.conv, every epilogue)
# ---------------------------------------------------------------------------------------------
def check_conv(x, w, scale, shift, k, s, p, y, K, residual=None, relu=False, sample_affine=None, residual_up=False,
               residual_pre=False, next_affine=None, y2=None, pool_w=False, in_affine=None, upsample=False, mask=None):
    """x fp16 [N, T, H, W, C] (the pitch C), w the filter the kernel multiplies ([K, taps, C]; [K, 16, C] phase bank with
    ``upsample``), scale / shift fp32 [K] or, with ``sample_affine``, per-sample [N][>= K]; y the fp16 output rows [M][ldy]."""
    dev = y.device
    N, T, H, W, C = x.shape
    kt, kh, kw = k
    To, Ho, Wo = ((T + 2 * p[0] - kt) // s[0] + 1, (H + 2 * p[1] - kh) // s[1] + 1, (W + 2 * p[2] - kw) // s[2] + 1)
    if upsample:
        Ho, Wo = 2 * Ho, 2 * Wo
    S = To * Ho * Wo                                   # conv output rows per sample (before the W pool)
    Wp = (Wo - 1) // 2 + 1 if pool_w else Wo
    Sy = To * Ho * Wp                                  # stored rows per sample
    if y.shape[0] != N * Sy:
        raise AuditError("conv output has %d rows, the geometry gives %d" % (y.shape[0], N * Sy))
    if pool_w and (not relu or residual is not None or sample_affine is not None or y2 is not None):
        raise AuditError("pool_w with an epilogue the audit does not model")
    if mask is not None and relu:
        raise AuditError("mask with relu")
    per = 8 * (2 * T * H * W * C + 8 * S * K) + (8 * 9 * S * C if in_affine is not None else 0)
    n_chunk = _samples_per_chunk(per)
    wst = _Worst()
    for n0 in range(0, N, n_chunk):
        n1 = min(N, n0 + n_chunk)
        xc = x[n0:n1]
        if in_affine is not None:
            if k != (1, 1, 1) or s != (1, 1, 1) or upsample:
                raise AuditError("input affine on a convolution that is not 1x1x1 stride 1")
            acc, mag = KR.in_affine_acc(xc.reshape(-1, C), w.reshape(K, C), in_affine[0][n0:n1], in_affine[1][n0:n1], T * H * W,
                                        device=dev)
        elif upsample:
            acc, mag = KR.upconv_acc(xc, w, device=dev)
        else:
            acc, mag = KR.conv_acc(xc, w, k, s, p, device=dev)
        r0, r1 = n0 * S, n1 * S
        if sample_affine is not None:
            sc, sh = _rows(sample_affine[0], r0, r1, S, K), _rows(sample_affine[1], r0, r1, S, K)
        else:
            sc, sh = scale[:K].double(), shift[:K].double()
        res = None
        if residual is not None:
            if residual_up:
                res = KR.nearest_up2(residual[n0 * S // 4:n1 * S // 4], n1 - n0, Ho, Wo, K, device=dev)
            else:
                res = residual[r0:r1, :K].double()
        v, A = KR.epilogue(acc, mag, sc, sh, res, pre=residual_pre, relu=relu, device=dev)
        del acc, mag
        yc = y[n0 * Sy:n1 * Sy]
        if pool_w:
            ref, bnd = KR.pool_w(v, A, Wo)
            wst.add("y", yc[:, :K], ref, bnd, n0 * Sy)
        else:
            ref = v if mask is None else torch.where(mask[r0:r1, :K] > 0, v, torch.zeros_like(v))
            wst.add("y", yc[:, :K], ref, KR.bound(v, A, True), r0)
        _pad_zero(wst, "y", yc, K, n0 * Sy)
        if y2 is not None:
            ref2, A2 = KR.second_output(v, A, _rows(next_affine[0], r0, r1, S, K), _rows(next_affine[1], r0, r1, S, K), device=dev)
            wst.add("y2", y2[r0:r1, :K], ref2, KR.bound(ref2, A2, True), r0)
            _pad_zero(wst, "y2", y2[r0:r1], K, r0)
        del v, A
    return wst.result()


def stem_filter(weight):
    """The stem pack's operand: the source weight rounded to fp16, as the [K, taps, 4] layout ``conv_ref`` reads."""
    if weight.dim() == 4:
        weight = weight.unsqueeze(2)
    K, Cin = weight.shape[:2]
    x = torch.zeros((1, Cin, 1, 1, 1), dtype=torch.float16)
    return KR.stem_operands(x, weight)[1]


def grouped_filter(weight, groups, C):
    """The grouped pack's operand: the block-diagonal dense filter of the fp16-rounded weight, [K, taps, C]."""
    from pretorched_x_b200 import ops
    if weight.dim() == 4:
        weight = weight.unsqueeze(2)
    dense = ops.dense_from_grouped(weight.detach().half(), groups)
    K = dense.shape[0]
    return dense.permute(0, 2, 3, 4, 1).reshape(K, -1, C)


def check_upconv_pack(wph, weight):
    """The upsampling pack [K, 16, C] against the fp64 fold of its 3x3 source weight: one fp32 sum of at most four weights and
    one fp16 rounding per folded tap (bound 2^-11 |fold| + 4 2^-24 sum |w| + 2^-25)."""
    if weight.dim() == 5:
        weight = weight[:, :, 0]
    fold, mag = KR.upconv_fold(weight)
    Cin = weight.shape[1]
    got = wph[:, :, :Cin].double().cpu()
    wst = _Worst()
    wst.add("phase filter", got.reshape(got.shape[0], -1), fold.reshape(fold.shape[0], -1),
            (KR.U_F16 * fold.abs() + 4 * KR.FLOOR * mag + 2.0 ** -25).reshape(fold.shape[0], -1))
    if wph.shape[2] > Cin:
        wst.exact("phase filter pad", wph[:, :, Cin:].reshape(wph.shape[0], -1), torch.zeros_like(wph[:, :, Cin:]).reshape(wph.shape[0], -1))
    return wst.result()


# ---------------------------------------------------------------------------------------------
# GEMMs
# ---------------------------------------------------------------------------------------------
def check_gemm(a, b, scale, shift, M, N, Kd, d, residual=None, relu=False, per_row=False, out_f32=False, base=None, second=None,
               aff_rows=0, next_affine=None, d2=None, mask=None, pad=False):
    """D[M][N] = act(scale * (A[:, :Kd] . B[:N, :Kd]^T [+ A2 . B2^T]) + shift + residual) (+ base when accumulating into fp32).
    scale / shift: [N]; [M] with ``per_row``; per-sample [M / aff_rows][>= N] with ``aff_rows``.  ``pad``: columns [N, ldd) of the
    fp16 outputs must be zero (an output the entry allocated, round_up(N, 8) wide)."""
    dev = d.device
    rows = aff_rows if aff_rows else 1
    k2 = second[2] if second is not None else 0
    per = 8 * (2 * (Kd + k2) + 8 * N)
    chunk = max(rows, _samples_per_chunk(per * rows) * rows)
    if next_affine is not None and d2 is None:
        raise AuditError("next_affine without its second output")
    wst = _Worst()
    for m0 in range(0, M, chunk):
        m1 = min(M, m0 + chunk)
        acc, mag = KR.gemm_acc(a[m0:m1, :Kd], b[:N, :Kd], device=dev)
        if second is not None:
            a2, b2, _ = second
            acc2, mag2 = KR.gemm_acc(a2[m0:m1, :k2], b2[:N, :k2], device=dev)
            acc, mag = acc + acc2, mag + mag2
            del acc2, mag2
        if aff_rows:
            sc, sh = _rows(scale, m0, m1, aff_rows, N), _rows(shift, m0, m1, aff_rows, N)
        elif per_row:
            sc, sh = scale[m0:m1].double()[:, None], shift[m0:m1].double()[:, None]
        else:
            sc, sh = scale[:N].double(), shift[:N].double()
        res = residual[m0:m1, :N].double() if residual is not None else None
        v, A = KR.epilogue(acc, mag, sc, sh, res, relu=relu, device=dev)
        del acc, mag
        if base is not None:
            bb = base[m0:m1, :N].double()
            v, A = v + bb, A + bb.abs()
        ref = v if mask is None else torch.where(mask[m0:m1, :N] > 0, v, torch.zeros_like(v))
        wst.add("d", d[m0:m1, :N], ref, KR.bound(v, A, not out_f32), m0)
        if pad:
            _pad_zero(wst, "d", d[m0:m1], N, m0)
        if d2 is not None:
            sc2, sh2, rows2 = next_affine
            ref2, A2 = KR.second_output(v, A, _rows(sc2, m0, m1, rows2, N), _rows(sh2, m0, m1, rows2, N), device=dev)
            wst.add("d2", d2[m0:m1, :N], ref2, KR.bound(ref2, A2, True), m0)
            if pad:
                _pad_zero(wst, "d2", d2[m0:m1], N, m0)
        del v, A
    return wst.result()


def check_chain_h1(d, N, w1, scale1, shift1, n1, h1):
    """h1 = relu(scale1 * (D . W1[:n1, :N]^T) + shift1) from the kernel's own fp16 D; columns [n1, ldd1) zero."""
    dev = h1.device
    M = d.shape[0]
    chunk = _samples_per_chunk(8 * (2 * N + 8 * n1))
    wst = _Worst()
    for m0 in range(0, M, chunk):
        m1 = min(M, m0 + chunk)
        acc, mag = KR.gemm_acc(d[m0:m1, :N], w1[:n1, :N], device=dev)
        v, A = KR.epilogue(acc, mag, scale1[:n1], shift1[:n1], relu=True, device=dev)
        wst.add("h1", h1[m0:m1, :n1], v, KR.bound(v, A, True), m0)
        _pad_zero(wst, "h1", h1[m0:m1], n1, m0)
    return wst.result()


# ---------------------------------------------------------------------------------------------
# attention
# ---------------------------------------------------------------------------------------------
def check_attention(q, k, v, d, dv, B, Nq, Nk, mode, o):
    """o fp16 [B * Nq][>= dv] against ``att_ref`` with the bound of ``att_bound``, in chunks of samples (and of query rows when one
    sample's probability matrix alone is over the cap)."""
    per_q = 8 * 4 * Nk + 8 * 8 * dv
    q_chunk = min(Nq, _samples_per_chunk(per_q))
    wst = _Worst()
    for b in range(B):
        kb, vb = k[b * Nk:(b + 1) * Nk, :d], v[b * Nk:(b + 1) * Nk, :dv]
        for i0 in range(0, Nq, q_chunk):
            i1 = min(Nq, i0 + q_chunk)
            r0, r1 = b * Nq + i0, b * Nq + i1
            ref, pv = KR.att_ref(q[r0:r1, :d], kb, vb, 1, i1 - i0, Nk, mode)
            bnd = KR.att_bound(ref, pv, vb, 1, i1 - i0, Nk, mode)
            wst.add("o", o[r0:r1, :dv], ref, bnd, r0)
    return wst.result()


# ---------------------------------------------------------------------------------------------
# pooling, shortcuts, copies
# ---------------------------------------------------------------------------------------------
def _ncdhw(x2d, N, T, H, W, C):
    return x2d[:, :C].reshape(N, T, H, W, C).permute(0, 4, 1, 2, 3)


def check_maxpool(x2d, N, T, H, W, C, k, s, p, y, out_size=None, ceil=False):
    """Bit-exact against F.max_pool3d of the same fp16 values (padding never wins: torch pads with -inf)."""
    wst = _Worst()
    per = 8 * 2 * T * H * W * C
    n_chunk = _samples_per_chunk(per)
    for n0 in range(0, N, n_chunk):
        n1 = min(N, n0 + n_chunk)
        xc = _ncdhw(x2d[n0 * T * H * W:n1 * T * H * W], n1 - n0, T, H, W, C).double()
        ref = F.max_pool3d(xc, k, s, p, ceil_mode=ceil)
        To, Ho, Wo = ref.shape[2:]
        ref = ref.permute(0, 2, 3, 4, 1).reshape(-1, C)
        r0 = n0 * To * Ho * Wo
        if out_size is not None and tuple(out_size) != (To, Ho, Wo):
            raise AuditError("pool output extent %s, torch gives %s" % (tuple(out_size), (To, Ho, Wo)))
        wst.exact("y", y[r0:r0 + ref.shape[0], :C], ref, r0)
    return wst.result()


def check_avgpool_global(x2d, N, S, C, y):
    """y[n] = fp16(mean over the S positions of sample n): any fp32 summation order of S terms errs by at most
    (S - 1) 2^-24 sum |x| (then a divide, 2^-24, and the fp16 rounding, 2^-11 |ref|)."""
    wst = _Worst()
    for n0, n1 in _chunks(N, 8 * 3 * S * C):
        xs = x2d[n0 * S:n1 * S, :C].reshape(n1 - n0, S, C).double()
        ref = xs.mean(1)
        bnd = KR.U_F16 * ref.abs() + (S + 1) * KR.FLOOR * xs.abs().sum(1) / S + KR.FLOOR
        wst.add("y", y[n0:n1, :C], ref, bnd, n0)
    return wst.result()


def check_shortcut_a(x2d, N, T, H, W, C, stride, y, out_channels):
    """Type-A shortcut: the strided pixel subset, channels [C, out_channels) zero -- bit-exact."""
    To, Ho, Wo = (T - 1) // stride + 1, (H - 1) // stride + 1, (W - 1) // stride + 1
    S, So = T * H * W, To * Ho * Wo
    wst = _Worst()
    for n0, n1 in _chunks(N, 8 * (S + 2 * So) * y.shape[1]):
        xs = x2d[n0 * S:n1 * S, :C].reshape(n1 - n0, T, H, W, C)[:, ::stride, ::stride, ::stride].reshape(-1, C)
        yc = y[n0 * So:n1 * So]
        wst.exact("y", yc[:, :C], xs, n0 * So)
        _pad_zero(wst, "y", yc, C, n0 * So)
    return wst.result()


def _row_chunks(rows, cols):
    n = _samples_per_chunk(8 * 4 * cols)
    return [(r0, min(rows, r0 + n)) for r0 in range(0, rows, n)]


def check_concat(a2d, Ca, b2d, Cb, y):
    wst = _Worst()
    for r0, r1 in _row_chunks(y.shape[0], Ca + Cb):
        wst.exact("y", y[r0:r1, :Ca + Cb], torch.cat([a2d[r0:r1, :Ca], b2d[r0:r1, :Cb]], 1), r0)
    return wst.result()


def check_relu6(x2d, y):
    wst = _Worst()
    for r0, r1 in _row_chunks(y.shape[0], y.shape[1]):
        wst.exact("y", y[r0:r1], x2d[r0:r1].clamp(0.0, 6.0), r0)
    return wst.result()


def check_dwconv(x2d, N, H, W, C, w9, scale, shift, stride, clamp_in, relu6, y):
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    S, So = H * W, Ho * Wo
    wst = _Worst()
    for n0, n1 in _chunks(N, 8 * (2 * S + 8 * So) * C):
        ref, A = KR.dw_ref(x2d[n0 * S:n1 * S, :C].reshape(n1 - n0, H, W, C), w9, scale, shift, stride, clamp_in, relu6,
                           device=y.device)
        wst.add("y", y[n0 * So:n1 * So, :C], ref, KR.bound(ref, A, True), n0 * So)
    return wst.result()


# ---------------------------------------------------------------------------------------------
# column-slice outputs (BNInception, Inception-v4, DenseNet), pre-activated GEMM, DenseNet pools, squeeze-excite
# ---------------------------------------------------------------------------------------------
class SliceGuard:
    """The slice contract of an entry that writes column slices of wider matrices: after the call, every column of the parent
    rows outside the slices is bit for bit what it was before (compared as int16, so NaN patterns in uninitialised columns
    compare equal).  ``views``: (fp16 [rows][cols] view, columns the entry writes from the view's first column on).  The parent
    is the view's base, which must be a 2-D matrix of the view's row pitch: its rows, not an assumed row grid of the storage,
    locate the slice (a view into a flat workspace raises).  A view of whole rows has nothing outside it; slices of the same
    rows are checked together."""

    def __init__(self, views):
        groups = {}
        for y, width in views:
            pitch, rows = y.stride(0), y.shape[0]
            if y.shape[1] == pitch:
                continue
            base = y._base
            if base is None or base.dim() != 2 or base.stride() != (pitch, 1):
                raise AuditError("the parent of a %s column slice of pitch %d is not a 2-D matrix of that pitch (%s): its rows "
                                 "cannot be located" % (tuple(y.shape), pitch, None if base is None else tuple(base.shape)))
            r0, c0 = divmod(y.storage_offset() - base.storage_offset(), pitch)
            if r0 < 0 or r0 + rows > base.shape[0] or c0 + width > pitch:
                raise AuditError("a %s column slice at row %d col %d does not lie inside its %s parent" % (tuple(y.shape), r0, c0,
                                                                                                      tuple(base.shape)))
            groups.setdefault((base.data_ptr(), r0, rows), (base, []))[1].append((c0, c0 + width))
        self.spans = []
        for (_, r0, rows), (base, cols) in groups.items():
            keep = torch.ones(base.shape[1], dtype=torch.bool, device=base.device)
            for c0, c1 in cols:
                keep[c0:c1] = False
            if bool(keep.any()):
                span = base[r0:r0 + rows].view(torch.int16)
                self.spans.append((span, keep, span.clone()))

    def check(self):
        """(0, ...) when every column outside the slices is unchanged, else (inf, the first changed element; its row counts from
        the slices' first row, as the output rows of the entry do)."""
        wst = _Worst()
        for span, keep, before in self.spans:
            diff = (span != before) & keep
            if bool(diff.any()):
                m, c = (int(v) for v in torch.nonzero(diff)[0])
                wst.ratio = float("inf")
                wst.where = "outside the slice row %d col %d: bits %#06x, were %#06x" % (m, c, int(span[m, c]) & 0xFFFF,
                                                                                         int(before[m, c]) & 0xFFFF)
                break
        return wst.result()


def check_gemm_split(a, b, scale, shift, M, Kd, dests, relu=True):
    """Destination d (fp16 [M][cols_d]) = act(scale * A[:, :Kd] . B[rows]^T + shift) over the packed rows
    [64 box0[d], 64 box0[d] + cols_d) of B / scale / shift (``ops.split_plan``): each held to the GEMM bound of ``check_gemm``."""
    from pretorched_x_b200 import ops
    _, box0 = ops.split_plan([y.shape[1] for y in dests])
    wst = _Worst()
    for d, y in enumerate(dests):
        r0, n = 64 * box0[d], y.shape[1]
        wst.merge("dest %d" % d, *check_gemm(a, b[r0:r0 + n], scale[r0:r0 + n], shift[r0:r0 + n], M, n, Kd, y, relu=relu))
    return wst.result()


def check_pool_slice(x2d, N, T, H, W, C, k, s, p, avg, y, count_include_pad=True, ceil_mode=True):
    """nn.MaxPool2d / nn.AvgPool2d over every frame of x2d (fp16 rows [N T H W][>= C], any row pitch) into y (fp16 rows
    [N T Ho Wo][>= C]); k, s, p are (h, w) pairs.  Max: bit-exact against F.max_pool2d of the same fp16 values.  Average: an fp32
    sum of at most kh kw taps (each addition errs by 2^-24 of the partial sum, at most the sum of the taps' magnitudes), one
    division by the divisor (2^-24) and the fp16 rounding, so |got - ref| <= 2^-11 |ref| + max(16, kh kw) 2^-24 mean|x| + 2^-24
    with mean|x| the same average of |x| (the padding counted or not): 2^-20 mean|x| for windows of at most 16 taps."""
    S = T * H * W
    wst = _Worst()
    rows_out = None
    for n0, n1 in _chunks(N, 8 * 6 * S * C):
        xs = x2d[n0 * S:n1 * S, :C].double().reshape((n1 - n0) * T, H, W, C).permute(0, 3, 1, 2)
        if avg:
            ref = F.avg_pool2d(xs, k, s, p, ceil_mode=ceil_mode, count_include_pad=count_include_pad)
            mag = F.avg_pool2d(xs.abs(), k, s, p, ceil_mode=ceil_mode, count_include_pad=count_include_pad)
        else:
            ref = F.max_pool2d(xs, k, s, p, ceil_mode=ceil_mode)
        Ho, Wo = ref.shape[2:]
        So = T * Ho * Wo
        if rows_out is None:
            rows_out = N * So
            if y.shape[0] != rows_out:
                raise AuditError("pool output has %d rows, torch gives %d" % (y.shape[0], rows_out))
        ref = ref.permute(0, 2, 3, 1).reshape(-1, C)
        yc = y[n0 * So:n1 * So, :C]
        if avg:
            mag = mag.permute(0, 2, 3, 1).reshape(-1, C)
            wst.add("y", yc, ref, KR.U_F16 * ref.abs() + max(16, k[0] * k[1]) * KR.FLOOR * mag + KR.FLOOR, n0 * So)
        else:
            wst.exact("y", yc, ref, n0 * So)
    return wst.result()


def check_gemm_preact(a, b, scale, shift, in_scale, in_shift, M, N, Kd, d, relu=True):
    """D[M][N] = act(scale * relu(in_scale * A[:, :Kd] + in_shift) . B[:N, :Kd]^T + shift), the in-affine operand rounded to fp16
    once (``KR.in_affine_acc``), held to the GEMM bound; the pad columns [N, ldd) of D are zero."""
    dev = d.device
    wst = _Worst()
    for m0, m1 in _chunks(M, 8 * 8 * (Kd + N)):
        acc, mag = KR.in_affine_acc(a[m0:m1, :Kd], b[:N, :Kd], in_scale[:Kd], in_shift[:Kd], m1 - m0, device=dev)
        v, A = KR.epilogue(acc, mag, scale[:N], shift[:N], relu=relu, device=dev)
        del acc, mag
        wst.add("d", d[m0:m1, :N], v, KR.bound(v, A, True), m0)
        _pad_zero(wst, "d", d[m0:m1], N, m0)
    return wst.result()


# What ``preact_contract`` puts past Kd: A's columns [Kd, lda) hold PREACT_A, the input affine's entries [Kd, round_up(Kd, 64))
# PREACT_IN (scale, shift) and B is handed over at a wider pitch whose extra columns hold PREACT_B.  Every value is finite and
# relu(PREACT_A s + t) > 0, so a kernel that reads any of them moves its output by about PREACT_B relu(PREACT_A s + t) per column
# read, far past the bound.
PREACT_A, PREACT_IN, PREACT_B = 2.0, (1.0, 0.5), 0.125


def preact_contract(ba):
    """The pre-activated GEMM's contract: its output depends only on A[:, :Kd], B[:N, :Kd] and in_scale / in_shift[:Kd] (its A
    and B tensor maps span Kd columns, and the hardware zero-fills the rest of the last 64-column K block).

    A poison has to survive the kernel's A transform to be seen: that computes fmaxf(fmaf(x, s, t), 0), and fmaxf returns its
    non-NaN operand, so a NaN (or fmaf(Inf, 0, 0)) past Kd would turn into 0 and vanish.  The call therefore gets finite
    values past Kd everywhere the kernel could look: A's columns [Kd, lda) are set to PREACT_A in place (their exact bits come
    back afterwards), and the call receives copies of the input affine that are PREACT_IN past Kd and a copy of B at a pitch 64
    columns wider, PREACT_B there.  Returns (the call's keyword arguments, the restoring function)."""
    a, b, M, Kd = ba["a2d"], ba["b2d"], ba["M"], ba["Kd"]
    lda = a.stride(0)
    call = dict(ba)
    restore = lambda: None                                   # noqa: E731
    if lda > Kd:
        if (a.storage_offset() + M * lda) * a.element_size() > a.untyped_storage().nbytes():
            raise AuditError("the %d rows of pitch %d of the pre-activated GEMM's A run past its storage" % (M, lda))
        tail = a.as_strided((M, lda - Kd), (lda, 1), a.storage_offset() + Kd).view(torch.int16)
        saved = tail.clone()
        tail.view(torch.float16).fill_(PREACT_A)
        restore = lambda: tail.copy_(saved)                  # noqa: E731
    for key, v in (("in_scale", PREACT_IN[0]), ("in_shift", PREACT_IN[1])):
        t = ba[key].clone()
        t[Kd:] = v
        call[key] = t
    wide = torch.full((b.shape[0], b.stride(0) + 64), PREACT_B, dtype=b.dtype, device=b.device)
    wide[:, :Kd] = b[:, :Kd]
    call["b2d"] = wide
    return call, restore


def _affine_relu(xs, scale, shift, C):
    """relu(scale * x + shift) of fp64 rows [..][C] and the magnitude |scale x| + |shift| of its terms."""
    sc, sh = scale[:C].double().to(xs.device), shift[:C].double().to(xs.device)
    return (xs * sc + sh).clamp_min(0.0), (xs * sc).abs() + sh.abs()


def check_transition_pool(x2d, N, H, W, C, scale, shift, y):
    """y = the 2x2 mean of relu(scale * x + shift) (floor extents): per tap one fp32 FMA (2^-24 of |s x| + |t|), three additions
    and a division, then the fp16 rounding: |got - ref| <= 2^-11 |ref| + 2^-20 mean(|s x| + |t|) + 2^-24."""
    S, Ho, Wo = H * W, H // 2, W // 2
    So = Ho * Wo
    wst = _Worst()
    for n0, n1 in _chunks(N, 8 * 6 * S * C):
        v, A = _affine_relu(x2d[n0 * S:n1 * S, :C].double(), scale, shift, C)
        ref, mag = (F.avg_pool2d(t.reshape(n1 - n0, H, W, C).permute(0, 3, 1, 2), 2, 2).permute(0, 2, 3, 1).reshape(-1, C)
                    for t in (v, A))
        wst.add("y", y[n0 * So:n1 * So, :C], ref, KR.U_F16 * ref.abs() + 2.0 ** -20 * mag + KR.FLOOR, n0 * So)
    return wst.result()


def check_head_pool(x2d, N, S, C, scale, shift, y):
    """y[n] = the mean over the S positions of relu(scale * x + shift): one FMA per term, S - 1 fp32 additions in any order, the
    multiplication by a rounded 1 / S (two roundings), the fp16 rounding: |got - ref| <= 2^-11 |ref| + max(64, S + 2) 2^-24
    mean(|s x| + |t|) + 2^-24 (2^-18 mean(|s x| + |t|) up to S = 62)."""
    wst = _Worst()
    for n0, n1 in _chunks(N, 8 * 6 * S * C):
        v, A = _affine_relu(x2d[n0 * S:n1 * S, :C].double(), scale, shift, C)
        ref, mag = (t.reshape(n1 - n0, S, C).mean(1) for t in (v, A))
        wst.add("y", y[n0:n1, :C], ref, KR.U_F16 * ref.abs() + max(64, S + 2) * KR.FLOOR * mag + KR.FLOOR, n0)
    return wst.result()


def check_se_excite(h2d, N, S, C2, w1, b1, w2, b2, s3, t3, scale, shift):
    """(scale, shift) fp32 [N][>= C] against ``KR.excite_ref`` of the kernel's own operands (the folded fp32 w1 / b1, then w2, b2,
    s3, t3) under ``KR.excite_bound``."""
    m, habs = KR.excite_mean(h2d, N, S, C2, device=scale.device)
    r = KR.excite_ref(m, habs, w1, b1, w2, b2, s3, t3)
    bs, bh = KR.excite_bound(r, w1, b1, w2, b2, s3, t3, S)
    C = w2.shape[0]
    wst = _Worst()
    wst.add("scale", scale[:, :C], r["scale"], bs)
    wst.add("shift", shift[:, :C], r["shift"], bh)
    return wst.result()


# ---------------------------------------------------------------------------------------------
# BigGAN helpers
# ---------------------------------------------------------------------------------------------
# One fp32 FMA or product (2^-24 of its magnitude), at most one fp32 sum on top, then the fp16 rounding: an element of a
# ccbn / embed / head output is held to 2^-11 |ref| + 2^-22 A + 2^-24, A the sum of the magnitudes of its terms.
EW_B = 2.0 ** -22
# tanh(v) = 1 - 2 / (exp(2v) + 1) with __expf (relative error <= (2 + 1.16 * 30) ulp for |2v| <= 30, < 2^-18.7) and __fdividef
# (2 ulp): the quotient, at most 2, errs by < 2^-17.5 in absolute terms, the subtraction adds 2^-24.  tanh is 1-Lipschitz, so
# an input error e moves the output by at most e.
TANH_ABS = 2.0 ** -17


def _chunks(N, per_sample_bytes):
    n = _samples_per_chunk(per_sample_bytes)
    return [(n0, min(N, n0 + n)) for n0 in range(0, N, n)]


def check_ccbn(x2d, N, H, W, C, scale, shift, up, relu, y):
    """y = act(x * scale[n] + shift[n]) (nearest ``up``-fold upsampled); scale None: a copy; [1][>= C]: shared by all samples."""
    S, So = H * W, H * W * up * up
    wst = _Worst()
    for n0, n1 in _chunks(N, 8 * 6 * So * C):
        xs = x2d[n0 * S:n1 * S, :C].double()
        if scale is not None:
            rows = S if scale.shape[0] > 1 else N * S
            sc, sh = _rows(scale, n0 * S, n1 * S, rows, C), _rows(shift, n0 * S, n1 * S, rows, C)
            v, A = xs * sc + sh, (xs * sc).abs() + sh.abs()
        else:
            v, A = xs, xs.abs()
        if relu:
            v = v.clamp_min(0.0)
        if up > 1:
            v, A = (t.reshape(n1 - n0, H, W, C).repeat_interleave(up, 1).repeat_interleave(up, 2).reshape(-1, C) for t in (v, A))
        yc = y[n0 * So:n1 * So]
        wst.add("y", yc[:, :C], v, KR.U_F16 * v.abs() + EW_B * A + KR.FLOOR, n0 * So)
        _pad_zero(wst, "y", yc, C, n0 * So)
    return wst.result()


def check_embed_concat(z, labels, table, split, y):
    """v = [table[labels] | z | 0]: y = fp16(v), or with ``split`` [hi | lo | hi] with hi = fp16(v) and hi + lo = v to
    2^-22 |v| + 2^-24 (lo is a second fp16 rounding, of v - hi)."""
    B, dz = z.shape
    ds = table.shape[1]
    D = (dz + ds + 7) // 8 * 8
    emb = table.double()[labels.long()] if labels.dim() == 1 else labels.double()
    v = torch.zeros((B, D), dtype=torch.float64, device=y.device)
    v[:, :ds], v[:, ds:ds + dz] = emb, z.double()
    wst = _Worst()
    hi = y[:, :D]
    wst.add("hi", hi, v, KR.U_F16 * v.abs() + 2.0 ** -25 + KR.FLOOR * 2.0 ** -30)
    if split:
        wst.add("hi + lo", hi.double() + y[:, D:2 * D].double(), v, 2.0 ** -22 * v.abs() + KR.FLOOR)
        wst.exact("third block", y[:, 2 * D:3 * D], hi)
    return wst.result()


def check_rgb_head(partial, bias, N, H, W, K, y):
    """y[n][k][h][w] = tanh(bias[k] + sum over the 3x3 taps of partial[(n, h + dh - 1, w + dw - 1)][(dh * 3 + dw) * 4 + k]): a
    sequential fp32 sum of at most ten terms (9 2^-24 of their magnitudes), the tanh (``TANH_ABS``), the output rounding."""
    S = H * W
    bb = bias[:K].double().view(1, K, 1, 1)
    f16 = y.dtype == torch.float16
    wst = _Worst()
    for n0, n1 in _chunks(N, 8 * (2 * 9 * K + 8 * K) * (H + 2) * (W + 2)):
        n = n1 - n0
        P = partial[n0 * S:n1 * S, :36].double().reshape(n, H, W, 9, 4)[..., :K]
        Pp = F.pad(P.permute(0, 3, 4, 1, 2), (1, 1, 1, 1))              # [n, 9, K, H + 2, W + 2]
        acc = torch.zeros((n, K, H, W), dtype=torch.float64, device=y.device)
        mag = torch.zeros_like(acc)
        for dh in range(3):
            for dw in range(3):
                t = Pp[:, dh * 3 + dw, :, dh:dh + H, dw:dw + W]
                acc, mag = acc + t, mag + t.abs()
        ref = torch.tanh(acc + bb)
        bnd = (KR.U_F16 if f16 else 2.0 ** -24) * ref.abs() + 9 * KR.FLOOR * (mag + bb.abs()) + TANH_ABS + KR.FLOOR
        wst.add("image", y[n0:n1].reshape(n * K, S), ref.reshape(n * K, S), bnd.reshape(n * K, S), n0 * K)
    return wst.result()


def check_tanh(x2d, N, C, S, y):
    """y[n][c][s] = tanh(x[n * S + s][c]) (NCHW, fp32 or fp16)."""
    f16 = y.dtype == torch.float16
    wst = _Worst()
    for n0, n1 in _chunks(N, 8 * 6 * S * C):
        n = n1 - n0
        ref = torch.tanh(x2d[n0 * S:n1 * S, :C].double()).reshape(n, S, C).permute(0, 2, 1)
        bnd = (KR.U_F16 if f16 else 2.0 ** -24) * ref.abs() + TANH_ABS + KR.FLOOR
        wst.add("image", y[n0:n1].reshape(n * C, S), ref.reshape(n * C, S), bnd.reshape(n * C, S), n0 * C)
    return wst.result()


# ---------------------------------------------------------------------------------------------
# the patching auditor
# ---------------------------------------------------------------------------------------------
class AuditReport:
    """``rows``: one dict per audited or recorded launch (index, entry, geometry, kernel, info, launches, ratio, where);
    ``launches``: the library launch-count delta of the whole call; ``counted``: the sum over the wrapped entries; ``ref_flops``:
    the fp64 operations of the reference products, each counted twice (the value and the magnitude sum |x| |w|)."""

    def __init__(self):
        self.rows, self.launches, self.counted, self.output = [], 0, 0, None
        self.ref_flops = 0.0           # fp64 floating-point operations of the references' products (convolutions, GEMMs, attention)

    @property
    def worst(self):
        return max([r["ratio"] for r in self.rows if r["ratio"] is not None] or [0.0])

    def failures(self):
        return [r for r in self.rows if r["ratio"] is not None and not r["ratio"] <= 1.0]

    def table(self, name):
        lines = []
        for r in self.rows:
            lines.append("[model-audit] %s #%-4d %-15s %-58s %-12s %-22s %s" % (
                name, r["index"], r["entry"], r["geometry"][:58], r["kernel"], r["info"],
                "-" if r["ratio"] is None else "%.4f" % r["ratio"]))
        return "\n".join(lines)


def _last_kernel(lib):
    info = (ctypes.c_int * 5)()
    kid = lib.b2_debug_last_kernel(info)
    return KIND.get(kid, str(kid)), tuple(info)


def _storage_of(t):
    return t.untyped_storage().data_ptr() if isinstance(t, torch.Tensor) else None


def _tensor_of(v):
    from pretorched_x_b200 import ops
    return v.data if isinstance(v, ops.Act) else v


class _Auditor:
    def __init__(self, lib, ops, chain_bitwise=True):
        self.lib, self.ops, self.report = lib, ops, AuditReport()
        self.sources = {}              # id(pack) -> (pack, source weight, kind)
        self.depth = 0
        self.extra = 0                 # launches the auditor itself made (the chain's stand-alone cross-check)
        self.chain_bitwise = chain_bitwise

    # -- bookkeeping --
    def record(self, entry, geometry, launches, ratio=None, where="", kernel="-", info="-"):
        self.report.rows.append(dict(index=len(self.report.rows), entry=entry, geometry=geometry, kernel=kernel, info=info,
                                     launches=launches, ratio=ratio, where=where))
        self.report.counted += launches

    def wrap(self, name, orig):
        sig = inspect.signature(orig)
        ops = self.ops

        @functools.wraps(orig)
        def wrapped(*args, **kwargs):
            if name in PASS_THROUGH:
                return orig(*args, **kwargs)
            if self.depth:
                raise AuditError("entry %s called inside another audited entry" % name)
            if name not in UNAUDITED:
                if not hasattr(self, "audit_" + name):
                    raise AuditError("%s launched on an audited forward, and the audit has no check for it" % name)
                unknown = set(sig.parameters) - set(KNOWN.get(name, ()))
                if unknown:
                    raise AuditError("%s takes %s, which its check does not model" % (name, ", ".join(sorted(unknown))))
            bound = sig.bind(*args, **kwargs)
            bound.apply_defaults()
            ba = dict(bound.arguments)
            snap = self.snapshot(name, ba)
            guard = SliceGuard(self.slices(name, ba))
            call, restore = preact_contract(ba) if name == "gemm_preact" else (None, lambda: None)
            self.depth += 1
            try:
                torch.cuda.synchronize()
                c0 = self.lib.b2_launch_count()
                out = orig(*args, **kwargs) if call is None else orig(**call)
                torch.cuda.synchronize()
                n = self.lib.b2_launch_count() - c0
            finally:
                self.depth -= 1
                restore()
            if name in UNAUDITED:
                self.record(name, "", n)
                return out
            kernel, info = _last_kernel(self.lib) if name in RECORDS_KERNEL else ("-", "-")
            if n < 1:
                raise AuditError("%s returned without a launch" % name)
            geometry, (ratio, where) = getattr(self, "audit_" + name)(snap, out)
            r_out, w_out = guard.check()
            if not r_out <= ratio:
                ratio, where = r_out, w_out
            self.record(name, geometry, n, ratio, where, kernel, str(info))
            return out
        return wrapped

    def snapshot(self, name, ba):
        """Clone every operand that shares storage with a caller-provided output (out=, an in-place Act, an fp32 base)."""
        outs = [ba.get("out"), ba.get("y")]
        if name == "relu6_":
            outs.append(ba["a"])
        if name == "gemm" and ba.get("accumulate"):
            ba["base"] = ba["out"].clone()
        if name == "gemm_split":
            outs.extend(ba["dests"])
        ptrs = {_storage_of(_tensor_of(o)) for o in outs if o is not None}
        ptrs.discard(None)
        if ptrs:
            for key, v in list(ba.items()):
                if key in ("out", "y", "base"):
                    continue
                t = _tensor_of(v)
                if isinstance(t, torch.Tensor) and _storage_of(t) in ptrs:
                    ba[key] = self.ops.Act(t.clone(), v.N, v.T, v.H, v.W, v.C) if isinstance(v, self.ops.Act) else t.clone()
        return ba

    @staticmethod
    def slices(name, ba):
        """(view, columns written) of every column slice of a wider matrix the entry writes (``SliceGuard``)."""
        if name == "conv_slice":
            return [(ba["y"], ba["pc"].K)]
        if name == "gemm_split":
            return [(y, y.shape[1]) for y in ba["dests"]]
        if name in ("pool_slice", "bn_relu_avgpool2") and ba["y"] is not None:
            return [(ba["y"], ba["a"].C)]
        return []

    # -- packs --
    def wrap_init(self, cls, kind):
        orig = cls.__init__
        aud = self

        @functools.wraps(orig)
        def init(pack, weight, *args, **kwargs):
            c0 = aud.lib.b2_launch_count() if aud.lib is not None else 0
            orig(pack, weight, *args, **kwargs)
            torch.cuda.synchronize()
            n = aud.lib.b2_launch_count() - c0
            aud.sources[id(pack)] = (pack, weight.detach().clone(), kind)
            aud.record(cls.__name__, "K%d Cin%d k%s%s" % (pack.K, pack.Cin, "x".join(map(str, pack.k)),
                                                         " up" if getattr(pack, "up", False) else ""), n)
        return orig, init

    def filter_of(self, pc, x_pitch):
        ops = self.ops
        src = self.sources.get(id(pc))
        if isinstance(pc, ops.PackedGroupedConv):
            if src is None:
                raise AuditError("grouped pack built before the audit: its filter cannot be read back")
            return grouped_filter(src[1], pc.groups, pc.C).to(pc.w.device)
        taps = pc.k[0] * pc.k[1] * pc.k[2]
        if pc.mode == ops.B2_CONV_STEM7:
            if src is None:
                raise AuditError("stem pack built before the audit: its filter cannot be read back")
            return stem_filter(src[1].cpu()).to(pc.w.device)
        if pc.up:
            wph = pc.w.view(pc.K, 16, pc.C)
            if src is None:
                raise AuditError("upsampling pack built before the audit")
            r, where = check_upconv_pack(wph, src[1])
            if not r <= 1.0:
                raise AuditError("upsampling pack differs from the fold of its weight: %s" % where)
            return wph
        return pc.w.view(pc.K, taps, pc.C)

    # -- entries --
    def audit_conv(self, b, y):
        ops = self.ops
        a, pc = b["a"], b["pc"]
        y2 = None
        if isinstance(y, tuple):
            y, y2 = y
        grouped = isinstance(pc, ops.PackedGroupedConv)
        w = self.filter_of(pc, a.ld)
        x = a.data.view(a.N, a.T, a.H, a.W, a.ld)
        if b["simt"]:
            raise AuditError("the CUDA-core cross-check is not a forward path")
        res = b["residual"].data if b["residual"] is not None else None
        flags = [f for f in ("relu", "residual_up", "residual_pre", "pool_w") if b[f]] + \
                [f for f in ("sample_affine", "next_affine", "in_affine", "mask", "out") if b[f] is not None]
        geom = "%s N%d %dx%dx%d C%d->%d k%s s%s p%s%s%s" % ("gconv" if grouped else "conv", a.N, a.T, a.H, a.W, a.ld, pc.K,
                                                         "".join(map(str, pc.k)), "".join(map(str, pc.s)), "".join(map(str, pc.p)),
                                                         " up" if getattr(pc, "up", False) else "", " " + ",".join(flags) if flags else "")
        taps = 4 if getattr(pc, "up", False) else pc.k[0] * pc.k[1] * pc.k[2]
        rows = y.M * (2 if b["pool_w"] else 1)
        self.report.ref_flops += 2 * 2.0 * rows * pc.K * a.ld * taps
        return geom, check_conv(x, w, pc.scale, pc.shift, pc.k, pc.s, pc.p, y.data, pc.K, residual=res, relu=b["relu"],
                                sample_affine=b["sample_affine"], residual_up=b["residual_up"], residual_pre=b["residual_pre"],
                                next_affine=b["next_affine"], y2=y2.data if y2 is not None else None, pool_w=b["pool_w"],
                                in_affine=b["in_affine"], upsample=getattr(pc, "up", False),
                                mask=b["mask"].data if b["mask"] is not None else None)

    def audit_gemm(self, b, out):
        d, d2 = (out if isinstance(out, tuple) else (out, None))
        flags = [f for f in ("relu", "per_row", "out_f32", "accumulate") if b[f]] + \
                [f for f in ("residual", "second", "next_affine", "mask", "out") if b[f] is not None] + \
                (["aff_rows=%d" % b["aff_rows"]] if b["aff_rows"] else [])
        if b["accumulate"] and not b["out_f32"]:
            raise AuditError("accumulate into an fp16 output")
        self.report.ref_flops += 2 * 2.0 * b["M"] * b["N"] * (b["Kd"] + (b["second"][2] if b["second"] is not None else 0))
        geom = "gemm M%d N%d K%d%s%s" % (b["M"], b["N"], b["Kd"], "+%d" % b["second"][2] if b["second"] is not None else "",
                                         " " + ",".join(flags) if flags else "")
        return geom, check_gemm(b["a2d"], b["b2d"], b["scale"], b["shift"], b["M"], b["N"], b["Kd"], d, residual=b["residual"],
                                relu=b["relu"], per_row=b["per_row"], out_f32=b["out_f32"], base=b.get("base"), second=b["second"],
                                aff_rows=b["aff_rows"], next_affine=b["next_affine"], d2=d2, mask=b["mask"],
                                pad=b["out"] is None and not b["out_f32"])

    def audit_gemm_sample_affine(self, b, d):
        self.report.ref_flops += 2 * 2.0 * b["M"] * b["N"] * b["Kd"]
        geom = "gemm_sa M%d N%d K%d rows%d%s" % (b["M"], b["N"], b["Kd"], b["aff_rows"], " res" if b["residual"] is not None else "")
        return geom, check_gemm(b["a2d"], b["b2d"], b["scale"], b["shift"], b["M"], b["N"], b["Kd"], d, residual=b["residual"],
                                relu=b["relu"], aff_rows=b["aff_rows"], pad=True)

    def audit_gemm_chain(self, b, out):
        d, h1 = out
        N, n1 = b["N"], b["n1"]
        geom = "chain M%d N%d K%d%s -> %d%s" % (b["M"], N, b["Kd"], "+%d" % b["second"][2] if b["second"] is not None else "", n1,
                                               " res" if b["residual"] is not None else "")
        r1, w1 = check_gemm(b["a2d"], b["b2d"], b["scale"], b["shift"], b["M"], N, b["Kd"], d, residual=b["residual"],
                            relu=b["relu"], second=b["second"])
        r2, w2 = check_chain_h1(d, N, b["w1"], b["scale1"], b["shift1"], n1, h1)
        self.report.ref_flops += 2 * 2.0 * b["M"] * (N * (b["Kd"] + (b["second"][2] if b["second"] is not None else 0)) + n1 * N)
        if self.chain_bitwise:
            # the documented contract: h1 equals the stand-alone GEMM of the kernel's own D bit for bit
            c0 = self.lib.b2_launch_count()
            alone = self._orig["gemm"](d, b["w1"], b["scale1"], b["shift1"], b["M"], n1, N, relu=True)
            torch.cuda.synchronize()
            self.extra += self.lib.b2_launch_count() - c0
            if not torch.equal(alone[:, :n1].view(torch.int16), h1[:, :n1].view(torch.int16)):
                r2, w2 = float("inf"), "h1 differs from the stand-alone conv1 GEMM of the same D"
        return geom, max([(r1, w1), (r2, w2)], key=lambda t: t[0] if t[0] == t[0] else float("inf"))

    def audit_attention(self, b, o):
        mode = b["mode"] if b["mode"] is not None else (1 if b["dot_product"] else 0)
        geom = "attention m%d B%d Nq%d Nk%d d%d dv%d" % (mode, b["B"], b["Nq"], b["Nk"], b["d"], b["dv"])
        self.report.ref_flops += 2.0 * b["B"] * b["Nq"] * b["Nk"] * (b["d"] + 2 * b["dv"])
        return geom, check_attention(b["q2d"], b["k2d"], b["v2d"], b["d"], b["dv"], b["B"], b["Nq"], b["Nk"], mode, o)

    def audit_maxpool3d(self, b, y):
        a = b["a"]
        geom = "maxpool N%d %dx%dx%d C%d k%s s%s p%s" % (a.N, a.T, a.H, a.W, a.C, b["kernel"], b["stride"], b["padding"])
        return geom, check_maxpool(a.data, a.N, a.T, a.H, a.W, a.C, b["kernel"], b["stride"], b["padding"], y.data, (y.T, y.H, y.W))

    def audit_maxpool2d_ceil(self, b, y):
        a, k, s, p = b["a"], b["k"], b["s"], b["p"]
        geom = "maxpool_ceil N%d %dx%dx%d C%d k%d s%d p%d" % (a.N, a.T, a.H, a.W, a.C, k, s, p)
        return geom, check_maxpool(a.data, a.N, a.T, a.H, a.W, a.C, (1, k, k), (1, s, s), (0, p, p), y.data, (y.T, y.H, y.W), ceil=True)

    def audit_avgpool_global(self, b, y):
        a = b["a"]
        # the kernel averages every one of the ld columns (the pad columns of a zero-padded input average to zero)
        return "avgpool N%d S%d C%d" % (a.N, a.positions, a.C), check_avgpool_global(a.data, a.N, a.positions, a.ld, y)

    def audit_shortcut_a(self, b, y):
        a = b["a"]
        return ("shortcut_a N%d %dx%dx%d C%d s%d" % (a.N, a.T, a.H, a.W, a.C, b["stride"]),
                check_shortcut_a(a.data, a.N, a.T, a.H, a.W, a.C, b["stride"], y.data, b["out_channels"]))

    def audit_concat_rows(self, b, y):
        return "concat rows%d C%d+%d" % (y.shape[0], b["Ca"], b["Cb"]), check_concat(b["a2d"], b["Ca"], b["b2d"], b["Cb"], y)

    def audit_relu6_(self, b, y):
        return "relu6 M%d C%d" % (y.M, y.C), check_relu6(b["a"].data, y.data)

    def audit_dwconv3x3(self, b, y):
        a = b["a"]
        geom = "dwconv N%d %dx%dx%d C%d s%d%s" % (a.N, a.T, a.H, a.W, a.C, b["stride"], " clamp_in" if b["clamp_in"] else "")
        return geom, check_dwconv(a.data, a.N * a.T, a.H, a.W, a.C, b["w9"], b["scale"], b["shift"], b["stride"], b["clamp_in"],
                                  b["relu6"], y.data)

    def audit_ccbn_act(self, b, y):
        a = b["a"]
        C = a.C if b["channels"] is None else b["channels"]
        geom = "ccbn N%d %dx%d C%d up%d%s" % (a.N, a.H, a.W, C, b["up"], " relu" if b["relu"] else "")
        return geom, check_ccbn(a.data, a.N, a.H, a.W, C, b["scale"], b["shift"], b["up"], b["relu"], y.data)

    def audit_embed_concat(self, b, y):
        z = b["z"]
        return ("embed B%d dz%d split%d" % (z.shape[0], z.shape[1], int(b["split"])),
                check_embed_concat(z.float(), b["labels"], b["table"], b["split"], y))

    def audit_rgb_head(self, b, y):
        return ("rgb_head N%d %dx%d K%d" % (b["N"], b["H"], b["W"], b["K"]),
                check_rgb_head(b["partial"], b["bias"], b["N"], b["H"], b["W"], b["K"], y))

    def audit_tanh_to_nchw(self, b, y):
        a = b["a"]
        return "tanh N%d %dx%d C%d" % (a.N, a.H, a.W, a.C), check_tanh(a.data, a.N, a.C, a.T * a.H * a.W, y)

    def audit_conv_slice(self, b, out):
        a, pc, y = b["a"], b["pc"], b["y"]
        w = self.filter_of(pc, a.ld)
        x = a.data.view(a.N, a.T, a.H, a.W, a.ld)
        geom = "conv_slice N%d %dx%dx%d C%d->%d k%s s%s p%s%s%s" % (a.N, a.T, a.H, a.W, a.ld, pc.K, "".join(map(str, pc.k)),
                                                                "".join(map(str, pc.s)), "".join(map(str, pc.p)),
                                                                " relu" if b["relu"] else "", " narrow" if b["narrow"] else "")
        self.report.ref_flops += 2 * 2.0 * y.shape[0] * pc.K * a.ld * pc.k[0] * pc.k[1] * pc.k[2]
        return geom, check_conv(x, w, pc.scale, pc.shift, pc.k, pc.s, pc.p, y, pc.K, relu=b["relu"])

    def audit_gemm_split(self, b, out):
        cols = [y.shape[1] for y in b["dests"]]
        self.report.ref_flops += 2 * 2.0 * b["M"] * sum(cols) * b["Kd"]
        geom = "gemm_split M%d K%d -> %s%s" % (b["M"], b["Kd"], "+".join(map(str, cols)), " relu" if b["relu"] else "")
        return geom, check_gemm_split(b["a2d"], b["b2d"], b["scale"], b["shift"], b["M"], b["Kd"], b["dests"], relu=b["relu"])

    def audit_pool_slice(self, b, y):
        a = b["a"]
        k, s, p = (self.ops._pair(b[f]) for f in ("k", "s", "p"))
        kind = ("avg" if b["count_include_pad"] else "avg_excl") if b["avg"] else "max"
        geom = "pool_slice %s N%d %dx%dx%d C%d k%dx%d s%dx%d p%dx%d %s" % (kind, a.N, a.T, a.H, a.W, a.C, k[0], k[1], s[0], s[1],
                                                                       p[0], p[1], "ceil" if b["ceil_mode"] else "floor")
        return geom, check_pool_slice(a.data, a.N, a.T, a.H, a.W, a.C, k, s, p, b["avg"], y.data,
                                      count_include_pad=b["count_include_pad"], ceil_mode=b["ceil_mode"])

    def audit_gemm_preact(self, b, d):
        self.report.ref_flops += 2 * 2.0 * b["M"] * b["N"] * b["Kd"]
        geom = "gemm_preact M%d N%d K%d lda%d" % (b["M"], b["N"], b["Kd"], b["a2d"].stride(0))
        return geom, check_gemm_preact(b["a2d"], b["b2d"], b["scale"], b["shift"], b["in_scale"], b["in_shift"], b["M"], b["N"],
                                       b["Kd"], d, relu=b["relu"])

    def audit_bn_relu_avgpool2(self, b, y):
        a = b["a"]
        geom = "bn_relu_avgpool2 N%d %dx%d C%d" % (a.N, a.H, a.W, a.C)
        return geom, check_transition_pool(a.data, a.N, a.H, a.W, a.C, b["scale"], b["shift"], y.data)

    def audit_avgpool_global_affine(self, b, y):
        a = b["a"]
        # the kernel averages every one of the ld columns with the affine of that column
        return ("avgpool_affine N%d S%d C%d" % (a.N, a.positions, a.ld),
                check_head_pool(a.data, a.N, a.positions, a.ld, b["scale"], b["shift"], y))

    def audit_se_excite(self, b, out):
        h = b["h"]
        R, C2 = b["w1"].shape
        return ("se_excite N%d S%d C2 %d R%d C%d" % (h.N, h.positions, C2, R, b["w2"].shape[0]),
                check_se_excite(h.data, h.N, h.positions, C2, b["w1"], b["b1"], b["w2"], b["b2"], b["s3"], b["t3"], *out))


ENTRIES = ("conv", "gemm", "gemm_chain", "gemm_sample_affine", "attention", "maxpool3d", "maxpool2d_ceil", "avgpool_global",
           "shortcut_a", "concat_rows", "relu6_", "dwconv3x3", "ccbn_act", "embed_concat", "rgb_head", "tanh_to_nchw", "conv_slice",
           "gemm_split", "pool_slice", "gemm_preact", "bn_relu_avgpool2", "avgpool_global_affine", "se_excite")


@contextlib.contextmanager
def patched(chain_bitwise=True):
    """Patch ``ops`` (every launching entry and the pack constructors) for the duration of the block; yields the auditor."""
    from pretorched_x_b200 import ops, _lib
    lib = _lib.load()
    lib.b2_launch_count.restype = ctypes.c_uint64
    aud = _Auditor(lib, ops, chain_bitwise)
    names = ENTRIES + tuple(UNAUDITED) + tuple(PASS_THROUGH)
    saved = {n: getattr(ops, n) for n in names}
    aud._orig = saved
    inits = {}
    try:
        for n in names:
            setattr(ops, n, aud.wrap(n, saved[n]))
        for cls, kind in ((ops.PackedConv, "dense"), (ops.PackedGroupedConv, "grouped")):
            orig, init = aud.wrap_init(cls, kind)
            inits[cls] = orig
            cls.__init__ = init
        yield aud
    finally:
        for n, f in saved.items():
            setattr(ops, n, f)
        for cls, orig in inits.items():
            cls.__init__ = orig


def audit(model_fn, chain_bitwise=True):
    """Run ``model_fn()`` (one forward of a freshly built model) under the patch; returns its AuditReport (``output``: what the
    forward returned).  Raises AuditError when the launch counts do not reconcile."""
    with torch.no_grad(), patched(chain_bitwise) as aud:
        torch.cuda.synchronize()
        c0 = aud.lib.b2_launch_count()
        out = model_fn()
        torch.cuda.synchronize()
        rep = aud.report
        rep.launches = aud.lib.b2_launch_count() - c0 - aud.extra
        rep.output = out
    if rep.launches != rep.counted:
        raise AuditError("the forward made %d library launches, the wrapped entries account for %d" % (rep.launches, rep.counted))
    return rep
