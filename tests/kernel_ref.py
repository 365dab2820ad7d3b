"""fp64 references of the convolution kernels and the elementwise error bound the kernel-matrix tests hold them to
(tests/test_gpu_kernel_matrix.py on the GPU; tests/test_kernel_matrix_cpu.py shows on the CPU that the bound catches faults a
max-relative metric lets through).

Bound, per output element:  |got - ref| <= a * 2^-11 * |ref| + b * A + 2^-24, with
  A = |scale| * sum |x * w| + |shift| + |residual|  over the element's own terms,
  a = 1 for fp16 output (one rounding to fp16), 0 for fp32 output,
  b = 2^-14: the fp32 accumulation inside wgmma is neither IEEE-sequential nor documented, so this allows 2^10 fp32 units
      of roundoff on the sum of magnitudes -- far below what one dropped tap, channel chunk or output row costs.
"""
import torch
import torch.nn.functional as F

U_F16 = 2.0 ** -11
B_ACC = 2.0 ** -14
FLOOR = 2.0 ** -24


def conv_ref(x, w, scale, shift, k, s, p, residual=None, relu=False, base=None):
    """fp64 reference of b2_conv_ndhwc_fprop from exactly the kernel's operands.

    x: [N, T, H, W, C] (C the channel pitch), w: [K, taps, C] (the packed filter), scale / shift: [K]; residual: [M, >= K];
    base: [M, K], the prior contents of an fp32 output with ``accumulate``.  Returns (ref, A), both fp64 [M, K]."""
    x, w = x.double().cpu(), w.double().cpu()
    K, C = w.shape[0], x.shape[-1]
    wt = w.reshape(K, k[0], k[1], k[2], C).permute(0, 4, 1, 2, 3)
    xt = x.permute(0, 4, 1, 2, 3)
    acc = F.conv3d(xt, wt, stride=s, padding=p)
    mag = F.conv3d(xt.abs(), wt.abs(), stride=s, padding=p)
    acc = acc.permute(0, 2, 3, 4, 1).reshape(-1, K)
    mag = mag.permute(0, 2, 3, 4, 1).reshape(-1, K)
    sc, sh = scale.double().cpu(), shift.double().cpu()
    ref = acc * sc + sh
    A = mag * sc.abs() + sh.abs()
    if residual is not None:
        r = residual[:, :K].double().cpu()
        ref, A = ref + r, A + r.abs()
    if relu:
        ref = ref.clamp_min(0.0)
    if base is not None:
        b = base.double().cpu()
        ref, A = ref + b, A + b.abs()
    return ref, A


def bound(ref, A, f16):
    return (U_F16 if f16 else 0.0) * ref.abs() + B_ACC * A + FLOOR


def worst_ratio(got, ref, A, f16):
    """max over elements of |got - ref| / bound; a NaN or inf in ``got`` counts as an infinite ratio."""
    err = (got.double().cpu() - ref).abs()
    err = torch.where(torch.isfinite(err), err, torch.full_like(err, float("inf")))
    return float((err / bound(ref, A, f16)).max())


def where_worst(got, ref, A, f16):
    err = (got.double().cpu() - ref).abs()
    err = torch.where(torch.isfinite(err), err, torch.full_like(err, float("inf")))
    r = err / bound(ref, A, f16)
    i = int(torch.argmax(r))
    m, c = divmod(i, ref.shape[1])
    return "row %d col %d: got %r ref %r A %r" % (m, c, float(got.reshape(ref.shape)[m, c]), float(ref[m, c]), float(A[m, c]))
