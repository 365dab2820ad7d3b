"""fp64 references of the convolution kernels and the elementwise error bound the kernel-matrix tests hold them to
(tests/test_gpu_kernel_matrix.py on the GPU; tests/test_kernel_matrix_cpu.py shows on the CPU that the bound catches faults a
max-relative metric lets through).

Bound, per output element:  |got - ref| <= a * 2^-11 * |ref| + b * A + 2^-24, with
  A = |scale| * sum |x * w| + |shift| + |residual|  over the element's own terms,
  a = 1 for fp16 output (one rounding to fp16), 0 for fp32 output,
  b = 2^-14: the fp32 accumulation inside wgmma is neither IEEE-sequential nor documented, so this allows 2^10 fp32 units
      of roundoff on the sum of magnitudes -- far below what one dropped tap, channel chunk or output row costs.
The generator epilogues (per-sample affine, fused upsample, upsampled / pre-affine residual, second output, input affine) use
the same bound with the magnitude of each epilogue's own terms; see ``epilogue`` below.

The builders take ``device=`` (default the CPU): whole-model audits (tests/model_audit.py) build the same fp64 references on
the GPU, where a CPU reference of a full-batch forward would take hours.
"""
import torch
import torch.nn.functional as F

U_F16 = 2.0 ** -11
B_ACC = 2.0 ** -14
FLOOR = 2.0 ** -24


def conv_ref(x, w, scale, shift, k, s, p, residual=None, relu=False, base=None, device="cpu"):
    """fp64 reference of b2_conv_ndhwc_fprop from exactly the kernel's operands.

    x: [N, T, H, W, C] (C the channel pitch), w: [K, taps, C] (the packed filter), scale / shift: [K]; residual: [M, >= K];
    base: [M, K], the prior contents of an fp32 output with ``accumulate``.  Returns (ref, A), both fp64 [M, K]."""
    x, w = x.double().to(device), w.double().to(device)
    K, C = w.shape[0], x.shape[-1]
    wt = w.reshape(K, k[0], k[1], k[2], C).permute(0, 4, 1, 2, 3)
    xt = x.permute(0, 4, 1, 2, 3)
    acc = F.conv3d(xt, wt, stride=s, padding=p)
    mag = F.conv3d(xt.abs(), wt.abs(), stride=s, padding=p)
    acc = acc.permute(0, 2, 3, 4, 1).reshape(-1, K)
    mag = mag.permute(0, 2, 3, 4, 1).reshape(-1, K)
    sc, sh = scale.double().to(device), shift.double().to(device)
    ref = acc * sc + sh
    A = mag * sc.abs() + sh.abs()
    if residual is not None:
        r = residual[:, :K].double().to(device)
        ref, A = ref + r, A + r.abs()
    if relu:
        ref = ref.clamp_min(0.0)
    if base is not None:
        b = base.double().to(device)
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
    return where_worst_of(got, ref, bound(ref, A, f16))


def worst_ratio_of(got, ref, bnd):
    """``worst_ratio`` against an explicit per-element bound (the pooled stem, the weight gradient and its dot product)."""
    err = (got.double().cpu().reshape(ref.shape) - ref).abs()
    err = torch.where(torch.isfinite(err), err, torch.full_like(err, float("inf")))
    return float((err / bnd).max())


def where_worst_of(got, ref, bnd):
    got = got.double().cpu().reshape(ref.shape)
    err = (got - ref).abs()
    err = torch.where(torch.isfinite(err), err, torch.full_like(err, float("inf")))
    r = (err / bnd).reshape(ref.shape[0], -1)
    i = int(torch.argmax(r))
    m, c = divmod(i, r.shape[1])
    return "row %d col %d: got %r ref %r bound %r" % (m, c, float(got.reshape(r.shape)[m, c]), float(ref.reshape(r.shape)[m, c]),
                                                      float(bnd.reshape(r.shape)[m, c]))


# ---------------------------------------------------------------------------------------------
# generator epilogues (tests/test_gpu_epilogue_matrix.py, tests/test_epilogue_matrix_cpu.py): the accumulator and its magnitude
# come from one of the *_acc functions, the epilogue from ``epilogue`` -- all in fp64 from exactly the operands the kernel reads,
# every element held to the same bound as above.
# ---------------------------------------------------------------------------------------------
def conv_acc(x, w, k, s, p, device="cpu"):
    """sum_{tap,c} x * w and sum |x * w| of a convolution (x [N, T, H, W, C], w [K, taps, C]): fp64 [M, K] each."""
    x, w = x.double().to(device), w.double().to(device)
    K, C = w.shape[0], x.shape[-1]
    wt = w.reshape(K, k[0], k[1], k[2], C).permute(0, 4, 1, 2, 3)
    xt = x.permute(0, 4, 1, 2, 3)
    acc = F.conv3d(xt, wt, stride=s, padding=p).permute(0, 2, 3, 4, 1).reshape(-1, K)
    mag = F.conv3d(xt.abs(), wt.abs(), stride=s, padding=p).permute(0, 2, 3, 4, 1).reshape(-1, K)
    return acc, mag


def gemm_acc(a, b, device="cpu"):
    """A[M][Kd] . B[N][Kd]^T and its magnitude, fp64."""
    a, b = a.double().to(device), b.double().to(device)
    return a @ b.t(), a.abs() @ b.abs().t()


def upconv_acc(x, wph, device="cpu"):
    """conv3x3(nearest_up2(x)) as the kernel computes it: four 2x2 phase convolutions of the LOW-res image x [N, H, W, C]
    (or [N, 1, H, W, C]) with the packed phase filter wph [K, 16, C] read back from the pack.  Output pixel (2h + py, 2w + px)
    reads low-res pixel (h - 1 + py + a, w - 1 + px + b) with tap (2 py + px) * 4 + 2 a + b.  fp64 [N * 2H * 2W, K] each."""
    x = x.double().to(device)
    if x.dim() == 5:
        x = x[:, 0]
    N, H, W, C = x.shape
    wph = wph.double().to(device)
    K = wph.shape[0]
    xp = F.pad(x.permute(0, 3, 1, 2), (1, 1, 1, 1))
    acc = torch.zeros(N, K, 2 * H, 2 * W, dtype=torch.float64, device=device)
    mag = torch.zeros_like(acc)
    for py in (0, 1):
        for px in (0, 1):
            ph = 2 * py + px
            f = wph[:, ph * 4:ph * 4 + 4].reshape(K, 2, 2, C).permute(0, 3, 1, 2)
            src = xp[:, :, py:py + H + 1, px:px + W + 1]
            acc[:, :, py::2, px::2] = F.conv2d(src, f)
            mag[:, :, py::2, px::2] = F.conv2d(src.abs(), f.abs())
    return acc.permute(0, 2, 3, 1).reshape(-1, K), mag.permute(0, 2, 3, 1).reshape(-1, K)


# low-res 3x3 rows (or columns) that fold into tap a of output phase p: p = 0 -> {0}, {1, 2}; p = 1 -> {0, 1}, {2}
UP_FOLD = {(0, 0): (0,), (0, 1): (1, 2), (1, 0): (0, 1), (1, 1): (2,)}


def upconv_fold(w):
    """fp64 fold of a 3x3 filter w [K, Cin, 3, 3] into the phase filter [K, 16, Cin] of b2_pack_upconv3x3_weight, and the sum of
    |w| over the taps each folded weight adds (its rounding scale)."""
    w = w.double().cpu()
    K, Cin = w.shape[:2]
    fold = torch.zeros(K, 16, Cin, dtype=torch.float64)
    mag = torch.zeros_like(fold)
    for py in (0, 1):
        for px in (0, 1):
            for a in (0, 1):
                for b in (0, 1):
                    t = (2 * py + px) * 4 + 2 * a + b
                    for r in UP_FOLD[(py, a)]:
                        for c in UP_FOLD[(px, b)]:
                            fold[:, t] += w[:, :, r, c]
                            mag[:, t] += w[:, :, r, c].abs()
    return fold, mag


def nearest_up2(skip, N, H, W, K, device="cpu"):
    """The first K channels of a low-res skip tensor [N * (H/2) * (W/2)][>= K], nearest-2x upsampled to [N * H * W][K] (fp64)."""
    s = skip[:, :K].double().to(device).reshape(N, H // 2, W // 2, K)
    return s.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2).reshape(-1, K)


def per_row(v, rows, M, K, device="cpu"):
    """Per-sample rows [N][>= K] -> the [M][K] rows the elements use (row m takes sample m // rows); [K] stays [K]."""
    v = v.double().to(device)
    if v.dim() == 1:
        return v[:K]
    return v[:, :K].repeat_interleave(rows, dim=0)[:M]


def epilogue(acc, mag, scale, shift, residual=None, pre=False, relu=False, device="cpu"):
    """Value of an output element before its fp16 rounding, and its magnitude A.  scale / shift: [K] or per-row [M][K] (see
    ``per_row``); residual: fp64 [M][K].  pre: the residual joins before the affine, v = s * (acc + r) + t with
    A = |s| * (sum |xw| + |r|) + |t|; otherwise v = s * acc + t + r with A = |s| * sum |xw| + |t| + |r|."""
    s, t = scale.double().to(device), shift.double().to(device)
    if residual is not None and pre:
        r = residual.double().to(device)
        v, A = s * (acc + r) + t, s.abs() * (mag + r.abs()) + t.abs()
    else:
        v, A = s * acc + t, s.abs() * mag + t.abs()
        if residual is not None:
            r = residual.double().to(device)
            v, A = v + r, A + r.abs()
    if relu:
        v = v.clamp_min(0.0)
    return v, A


def second_output(v, A, scale2, shift2, device="cpu"):
    """y2 = relu(s2 * v + t2) from the first output's value v BEFORE its fp16 rounding: (ref2, A2 = |s2| A + |t2|)."""
    s2, t2 = scale2.double().to(device), shift2.double().to(device)
    return (s2 * v + t2).clamp_min(0.0), s2.abs() * A + t2.abs()


# relative distance to an fp16 rounding midpoint inside which an fp32 FMA followed by a rounding to fp16 may round the other way
MIDPOINT_REL = 2.0 ** -23


def in_affine_operand(x, scale, shift, rows, device="cpu"):
    """The A operand of a convolution with an input affine: x' = fp16(relu(x * s_n + t_n)), x fp16 [M][C], scale / shift fp32
    [N][>= C].  Returns (x', other): x' the fp16 rounding of the fp64 value, ``other`` the magnitude of the neighbouring fp16
    value where the fp64 value lies within MIDPOINT_REL of a rounding midpoint (the kernel's fp32 FMA may land on either side;
    0 elsewhere)."""
    x = x.double().to(device)
    M, C = x.shape
    v = (x * per_row(scale, rows, M, C, device) + per_row(shift, rows, M, C, device)).clamp_min(0.0)
    lo = (v * (1 - MIDPOINT_REL)).half().double()
    hi = (v * (1 + MIDPOINT_REL)).half().double()
    amb = lo != hi
    return v.half().double(), torch.where(amb, torch.maximum(lo.abs(), hi.abs()), torch.zeros_like(v))


def in_affine_acc(x, w, scale, shift, rows, device="cpu"):
    """acc / magnitude of relu(x * s_n + t_n) . w^T (w [K][C]).  An operand that may round either way moves by at most one
    fp16 unit, 2^-10 |x'|: its products enter A with the weight 2^-10 / B_ACC, so the bound B_ACC * A covers the flip."""
    xq, other = in_affine_operand(x, scale, shift, rows, device)
    acc, mag = gemm_acc(xq, w, device)
    if bool((other > 0).any()):
        mag = mag + (2.0 ** -10 / B_ACC) * (other @ w.double().to(device).abs().t())
    return acc, mag


# ---------------------------------------------------------------------------------------------
# non-local attention (tests/test_gpu_kernel_matrix.py, tests/model_audit.py)
# ---------------------------------------------------------------------------------------------
ATT_C = 4.0


def att_ref(q, k, v, B, Nq, Nk, mode):
    """fp64 softmax(Q K^T) V (mode 0), (Q K^T / Nk) V (mode 1) or (relu(Q K^T) / Nk) V (mode 2) of q [B * Nq][d], k [B * Nk][d],
    v [B * Nk][dv], on their device.  Returns (ref [B * Nq][dv], |P| |V| [B][Nq][dv])."""
    q, k, v = (t.double().view(B, -1, t.shape[1]) for t in (q, k, v))
    s = q @ k.transpose(1, 2)
    if mode == 0:
        p = torch.softmax(s, dim=-1)
    else:
        p = (s if mode == 1 else s.clamp_min(0.0)) / Nk
    return (p @ v).reshape(B * Nq, -1), p.abs() @ v.abs()


def att_bound(ref, pv, v, B, Nq, Nk, mode):
    """Per-element bound of the attention output.  Mode 0: a convex combination of the values, with fp16 P and output roundings,
    relative to max_j |v_j| of its sample: ATT_C 2^-11 max_j |v_j|.  Modes 1 / 2: 2^-11 |ref| + ATT_C 2^-11 |P| |V|.  Plus the
    floor 2^-24."""
    dv = ref.shape[1]
    if mode == 0:
        vmax = v.double().abs().view(B, Nk, dv).amax(dim=1)
        bnd = ATT_C * U_F16 * vmax.repeat_interleave(Nq, dim=0)
    else:
        bnd = U_F16 * ref.abs() + ATT_C * U_F16 * pv.reshape(B * Nq, dv)
    return bnd + FLOOR


# ---------------------------------------------------------------------------------------------
# squeeze-and-excitation (tests/test_gpu_senet.py, tests/model_audit.py)
# ---------------------------------------------------------------------------------------------
def excite_mean(h, N, S, C2, device="cpu"):
    """Per-sample channel means of h (fp16 [N * S][>= C2]) and of |h|: fp64 [N][C2] each."""
    hd = h[:, :C2].double().to(device).reshape(N, S, C2)
    return hd.mean(1), hd.abs().mean(1)


def excite_ref(m, habs, w1, b1, w2, b2, s3, t3):
    """fp64 excitation from the operands b2_se_excite reads: the means ``m`` (and mean |h|, ``habs``) of ``excite_mean``, fc1
    folded through conv3 + bn3 (w1 [R][C2], b1 [R]), fc2 (w2 [C][R], b2 [C]) and the bn3 affine (s3, t3 [C]).  Returns the dict
    ``excite_bound`` reads: m, habs, a = relu(fc1), e = sigmoid(fc2), scale = e s3, shift = e t3."""
    dev = m.device
    w1, b1, w2, b2, s3, t3 = (t.double().to(dev) for t in (w1, b1, w2, b2, s3, t3))
    a = (m @ w1.t() + b1).clamp_min(0)
    e = torch.sigmoid(a @ w2.t() + b2)
    return dict(m=m, habs=habs, a=a, e=e, scale=e * s3, shift=e * t3)


def excite_bound(r, w1, b1, w2, b2, s3, t3, S, fold_rounding=False):
    """Per-element bound of (scale, shift), from fp32 roundoff (u = 2^-24) stage by stage, r the dict of ``excite_ref``:
      mean   |dm| <= (S + 34) u mean|h|          (stripe sums of <= ceil(S/32) terms, 32-term stripe sum, one division)
      fc1    |da| <= (C2 + 1) u (sum |w1| |m| + |b1|) + sum |w1| |dm|    (one fmaf chain and the bias)
      fc2    |dv| <= (R + 1) u (sum |w2| |a| + |b2|) + sum |w2| |da|
      sigmoid |de| <= |dv| / 4 + 2^-19        (Lipschitz 1/4; the fast-math exp and reciprocal)
      output |d(e s)| <= |s| |de| + u |e s|
    ``fold_rounding``: r was computed from the unfolded fp64 weights, so fc1 also carries the fp32 rounding of the fold
    w1 = W_fc1 diag(s3) W3, b1 = W_fc1 t3 + b_fc1: (C2 + 2) u."""
    dev = r["m"].device
    w1a, b1a, w2a, b2a = (t.double().to(dev).abs() for t in (w1, b1, w2, b2))
    s3d, t3d = s3.double().to(dev), t3.double().to(dev)
    C2, R = w1a.shape[1], w1a.shape[0]
    dm = (S + 34) * FLOOR * r["habs"]
    da = (C2 + 1 + int(fold_rounding)) * FLOOR * (r["m"].abs() @ w1a.t() + b1a) + dm @ w1a.t()
    dv = (R + 1) * FLOOR * (r["a"].abs() @ w2a.t() + b2a) + da @ w2a.t()
    de = dv / 4 + 2.0 ** -19
    return de * s3d.abs() + FLOOR * r["scale"].abs(), de * t3d.abs() + FLOOR * r["shift"].abs()


# ---------------------------------------------------------------------------------------------
# stem convolution with the fused W max-pool, depthwise 3x3, weight gradient (tests/test_gpu_kernel_bounds.py,
# tests/test_kernel_bounds_cpu.py): fp64 from exactly the operands each kernel reads.
# ---------------------------------------------------------------------------------------------
def stem_operands(x, weight):
    """The stem's operands: x fp32/fp16 NCDHW [N, 3, T, H, W] -> fp16 NDHWC4 [N, T, H, W, 4] with channel 3 zero; the filter
    weight [K, 3, kt, kh, kw] -> weight.half() (pack_weight_stem7_kernel rounds each weight with __float2half_rn; the BN affine
    is applied afterwards, in the fp32 epilogue) as the [K, taps, 4] layout conv_ref reads, zero in channel 3."""
    x = x.detach().cpu()
    N, Cin, T, H, W = x.shape
    x4 = torch.zeros(N, T, H, W, 4, dtype=torch.float16)
    x4[..., :Cin] = x.half().permute(0, 2, 3, 4, 1)
    w = weight.detach().cpu().half()
    K, taps = w.shape[0], w.shape[2] * w.shape[3] * w.shape[4]
    w4 = torch.zeros(K, taps, 4, dtype=torch.float16)
    w4[..., :Cin] = w.permute(0, 2, 3, 4, 1).reshape(K, taps, Cin)
    return x4, w4


def pool_w(ref, A, Wo, f16=True):
    """The stem's fused max-pool along W (k 3, stride 2, padding 1) of a ReLU'd fp64 result ref [rows * Wo, K] (rows = N To Ho)
    with its bound.  Reference: the max over each window; bound: the largest per-element bound in the window -- the max is
    1-Lipschitz in the inf-norm and fp16 rounding is monotone, so |max got - max ref| <= max |got - ref|.  Returns
    (ref, bound), fp64 [rows * Wp, K] with Wp = (Wo - 1) // 2 + 1."""
    K = ref.shape[1]

    def pool(v):
        v = v.reshape(-1, Wo, K).permute(0, 2, 1)
        return F.max_pool1d(v, 3, 2, 1).permute(0, 2, 1).reshape(-1, K)
    return pool(ref), pool(bound(ref, A, f16))


def dw_ref(x, w9, scale, shift, stride, clamp_in, relu6, device="cpu"):
    """fp64 reference of b2_dwconv3x3_ndhwc (padding 1): x fp16 [B, H, W, C] (the C used channels), w9 fp32 [9][C] (tap
    kh * 3 + kw), scale / shift fp32 [C].  The kernel reads min(x, 6) with clamp_in (exact in fp16).  A = |s| sum |x w| + |t|;
    the ReLU6 clamp comes after the bound is formed (1-Lipschitz).  Returns (ref, A), fp64 [B * Ho * Wo, C]."""
    x = x.double().to(device)
    if clamp_in:
        x = x.clamp(max=6.0)
    C = x.shape[-1]
    xt = x.permute(0, 3, 1, 2)
    wt = w9.double().to(device).t().reshape(C, 1, 3, 3)
    acc = F.conv2d(xt, wt, stride=stride, padding=1, groups=C).permute(0, 2, 3, 1).reshape(-1, C)
    mag = F.conv2d(xt.abs(), wt.abs(), stride=stride, padding=1, groups=C).permute(0, 2, 3, 1).reshape(-1, C)
    s, t = scale.double().to(device), shift.double().to(device)
    ref, A = acc * s + t, mag * s.abs() + t.abs()
    if relu6:
        ref = ref.clamp(0.0, 6.0)
    return ref, A


def wgrad_ref(x, g, k, stride, pad, scale=None, inv=None):
    """fp64 weight gradient of b2_conv_wgrad_thw from its fp16 operands x [N, Cin, T, H, W] and g [N, Cout, To, Ho, Wo]:
    G = conv3d_weight(x, g), M = conv3d_weight(|x|, |g|), dW = scale * inv * G, A = |scale| * inv * M.
    Returns (G, M, dW, A), fp64 [Cout, Cin, kt, kh, kw]."""
    x, g = x.double(), g.double().to(x.device)
    shape = (g.shape[1], x.shape[1]) + tuple(k)
    G = torch.nn.grad.conv3d_weight(x, shape, g, stride=stride, padding=pad)
    M = torch.nn.grad.conv3d_weight(x.abs(), shape, g.abs(), stride=stride, padding=pad)
    s = scale.double().to(x.device).view(-1, 1, 1, 1, 1) if scale is not None else torch.ones(1, dtype=torch.float64, device=x.device)
    i = float(inv) if inv is not None else 1.0
    return G, M, s * i * G, s.abs() * i * M


def wgrad_b(nbox, splits):
    """Accumulation coefficient of the fp32 weight gradient: one split sums 64 positions of each of its ceil(nbox / splits)
    position blocks, then the reduce kernel adds the splits in order and applies inv and scale (2 roundings)."""
    L = 64 * -(-nbox // splits)
    return max(B_ACC, (L + splits + 2) * FLOOR)


def wgrad_bound(A, nbox, splits, floor=FLOOR):
    """Per-element bound of dW (fp32 output: no output-rounding term)."""
    return wgrad_b(nbox, splits) * A + floor


def wdot_ref(G, M, w, inv, nbox, splits, floor=FLOOR):
    """wdot[co] = inv * sum w G and its bound: the error of each inv * G element (b M) weighted by |w|, the reduce kernel's fp32
    dot product chain (strided per-thread sum over ceil(n / 256) terms, a 5-level shuffle, 8 warp sums) on inv sum |w| |G|,
    and the floor; n = Cin * taps.  Returns (ref, bound), fp64 [Cout]."""
    Cout = G.shape[0]
    i = float(inv) if inv is not None else 1.0
    w = w.double().to(G.device).reshape(Cout, -1)
    G, M = G.reshape(Cout, -1), M.reshape(Cout, -1)
    n = G.shape[1]
    ref = i * (w * G).sum(1)
    bnd = (i * (w.abs() * (wgrad_b(nbox, splits) * M)).sum(1)
           + (-(-n // 256) + 5 + 8) * FLOOR * i * (w.abs() * G.abs()).sum(1) + floor)
    return ref, bnd


# ---------------------------------------------------------------------------------------------
# fine-tuning backward (tests/test_gpu_finetune_bounds.py on the GPU, tests/test_finetune_bounds_cpu.py on the CPU): the head's
# gradient products, the pool hand-off and every stage of engine.block_backward, each in fp64 from the true operands.
#
# Bound of a gradient element, in the units it is stored in (the trunk's gradients carry the loss scale, the parameter
# gradients do not):  a * 2^-11 |ref| + 2^-14 A + R + floor, with
#   a, 2^-14 A   as above (a = 1 for fp16 output, 0 for fp32);
#   R            the rounding of every operand the function under test rounds to fp16 itself, element by element:
#                |fp16(v) - v| <= max(2^-11 |v|, 2^-25) for |v| < 65504 (2^-25 is half of fp16's subnormal quantum 2^-24), so
#                R = sum_j max(2^-11 |u_j|, 2^-25 / s) |v_j| for a rounded operand u multiplied by 2^s before the cast (s = 1
#                without a scale) and the other operand v.  Operands that arrive in fp16 (activations, incoming gradients)
#                enter exactly and carry no R;
#   floor        the fp16 quantum at the scale in use: 2^-24 / s (per row where the scale is per row), i.e. 2^-24 for a gradient
#                stored with the loss scale.  Elements more than ~2^-31 below their row's peak may be flushed, none above.
# ---------------------------------------------------------------------------------------------
SUB_F16 = 2.0 ** -25


def r16(v, scale=None):
    """Bound on |fp16(v * scale) / scale - v|, element by element (fp64): max(2^-11 |v|, 2^-25 / scale); scale broadcasts
    against v (a power of two per row, or None for an unscaled cast)."""
    v = v.double()
    q = SUB_F16 if scale is None else SUB_F16 / scale.double()
    return torch.maximum(U_F16 * v.abs(), torch.as_tensor(q, dtype=torch.float64, device=v.device))


def row_scale(g, dim):
    """The power of two that puts the peak of each row (dim = 1) or column (dim = 0) of an fp32 gradient in [2^7, 2^8) (the
    target of b2_loss_scale_f32), 1 for an all-zero row.  fp64, the reduced dimension kept."""
    amax = g.double().abs().amax(dim, keepdim=True)
    _, e = torch.frexp(amax)
    k = torch.where(amax > 0, 8 - e, torch.zeros_like(e)).clamp(-126, 126)
    return torch.pow(2.0, k.double())


def head_ref(gy, w, x16, relu_mask=None):
    """LinearFunction's two gradient products against the true gradients, from the fp32 logit gradient gy [B][C], the fp32 weight
    w [C][F] and the fp16 input x16 [B][F] the forward saved:
      dX = gy w (times relu_mask), A = |gy| |w|; gy is rounded with a power of two per sample row s_b (``row_scale``) and w is
      rounded unscaled inside the backward: R = max(2^-11 |gy|, 2^-25 / s_b) |w| + |gy| max(2^-11 |w|, 2^-25); floor 2^-24 / s_b;
      dW = gy^T x16, A = |gy^T| |x16|; gy^T is rounded with a power of two per class row s_c: R = max(2^-11 |gy^T|, 2^-25 / s_c)
      |x16|; floor 2^-24 / s_c.
    Both outputs are fp32 (no output-rounding term).  Returns (dx, dx bound, dw, dw bound), fp64."""
    g, w, x = gy.double(), w.double(), x16.double()
    sb, sc = row_scale(g, 1), row_scale(g.t(), 1)
    dx = g @ w
    bx = B_ACC * (g.abs() @ w.abs()) + r16(g, sb) @ w.abs() + g.abs() @ r16(w) + FLOOR / sb
    if relu_mask is not None:
        dx = dx * relu_mask.double()
    gt = g.t()
    dw = gt @ x
    bw = B_ACC * (gt.abs() @ x.abs()) + r16(gt, sc) @ x.abs() + FLOOR / sc
    return dx, bx, dw, bw


def bias_grad_bound(gy):
    """torch's fp32 column sum of gy [B][C]: any summation order of B terms errs by at most (B - 1) 2^-24 sum |g|."""
    g = gy.double()
    return g.sum(0), max(g.shape[0] - 1, 1) * FLOOR * g.abs().sum(0) + FLOOR * 2.0 ** -30


def pool_backward_ref(gf, y_out, scale, S):
    """FineTunePoolFunction.backward: fp16(gf[n] * (scale / S)) where the block output y_out [N * S][C] is positive.  The kernel
    forms scale / S and the product in fp32 (two roundings, 2^-23 |ref|) and rounds once to fp16.  Returns (ref, bound)."""
    ref = gf.double().repeat_interleave(S, dim=0) * (float(scale) / S)
    ref = torch.where(y_out.double() > 0, ref, torch.zeros_like(ref))
    return ref, (U_F16 + 2.0 ** -23) * ref.abs() + FLOOR


def ncdhw(m, N, T, H, W):
    """[N*T*H*W][C] rows (fp64) -> NCDHW."""
    return m.double().reshape(N, T, H, W, -1).permute(0, 4, 1, 2, 3)


def rows_of(t):
    """NCDHW -> [N*T*H*W][C] rows."""
    return t.permute(0, 2, 3, 4, 1).reshape(-1, t.shape[1])


def zero_insert_ref(g, size, stride, channels=None):
    """Adjoint of the type-A / strided subsampling (NCDHW, fp64): g at every ``stride``-th pixel of ``size``, its first ``channels``
    channels, zeros elsewhere."""
    N, C = g.shape[0], g.shape[1] if channels is None else channels
    y = g.new_zeros((N, C) + tuple(size))
    y[:, :, ::stride, ::stride, ::stride] = g[:, :C]
    return y


def folded(w, s):
    """The BN-scaled filter s[co] * w[co] of a dgrad, formed in fp32 exactly as the engine forms it, as fp64."""
    w = w.detach().float()
    return (w * s.detach().float().to(w.device).view((-1,) + (1,) * (w.dim() - 1))).double()


def folded_operand(w, s, pack):
    """The dgrad's filter operand: with ``pack`` the fp16 rounding of the fp32 s W (what the engine packs, held to it bit for bit by
    the derived-filter test), R = 0; without, the fp32 s W itself, whose rounding inside the backward R carries."""
    f = folded(w, s)
    return (f.half().double(), torch.zeros_like(f)) if pack else (f, r16(f))


def dgrad_1x1(g, w, s, mask=None, residual=None, second=None, pack=True):
    """Input gradient of a 1x1(x1) convolution followed by eval BN: g [M][Cout] (fp16, loss-scaled) . (s W) [Cout][Cin]
    (+ residual [M][Cin]) (+ second = (g2, w2, s2), another such product), zeroed where mask [M][Cin] <= 0.  ``pack``: see
    ``folded_operand``.  Returns (ref, A, R), fp64 [M][Cin]."""
    terms = [(g, w, s)] + ([second] if second is not None else [])
    ref = A = R = 0
    for gg, ww, ss in terms:
        gg = gg.double()
        f, rf = (t.reshape(ww.shape[0], -1).to(gg.device) for t in folded_operand(ww, ss, pack))                   # [Cout][Cin]
        ref, A, R = ref + gg @ f, A + gg.abs() @ f.abs(), R + gg.abs() @ rf
    if residual is not None:
        r = residual.double()
        ref, A = ref + r, A + r.abs()
    if mask is not None:
        ref = torch.where(mask > 0, ref, torch.zeros_like(ref))
    return ref, A, R


def dgrad_3x3(z, w, s, mask=None, residual=None, pack=True):
    """Input gradient of a 3x3x3 (or 2-D 3x3, as 1x3x3) convolution followed by eval BN, as the stride-1 convolution of the
    zero-inserted gradient z (NCDHW fp16 values, loss-scaled) with the flipped, transposed, s-folded filter, padding k // 2.
    (+ residual, NCDHW), zeroed where mask (NCDHW) <= 0.  ``pack``: see ``folded_operand``.  Returns (ref, A, R) as [rows][Cin],
    fp64."""
    f, rf = (t.to(z.device) for t in folded_operand(w, s, pack))
    if f.dim() == 4:
        f, rf = f.unsqueeze(2), rf.unsqueeze(2)
    pad = tuple(k // 2 for k in f.shape[2:])
    ft, rt = f.flip(2, 3, 4).transpose(0, 1), rf.flip(2, 3, 4).transpose(0, 1)
    z = z.double()
    ref = rows_of(F.conv3d(z, ft, padding=pad))
    A = rows_of(F.conv3d(z.abs(), ft.abs(), padding=pad))
    R = rows_of(F.conv3d(z.abs(), rt, padding=pad))
    if residual is not None:
        r = rows_of(residual.double())
        ref, A = ref + r, A + r.abs()
    if mask is not None:
        ref = torch.where(rows_of(mask) > 0, ref, torch.zeros_like(ref))
    return ref, A, R


def grad_bound(ref, A, R):
    """Bound of an fp16 loss-scaled gradient (floor: fp16's quantum in the scaled units)."""
    return bound(ref, A, True) + R


def colsum_bound(g, inv):
    """dbeta = inv * column sums of the fp16 gradient g [rows][C] (b2_colsum_f16, the chain of its two fixed-order passes) and its
    bound, floor 2^-24 * inv (fp16's quantum of g, unscaled).  Returns (ref, bound), fp64 [C]."""
    g = g.double()
    chain = g.shape[0] / (128 * 8) + 8 + 128 + 2
    return inv * g.sum(0), chain * FLOOR * inv * g.abs().sum(0) + FLOOR * inv


def dgamma_ref(wdot, wdot_bnd, dbeta, dbeta_bnd, mean, var, eps):
    """dgamma = (wdot - mean * dbeta) * rsqrt(var + eps), two fp32 torch ops on top of the kernels' results.  The bound carries
    the cancellation term r (bnd(wdot) + |mean| bnd(dbeta)) and the fp32 roundings of the product mean * dbeta, the difference,
    var + eps, rsqrt (<= 2 ulp) and the last product, 7.5 units of 2^-24 at most: 2^-21 r (|wdot| + |mean dbeta|).
    mean / var: the fp32 running statistics.  Returns (ref, bound), fp64 [C]."""
    mean, var = mean.double().to(wdot.device), var.float().double().to(wdot.device)
    r = 1.0 / torch.sqrt(var + float(torch.tensor(eps, dtype=torch.float32)))
    ref = (wdot - mean * dbeta) * r
    return ref, r * (wdot_bnd + mean.abs() * dbeta_bnd) + 2.0 ** -21 * r * (wdot.abs() + (mean * dbeta).abs()) + FLOOR * 2.0 ** -30
