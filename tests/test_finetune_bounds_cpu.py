"""CPU: the fp64 references and bounds of the fine-tuning backward (tests/kernel_ref.py, used by tests/test_gpu_finetune_bounds.py)
pass the exact result rounded once, and each fault below fails them.  For every fault the per-tensor metric of the block-level
GPU tests (max |err| / max |ref| <= 2e-2 and cosine >= 0.9995) is evaluated too; ``OLD`` records whether it notices.

The faults are simulated on the CPU with the operands the kernels read (fp16 values, fp32 products): no GPU is involved."""
import pytest
import torch
import torch.nn.functional as F

from tests.kernel_ref import (FLOOR, bias_grad_bound, colsum_bound, dgamma_ref, dgrad_1x1, dgrad_3x3, grad_bound, head_ref,
                              ncdhw, row_scale, rows_of, wdot_ref, wgrad_bound, wgrad_ref, worst_ratio_of, zero_insert_ref)

# does the block tests' per-tensor metric (2e-2 of max |ref|, cosine 0.9995) catch the fault, on the operands below?  It misses
# the head faults, which live in the small elements of a tensor; the block-stage faults here move elements near the peak.
OLD = {
    "unscaled_head_cast_dw": False,
    "unscaled_head_cast_dx": False,
    "unflipped_filter": True,
    "untransposed_filter": True,
    "h1_mask_for_g2": True,
    "dgamma_without_mean": True,
    "odd_border_zero_insert": True,
    "type_a_wrong_channel_block": True,
    "pg_added_before_rounding": True,
    "inv_applied_twice": True,
}


def old_metric_catches(got, ref):
    got, ref = got.double().reshape(-1), ref.double().reshape(-1)
    rel = float((got - ref).abs().max()) / max(float(ref.abs().max()), 1e-30)
    cos = float(F.cosine_similarity(got, ref, dim=0))
    return not (rel <= 2e-2 and cos >= 0.9995)


def f16(t):
    return t.half().double()


def f32(t):
    return t.float().double()


def fault(name, got, ref, bnd):
    r = worst_ratio_of(got, ref, bnd)
    old = old_metric_catches(got, ref)
    print("[finetune-bounds-cpu] %-28s err/bound %10.3f  old metric catches it: %s" % (name, r, old))
    assert r > 1.0, "%s: the bound does not see the fault (%.3f)" % (name, r)
    assert old == OLD[name], "%s: the per-tensor metric %s it" % (name, "catches" if old else "misses")


def passes(name, got, ref, bnd):
    r = worst_ratio_of(got, ref, bnd)
    print("[finetune-bounds-cpu] %-28s err/bound %10.3f" % (name, r))
    assert r <= 1.0, name


# ---------------------------------------------------------------------------------------------
# head: LinearFunction's gradient products
# ---------------------------------------------------------------------------------------------
def head_problem(B, C, temp, mult, seed, Fdim=256):
    """Cross-entropy logit gradient (p - onehot) * temp / B * mult of a random head, with the operands the backward reads."""
    g = torch.Generator().manual_seed(seed)
    x16 = torch.randn(B, Fdim, generator=g).relu().half()
    w = torch.randn(C, Fdim, generator=g) / Fdim ** 0.5
    logits = (x16.float() @ w.t()) * temp
    t = torch.randint(0, C, (B,), generator=g)
    gy = ((torch.softmax(logits.double(), 1) - F.one_hot(t, C).double()) * temp / B * mult).float()
    return gy, w, x16


def head_products(gy, w, x16, scaled):
    """dX and dW as LinearFunction forms them: gy (per-row power of two when ``scaled``) and w rounded to fp16, exact products
    rounded once to fp32."""
    sb = row_scale(gy, 1) if scaled else 1.0
    sc = row_scale(gy.t(), 1) if scaled else 1.0
    g = gy.double()
    dx = f32((f16(g * sb) / sb) @ f16(w.double()))
    dw = f32((f16(g.t() * sc) / sc) @ x16.double())
    return dx, dw


HEAD_CASES = [(256, 1000, 1.0, 1.0), (256, 339, 8.0, 1.0), (32, 400, 1.0, 1e-3), (3, 7, 8.0, 1.0)]


@pytest.mark.parametrize("B,C,temp,mult", HEAD_CASES)
def test_head_reference_passes_the_scaled_cast(B, C, temp, mult):
    gy, w, x16 = head_problem(B, C, temp, mult, B + C)
    dx_ref, bx, dw_ref, bw = head_ref(gy, w, x16)
    dx, dw = head_products(gy, w, x16, scaled=True)
    passes("head dX B%d C%d" % (B, C), dx, dx_ref, bx)
    passes("head dW B%d C%d" % (B, C), dw, dw_ref, bw)
    db_ref, bb = bias_grad_bound(gy)
    passes("head db B%d C%d" % (B, C), f32(gy.double().sum(0)), db_ref, bb)


def test_unscaled_head_cast_fails():
    """The fp32 logit gradient cast to fp16 as it is (the head's backward before the per-row scale).  A peaked softmax at
    B = 256 puts most entries of an improbable class's row of g^T below fp16's smallest subnormal: they flush to zero and dW
    loses that class.  A near-uniform softmax at B = 32 with the loss times 1e-3 leaves every entry but the target's in fp16's
    subnormal range, where the rounding error is a large part of each value: dX of every sample."""
    gy, w, x16 = head_problem(256, 339, 8.0, 1.0, 7)
    _, _, dw_ref, bw = head_ref(gy, w, x16)
    fault("unscaled_head_cast_dw", head_products(gy, w, x16, scaled=False)[1], dw_ref, bw)
    gy, w, x16 = head_problem(32, 400, 1.0, 1e-3, 8)
    dx_ref, bx, _, _ = head_ref(gy, w, x16)
    fault("unscaled_head_cast_dx", head_products(gy, w, x16, scaled=False)[0], dx_ref, bx)


# ---------------------------------------------------------------------------------------------
# block stages
# ---------------------------------------------------------------------------------------------
def gen(seed):
    return torch.Generator().manual_seed(seed)


def act16(shape, g, relu=False, scale=1.0):
    t = torch.randn(shape, generator=g) * scale
    return (t.relu() if relu else t).half()


def conv_problem(seed, N=2, C=16, K=16, size=(3, 7, 7)):
    g = gen(seed)
    gy = act16((N, K) + size, g)
    w = torch.randn(K, C, 3, 3, 3, generator=g) / (27 * C) ** 0.5
    s = torch.rand(K, generator=g) + 0.5
    mask = act16((N, C) + size, g)
    return gy, w, s, mask


def masked_conv16(z, f, mask, residual=None):
    """fp16(conv(z, f) (+ residual)) zeroed where mask <= 0: the kernel's exact result rounded once."""
    out = F.conv3d(z.double(), f, padding=1)
    if residual is not None:
        out = out + residual.double()
    return rows_of(f16(out * (mask > 0)))


def w16_folded(w, s):
    return f16(w.float() * s.float().view(-1, 1, 1, 1, 1))


def test_dgrad_3x3_reference_passes_and_bad_filters_fail():
    gy, w, s, mask = conv_problem(1)
    wf = w16_folded(w, s)
    ref, A, R = dgrad_3x3(gy, w, s, mask=mask, pack=False)
    passes("dgrad 3x3, fp32 sW + R", masked_conv16(gy, wf.flip(2, 3, 4).transpose(0, 1), mask), ref, grad_bound(ref, A, R))
    ref, A, R = dgrad_3x3(gy, w, s, mask=mask)
    bnd = grad_bound(ref, A, R)
    passes("dgrad 3x3", masked_conv16(gy, wf.flip(2, 3, 4).transpose(0, 1), mask), ref, bnd)
    fault("unflipped_filter", masked_conv16(gy, wf.transpose(0, 1), mask), ref, bnd)
    fault("untransposed_filter", masked_conv16(gy, wf.flip(2, 3, 4), mask), ref, bnd)


def test_g2_with_the_h1_mask_fails():
    g = gen(2)
    M, Cout, Cin = 300, 64, 16
    gy, h1, h2 = act16((M, Cout), g), act16((M, Cin), g, relu=True), act16((M, Cin), g, relu=True)
    w, s = torch.randn(Cout, Cin, 1, 1, 1, generator=g) * 0.1, torch.rand(Cout, generator=g) + 0.5
    ref, A, R = dgrad_1x1(gy, w, s, mask=h2)
    bnd = grad_bound(ref, A, R)
    prod = gy.double() @ w16_folded(w, s).reshape(Cout, Cin)
    passes("g2", f16(prod * (h2 > 0)), ref, bnd)
    fault("h1_mask_for_g2", f16(prod * (h1 > 0)), ref, bnd)


def test_small_bn_scale_channel_and_inv_paths():
    """A BN scale of 1e-3 folds weights into fp16's subnormal range; its rounding is carried by R.  ``inv`` applied twice
    (once in the kernel, once more) fails the weight and beta gradients."""
    g = gen(3)
    M, Cout, Cin = 200, 32, 24
    gy = act16((M, Cout), g)
    w = torch.randn(Cout, Cin, 1, 1, 1, generator=g) * 0.03
    s = torch.rand(Cout, generator=g) + 0.5
    s[:4] = 1e-3
    got = f16(gy.double() @ w16_folded(w, s).reshape(Cout, Cin))
    for pack in (True, False):
        ref, A, R = dgrad_1x1(gy, w, s, pack=pack)
        passes("g small scale%s" % ("" if pack else ", fp32 sW + R"), got, ref, grad_bound(ref, A, R))

    inv = 2.0 ** 10                                              # loss scale 2^-10
    x = act16((2, Cin, 2, 10, 10), g, relu=True)
    gg = act16((2, Cout, 2, 10, 10), g)
    G, Mg, dw_ref, Aw = wgrad_ref(x, gg, (1, 1, 1), (1, 1, 1), (0, 0, 0), s, inv)
    bw = wgrad_bound(Aw, 8, 1, floor=FLOOR * inv)
    passes("dW inv", f32(dw_ref), dw_ref, bw)
    fault("inv_applied_twice", f32(dw_ref * inv), dw_ref, bw)
    db_ref, bb = colsum_bound(rows_of(gg.double()), inv)
    passes("dbeta inv", f32(db_ref), db_ref, bb)


def test_dgamma_needs_the_running_mean_term():
    g = gen(4)
    Cout, Cin = 32, 24
    x = act16((2, Cin, 2, 9, 9), g, relu=True)
    gg = act16((2, Cout, 2, 9, 9), g)
    w = torch.randn(Cout, Cin, 1, 1, 1, generator=g) * 0.05
    mean = torch.randn(Cout, generator=g) * 0.1
    mean[:8] += 40.0                                             # |running_mean| >> spread of the convolution output
    var = torch.rand(Cout, generator=g) + 0.5
    inv = 2.0 ** -6
    G, Mg, _, _ = wgrad_ref(x, gg, (1, 1, 1), (1, 1, 1), (0, 0, 0), None, inv)
    wd, wb = wdot_ref(G, Mg, w, inv, 6, 1, floor=FLOOR * inv)
    db, bb = colsum_bound(rows_of(gg.double()), inv)
    ref, bnd = dgamma_ref(wd, wb, db, bb, mean, var, 1e-5)
    r = 1.0 / torch.sqrt(var.double() + 1e-5)
    passes("dgamma", f32(f32(f32(wd) - f32(mean.double() * f32(db))) * f32(r)), ref, bnd)
    fault("dgamma_without_mean", f32(f32(wd) * f32(r)), ref, bnd)


def stride2_problem(seed, cancel):
    """Type-B shortcut at stride 2 on an odd-sized input (3, 7, 9): pg = fp16(gy . (sd Wd)) at low resolution, zero-inserted as the
    residual of dx = [x > 0] (g1 . (s1 W1) + residual).  ``cancel``: positive operands, and g1 = -0.996 gy at the kept pixels with
    W1 = Wd, so that the main path cancels the shortcut to 2^-8 of it (where the residual's own rounding shows)."""
    g = gen(seed)
    N, C, Cin, size = 2, 32, 16, (3, 7, 9)
    lo = tuple((n - 1) // 2 + 1 for n in size)
    gy = act16((N, C) + lo, g)
    wd = torch.randn(C, Cin, 1, 1, 1, generator=g) * 0.1
    sd = torch.rand(C, generator=g) + 0.5
    w1, s1 = torch.randn(C, Cin, 1, 1, 1, generator=g) * 0.1, torch.rand(C, generator=g) + 0.5
    g1 = act16((N, C) + size, g)
    if cancel:
        gy, wd = gy.abs(), wd.abs()
        w1, s1 = wd, sd
        g1 = zero_insert_ref((-0.996 * gy.double()).half().double(), size, 2).half()
    x = act16((N, Cin) + size, g, relu=True)
    if cancel:
        x = x.abs() + 1
    pg_exact = rows_of(gy.double()) @ w16_folded(wd, sd).reshape(C, Cin)
    pg16 = ncdhw(f16(pg_exact), N, *lo)
    res = zero_insert_ref(pg16, size, 2)
    ref, A, R = dgrad_1x1(rows_of(g1), w1, s1, mask=rows_of(x), residual=rows_of(res))
    main = rows_of(g1.double()) @ w16_folded(w1, s1).reshape(C, Cin)
    return (ref, grad_bound(ref, A, R), main, rows_of(x) > 0, res, zero_insert_ref(ncdhw(pg_exact, N, *lo), size, 2), lo)


def test_stride2_projection_faults():
    for cancel in (False, True):
        ref, bnd, main, keep, res, res_exact, lo = stride2_problem(5, cancel)
        passes("type B s2 dx%s" % (" cancelling" if cancel else ""), f16((main + rows_of(res)) * keep), ref, bnd)
    fault("pg_added_before_rounding", f16((main + rows_of(res_exact)) * keep), ref, bnd)
    ref, bnd, main, keep, res, _, lo = stride2_problem(6, False)
    shifted = res.clone()
    shifted[:, :, :, -1] = 0                                     # the last low-res row of an odd H dropped (Ho = H // 2)
    fault("odd_border_zero_insert", f16((main + rows_of(shifted)) * keep), ref, bnd)


def test_type_a_channel_block():
    """Type A: channels [0, Cin) of the block-output gradient go to the input, the rest belong to the zero padding."""
    g = gen(7)
    N, Cin, size = 2, 16, (3, 7, 9)
    lo = tuple((n - 1) // 2 + 1 for n in size)
    gA = act16((N, 2 * Cin) + lo, g)
    g1 = act16((N, 24) + size, g)
    w1, s1 = torch.randn(24, Cin, 1, 1, 1, generator=g) * 0.1, torch.rand(24, generator=g) + 0.5
    x = act16((N, Cin) + size, g, relu=True)
    res = zero_insert_ref(gA.double(), size, 2, channels=Cin)
    ref, A, R = dgrad_1x1(rows_of(g1), w1, s1, mask=rows_of(x), residual=rows_of(res))
    bnd = grad_bound(ref, A, R)
    main = rows_of(g1.double()) @ w16_folded(w1, s1).reshape(24, Cin)
    keep = rows_of(x) > 0
    passes("type A dx", f16((main + rows_of(res)) * keep), ref, bnd)
    wrong = zero_insert_ref(gA.double()[:, Cin:], size, 2, channels=Cin)
    fault("type_a_wrong_channel_block", f16((main + rows_of(wrong)) * keep), ref, bnd)
