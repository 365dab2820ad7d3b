"""CPU: the check functions of tests/model_audit.py catch faults that the benchmark's parity metric (the globally pooled output
of the first clips, 5e-3 of its max) lets through, and the filter routes of the packs the audit cannot read back agree with the
references the kernel-matrix files use.  Each fault is injected into an otherwise correctly rounded output."""
import pytest
import torch
import torch.nn.functional as F

from tests import kernel_ref as KR
from tests import model_audit as MA


def bench_metric(got, ref, N, clips=2):
    """bench.py's parity check on an activation: the global average of each of the first ``clips`` samples, max abs error over
    the max |ref|."""
    g = got.double().reshape(N, -1, got.shape[-1]).mean(1)[:clips]
    r = ref.double().reshape(N, -1, ref.shape[-1]).mean(1)[:clips]
    return float((g - r).abs().max() / r.abs().max())


def conv_case(seed, N=4, T=4, H=8, W=8, C=16, K=24, scale=None):
    g = torch.Generator().manual_seed(seed)
    k, s, p = (3, 3, 3), (1, 1, 1), (1, 1, 1)
    x = torch.randn(N, T, H, W, C, generator=g).half()
    w = (torch.randn(K, 27, C, generator=g) / (27 * C) ** 0.5).half()
    sc = torch.rand(K, generator=g) + 0.5 if scale is None else scale
    sh = torch.randn(K, generator=g) * 0.1
    ref, _ = KR.conv_ref(x, w, sc, sh, k, s, p, relu=True)
    return x, w, sc, sh, k, s, p, ref


def test_clean_outputs_pass():
    x, w, sc, sh, k, s, p, ref = conv_case(1)
    r, _ = MA.check_conv(x, w, sc, sh, k, s, p, ref.half(), 24, relu=True)
    assert r <= 1.0


def test_error_in_the_last_clip_fails_the_audit_only():
    N = 4
    x, w, sc, sh, k, s, p, ref = conv_case(2, N=N)
    y = ref.half()
    rows = ref.shape[0] // N
    y[(N - 1) * rows + 5, 3] += 0.25
    assert bench_metric(y, ref, N) <= 5e-3
    r, where = MA.check_conv(x, w, sc, sh, k, s, p, y, 24, relu=True)
    assert r > 1.0 and "row %d col 3" % ((N - 1) * rows + 5) in where


def test_one_m_tile_off_by_a_few_ulps_fails_the_audit_only():
    g = torch.Generator().manual_seed(3)
    M, N, Kd = 1024, 64, 256
    a = torch.randn(M, Kd, generator=g).half()
    b = (torch.randn(N, Kd, generator=g) / 16).half()
    sc, sh = torch.rand(N, generator=g) + 0.5, torch.randn(N, generator=g) * 0.1
    v, _ = KR.epilogue(*KR.gemm_acc(a, b), sc, sh)
    d = v.half()
    t0 = 4 * 128                                       # one 128-row tile in the middle of the batch: 3 fp16 ulps off
    tile = d[t0:t0 + 128].float()
    d[t0:t0 + 128] = (tile + 3 * tile.abs() * 2.0 ** -10).half()
    assert bench_metric(d, v, 8) <= 5e-3
    r, where = MA.check_gemm(a, b, sc, sh, M, N, Kd, d)
    assert r > 1.0 and 128 * 4 <= int(where.split()[2]) < 128 * 5


def test_small_bn_scale_channel_dropping_a_tap_fails_the_audit_only():
    K = 24
    scale = torch.full((K,), 1.0)
    scale[7] = 2.0 ** -8
    x, w, sc, sh, k, s, p, ref = conv_case(4, K=K, scale=scale)
    w_drop = w.clone()
    w_drop[7, 13] = 0                                  # channel 7 loses tap 13
    bad, _ = KR.conv_ref(x, w_drop, sc, sh, k, s, p, relu=True)
    y = ref.half()
    y[:, 7] = bad[:, 7].half()
    assert bench_metric(y, ref, 4) <= 5e-3
    r, where = MA.check_conv(x, w, sc, sh, k, s, p, y, K, relu=True)
    assert r > 1.0 and "col 7" in where


def test_chain_h1_from_unrounded_d_fails_the_audit():
    """h1 must be formed from the fp16 D the kernel stored.  D values whose fp16 rounding errors line up with the signs of W1
    make a chain that reads the fp32 D instead visible: the errors add instead of cancelling."""
    g = torch.Generator().manual_seed(5)
    M, N, n1 = 256, 256, 64
    w1 = (torch.randn(n1, N, generator=g) / 16).half()
    sgn = torch.sign(w1[0].float())
    d16 = (torch.rand(M, N, generator=g) * 2 + 1).half()
    ulp = torch.full_like(d16.float(), 2.0 ** -10) * torch.where(d16.float() >= 2, 2.0, 1.0)
    d32 = d16.double() + 0.2 * ulp.double() * sgn.double()             # rounds to d16
    assert torch.equal(d32.half(), d16)
    sc1, sh1 = torch.ones(n1), torch.zeros(n1)
    # a bias that puts output 0 near zero, so that the error is not hidden behind 2^-11 |h1|
    sh1[0] = -float((d16.double() @ w1.double()[0]).mean())
    good = (d16.double() @ w1.double().t() + sh1.double()).clamp_min(0).half()
    r_good, _ = MA.check_chain_h1(d16, N, w1, sc1, sh1, n1, good)
    assert r_good <= 1.0
    bad = (d32 @ w1.double().t() + sh1.double()).clamp_min(0).half()
    r_bad, where = MA.check_chain_h1(d16, N, w1, sc1, sh1, n1, bad)
    assert r_bad > 1.0 and "col 0" in where


def test_attention_row_missing_a_key_tile_fails_the_audit_only():
    g = torch.Generator().manual_seed(6)
    B, Nq, Nk, d, dv = 2, 256, 512, 64, 64
    q = (torch.randn(B * Nq, d, generator=g) * 0.3).half()
    k = (torch.randn(B * Nk, d, generator=g) * 0.3).half()
    v = torch.randn(B * Nk, dv, generator=g).half()
    ref, _ = KR.att_ref(q, k, v, B, Nq, Nk, 0)
    o = ref.half()
    row = Nq + 17                                      # sample 1, query 17: keys [128, 192) dropped
    keep = torch.ones(Nk, dtype=torch.bool)
    keep[128:192] = False
    kb, vb = k[Nk:][keep], v[Nk:][keep]
    o[row] = KR.att_ref(q[row:row + 1], kb, vb, 1, 1, int(keep.sum()), 0)[0][0].half()
    assert bench_metric(o, ref, B) <= 5e-3
    r, where = MA.check_attention(q, k, v, d, dv, B, Nq, Nk, 0, o)
    assert r > 1.0 and "row %d" % row in where


def test_stem_route_equals_stem_operands():
    g = torch.Generator().manual_seed(7)
    weight = torch.randn(64, 3, 3, 7, 7, generator=g)
    x = torch.randn(1, 3, 4, 16, 16, generator=g)
    x4, w4 = KR.stem_operands(x, weight)
    assert torch.equal(MA.stem_filter(weight), w4)
    sc, sh = torch.rand(64, generator=g) + 0.5, torch.randn(64, generator=g)
    ref, A = KR.conv_ref(x4, w4, sc, sh, (3, 7, 7), (1, 2, 2), (1, 3, 3), relu=True)
    r, _ = MA.check_conv(x4, MA.stem_filter(weight), sc, sh, (3, 7, 7), (1, 2, 2), (1, 3, 3), ref.half(), 64, relu=True)
    assert r <= 1.0


def test_grouped_route_equals_the_dense_grouped_conv():
    g = torch.Generator().manual_seed(8)
    C, groups = 64, 16
    weight = torch.randn(C, C // groups, 3, 3, 3, generator=g) / 6
    x = torch.randn(2, C, 4, 6, 6, generator=g).half()
    want = F.conv3d(x.double(), weight.half().double(), padding=1, groups=groups)
    w = MA.grouped_filter(weight, groups, C)
    got, _ = KR.conv_acc(x.permute(0, 2, 3, 4, 1), w, (3, 3, 3), (1, 1, 1), (1, 1, 1))
    assert torch.allclose(got, want.permute(0, 2, 3, 4, 1).reshape(-1, C), rtol=0, atol=1e-12)


def test_upsample_route_equals_upconv_of_the_fold():
    g = torch.Generator().manual_seed(9)
    K, Cin, H, W = 16, 8, 5, 6
    weight = torch.randn(K, Cin, 3, 3, generator=g)
    x = torch.randn(2, H, W, Cin, generator=g).half()
    fold, _ = KR.upconv_fold(weight)
    wph = fold.float().half()
    r, _ = MA.check_upconv_pack(wph, weight)
    assert r <= 1.0
    acc, _ = KR.upconv_acc(x, wph)
    up = x.double().permute(0, 3, 1, 2).repeat_interleave(2, 2).repeat_interleave(2, 3)
    want = F.conv2d(up, weight.double(), padding=1)                                     # the unfolded 3x3 on the upsampled image
    err = (acc - want.permute(0, 2, 3, 1).reshape(-1, K)).abs().max()
    assert float(err) <= 2.0 ** -9 * float(want.abs().max())                           # only the pack's fp16 rounding differs
    bad = wph.clone()
    bad[3, 5, 2] += 0.5
    assert MA.check_upconv_pack(bad, weight)[0] > 1.0


def test_unknown_entry_or_flag_raises():
    aud = MA._Auditor(None, None)

    def mystery(a, b=1):
        raise RuntimeError("must not launch")
    with pytest.raises(MA.AuditError, match="no check"):
        aud.wrap("mystery", mystery)(0)

    def conv(a, pc, residual=None, relu=False, new_flag=False):
        raise RuntimeError("must not launch")
    with pytest.raises(MA.AuditError, match="new_flag"):
        aud.wrap("conv", conv)(0, 0)
    x, w, sc, sh, k, s, p, ref = conv_case(10)
    with pytest.raises(MA.AuditError):
        MA.check_conv(x, w, sc, sh, k, s, p, ref.half(), 24, relu=True, pool_w=True, residual=ref.half())
    with pytest.raises(MA.AuditError):
        MA.check_gemm(ref.half(), ref.half(), sc, sh, ref.shape[0], 8, 8, ref.half(), next_affine=(sc, sh, 1))


def test_unaudited_and_pass_through_tables_name_real_entries():
    from pretorched_x_b200 import ops
    for name in list(MA.UNAUDITED) + list(MA.PASS_THROUGH) + list(MA.PASS_THROUGH.values()) + list(MA.ENTRIES):
        assert callable(getattr(ops, name)), name
    assert not set(MA.UNAUDITED) & set(MA.ENTRIES)


# ---------------------------------------------------------------------------------------------
# the column-slice, DenseNet and squeeze-excite entries: faults a logit check cannot see, and the positive controls
# ---------------------------------------------------------------------------------------------
INF = float("inf")


def test_slice_conv_writing_the_next_column_fails_the_slice_contract():
    """A dense layer's 3x3 convolution that also writes the first column after its slice: its own columns are right, and the
    next layer overwrites that column before anything reads it, so the logits are unchanged.  Only the slice contract sees it."""
    K, c0 = 24, 40
    x, w, sc, sh, k, s, p, ref = conv_case(11, K=K)
    M = ref.shape[0]
    parent = torch.full((M, c0 + K + 16), float("nan"), dtype=torch.float16)      # uninitialised columns: NaN patterns
    parent[:, :c0] = torch.randn(M, c0, generator=torch.Generator().manual_seed(12)).half()
    y = parent[:, c0:c0 + K]
    guard = MA.SliceGuard([(y, K)])
    y.copy_(ref.half())
    assert MA.check_conv(x, w, sc, sh, k, s, p, y, K, relu=True)[0] <= 1.0
    assert guard.check()[0] == 0.0
    parent[M - 1, c0 + K] = 0.5
    assert MA.check_conv(x, w, sc, sh, k, s, p, y, K, relu=True)[0] <= 1.0
    r, where = guard.check()
    assert r == INF and "row %d col %d" % (M - 1, c0 + K) in where


def _split_case(seed, cols, M=200, Kd=96):
    from pretorched_x_b200 import ops
    g = torch.Generator().manual_seed(seed)
    npad, box0 = ops.split_plan(cols)
    a = (torch.rand(M, Kd, generator=g) - 0.3).half()
    b = torch.zeros(npad, Kd, dtype=torch.float16)
    scale, shift = torch.zeros(npad), torch.zeros(npad)
    for d, n in enumerate(cols):
        r0 = 64 * box0[d]
        b[r0:r0 + n] = ((torch.rand(n, Kd, generator=g) - 0.5) / Kd ** 0.5).half()
        scale[r0:r0 + n], shift[r0:r0 + n] = torch.rand(n, generator=g) + 0.5, torch.rand(n, generator=g) - 0.5
    return a, b, scale, shift, box0, M, Kd


def test_split_gemm_reading_the_previous_destinations_rows_fails_the_audit():
    cols = [96, 40]
    a, b, scale, shift, box0, M, Kd = _split_case(13, cols)

    def dest(r0, n):
        v, _ = KR.epilogue(*KR.gemm_acc(a, b[r0:r0 + n]), scale[r0:r0 + n], shift[r0:r0 + n], relu=True)
        return v.half()
    parent = torch.zeros(M, 8 + sum(cols), dtype=torch.float16)
    dests = [parent[:, 8:8 + cols[0]], parent[:, 8 + cols[0]:]]
    dests[0].copy_(dest(64 * box0[0], cols[0]))
    dests[1].copy_(dest(64 * box0[1], cols[1]))
    assert MA.check_gemm_split(a, b, scale, shift, M, Kd, dests)[0] <= 1.0
    dests[1].copy_(dest(64 * (box0[1] - 1), cols[1]))                # box0 off by one: dest 0's packed rows 64 ..
    r, where = MA.check_gemm_split(a, b, scale, shift, M, Kd, dests)
    assert r > 1.0 and where.startswith("dest 1")


def test_transition_pool_with_relu_after_the_mean_fails_the_audit():
    g = torch.Generator().manual_seed(14)
    N, H, W, C = 2, 6, 6, 16
    x = torch.randn(N * H * W, C + 8, generator=g).half()
    s, t = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.1
    v = (x[:, :C].double() * s.double() + t.double()).reshape(N, H, W, C).permute(0, 3, 1, 2)
    good = F.avg_pool2d(v.clamp_min(0.0), 2, 2).permute(0, 2, 3, 1).reshape(-1, C)
    bad = F.avg_pool2d(v, 2, 2).clamp_min(0.0).permute(0, 2, 3, 1).reshape(-1, C)
    mixed = (F.max_pool2d(v, 2, 2) > 0) & (-F.max_pool2d(-v, 2, 2) < 0)
    assert bool(mixed.any())                                          # windows whose signs differ
    assert MA.check_transition_pool(x, N, H, W, C, s, t, good.half())[0] <= 1.0
    assert MA.check_transition_pool(x, N, H, W, C, s, t, bad.half())[0] > 1.0


@pytest.mark.parametrize("avg,count_include_pad,ceil_mode,k,st,p", [
    (False, True, False, (3, 3), (2, 2), (1, 1)),         # DenseNet's pool0
    (False, True, False, (3, 1), (2, 1), (1, 0)),         # its H pass after the stem's W pool
    (False, True, True, (3, 3), (2, 2), (0, 0)),          # BNInception's ceil-mode pass-through pools
    (True, True, True, (3, 3), (1, 1), (1, 1)),           # BNInception's pool branches
    (True, False, True, (3, 3), (1, 1), (1, 1)),          # Inception-v4's pool branches
])
def test_slice_pool_check_passes_the_rounded_reference(avg, count_include_pad, ceil_mode, k, st, p):
    g = torch.Generator().manual_seed(15)
    N, H, W, C, off = 2, 9, 8, 16, 8
    src = torch.randn(N * H * W, off + C + 8, generator=g).half()
    x = src[:, off:off + C]                                           # the input is itself a column slice
    xs = x.double().reshape(N, H, W, C).permute(0, 3, 1, 2)
    if avg:
        ref = F.avg_pool2d(xs, k, st, p, ceil_mode=ceil_mode, count_include_pad=count_include_pad)
    else:
        ref = F.max_pool2d(xs, k, st, p, ceil_mode=ceil_mode)
    y = ref.permute(0, 2, 3, 1).reshape(-1, C).half()
    assert MA.check_pool_slice(x, N, 1, H, W, C, k, st, p, avg, y, count_include_pad, ceil_mode)[0] <= 1.0
    y[5, 3] = -y[5, 3] if float(y[5, 3]) != 0 else 1.0
    assert MA.check_pool_slice(x, N, 1, H, W, C, k, st, p, avg, y, count_include_pad, ceil_mode)[0] > 1.0


def test_exclude_pad_average_divided_by_the_full_window_fails_the_audit():
    g = torch.Generator().manual_seed(16)
    N, H, C = 2, 8, 16
    x = (torch.rand(N * H * H, C, generator=g) * 4 - 1).half()
    xs = x.double().reshape(N, H, H, C).permute(0, 3, 1, 2)
    good = F.avg_pool2d(xs, 3, 1, 1, count_include_pad=False).permute(0, 2, 3, 1).reshape(-1, C).half()
    bad = F.avg_pool2d(xs, 3, 1, 1, count_include_pad=True).permute(0, 2, 3, 1).reshape(-1, C).half()
    args = (x, N, 1, H, H, C, (3, 3), (1, 1), (1, 1), True)
    assert MA.check_pool_slice(*args, good, count_include_pad=False)[0] <= 1.0
    r, where = MA.check_pool_slice(*args, bad, count_include_pad=False)
    row = int(where.split()[2]) % (H * H)
    assert r > 1.0 and (row // H in (0, H - 1) or row % H in (0, H - 1))          # a border window


def test_head_pool_without_the_relu_fails_the_audit():
    g = torch.Generator().manual_seed(17)
    N, S, C = 3, 49, 64
    x = torch.randn(N * S, C, generator=g).half()
    s, t = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.2
    v = (x.double() * s.double() + t.double()).reshape(N, S, C)
    good, bad = v.clamp_min(0.0).mean(1).half(), v.mean(1).half()
    assert MA.check_head_pool(x, N, S, C, s, t, good)[0] <= 1.0
    assert MA.check_head_pool(x, N, S, C, s, t, bad)[0] > 1.0


def test_excite_scales_from_the_next_sample_fail_the_audit():
    g = torch.Generator().manual_seed(18)
    N, S, C2, C = 4, 49, 64, 256
    R = C // 16
    h = (torch.rand(N * S, C2 + 8, generator=g) * 3).half()
    w1, b1 = torch.randn(R, C2, generator=g) / C2 ** 0.5, torch.randn(R, generator=g) * 0.1
    w2, b2 = torch.randn(C, R, generator=g) / R ** 0.5, torch.randn(C, generator=g) * 0.1
    s3, t3 = torch.rand(C, generator=g) + 0.5, torch.randn(C, generator=g) * 0.2
    r = KR.excite_ref(*KR.excite_mean(h, N, S, C2), w1, b1, w2, b2, s3, t3)
    scale, shift = r["scale"].float(), r["shift"].float()
    assert MA.check_se_excite(h, N, S, C2, w1, b1, w2, b2, s3, t3, scale, shift)[0] <= 1.0
    r_bad, where = MA.check_se_excite(h, N, S, C2, w1, b1, w2, b2, s3, t3, scale.roll(-1, 0), shift.roll(-1, 0))
    assert r_bad > 1.0


def _preact_kernel_model(a, b, s1, t1, s2, t2, k):
    """b2_gemm_preact_f16's arithmetic over the first k columns of A, B and the input affine: x' = fp16(fmaxf(x s + t, 0)) --
    torch.fmax, like CUDA's fmaxf, returns the operand that is not NaN -- then the GEMM and relu(s2 acc + t2) in fp64, rounded to
    fp16 into an output eight columns wider than N."""
    v = a[:, :k].double() * s1[:k].double() + t1[:k].double()
    x = torch.fmax(v, torch.zeros_like(v)).half().double()
    acc = x @ b[:, :k].double().t()
    d = torch.zeros(a.shape[0], b.shape[0] + 8, dtype=torch.float16)
    d[:, :b.shape[0]] = (acc * s2.double() + t2.double()).clamp_min(0.0).half()
    return d


def test_preact_gemm_reading_past_kd_fails_the_audit():
    """A pre-activated GEMM that also reads column Kd (or the rest of its last 64-column K block) of A, B and the input affine.
    In the model its input affine is zero past Kd, so a NaN there is invisible: fmaxf(fmaf(NaN, 0, 0), 0) = 0.  The audit's
    finite values past Kd (``preact_contract``) make every such read move the output far past the bound."""
    g = torch.Generator().manual_seed(19)
    M, N, Kd, lda = 300, 128, 96, 136
    a = torch.randn(M, lda, generator=g).half()
    b = (torch.randn(N, Kd + 8, generator=g) * Kd ** -0.5).half()
    kpad = 128
    s1, t1 = torch.zeros(kpad), torch.zeros(kpad)
    s1[:Kd], t1[:Kd] = torch.rand(Kd, generator=g) + 0.5, torch.rand(Kd, generator=g) * 0.5
    s2, t2 = torch.rand(N, generator=g) + 0.5, torch.randn(N, generator=g) * 0.1
    good = _preact_kernel_model(a, b, s1, t1, s2, t2, Kd)
    assert MA.check_gemm_preact(a, b, s2, t2, s1, t1, M, N, Kd, good)[0] <= 1.0
    # why the audit does not use NaN: with the model's own zero affine past Kd, a NaN-poisoned over-read changes no bit
    a_nan = a.clone()
    a_nan[:, Kd:] = float("nan")
    assert torch.equal(_preact_kernel_model(a_nan, b, s1, t1, s2, t2, Kd + 1), good)
    # the audited call: finite values past Kd in A (in place), and in copies of B and of the input affine
    bits = a.view(torch.int16).clone()
    call, restore = MA.preact_contract(dict(a2d=a, b2d=b, scale=s2, shift=t2, in_scale=s1, in_shift=t1, M=M, N=N, Kd=Kd, relu=True))
    assert bool((a[:, Kd:] == MA.PREACT_A).all()) and torch.equal(a[:, :Kd].view(torch.int16), bits[:, :Kd])
    assert call["b2d"].stride(0) == b.stride(0) + 64 and torch.equal(call["b2d"][:, :Kd], b[:, :Kd])
    assert torch.equal(call["in_scale"][:Kd], s1[:Kd]) and torch.equal(call["in_shift"][:Kd], t1[:Kd])
    args = (call["a2d"], call["b2d"], call["in_scale"], call["in_shift"], s2, t2)
    assert torch.equal(_preact_kernel_model(*args, Kd), good)                    # a kernel that keeps to Kd: the same output
    for k in (Kd + 1, kpad):
        r, where = MA.check_gemm_preact(a, b, s2, t2, s1, t1, M, N, Kd, _preact_kernel_model(*args, k))
        assert r > 1.0, (k, where)
    restore()
    assert torch.equal(a.view(torch.int16), bits)                                 # the exact bits are back
    good[7, N + 3] = 1.0                                                          # a pad column that is not zero
    assert MA.check_gemm_preact(a, b, s2, t2, s1, t1, M, N, Kd, good)[0] == INF


def test_slice_guard_locates_the_parent_rows_from_the_base_matrix():
    """A block matrix that starts mid-row of a flat workspace has no row grid the guard could assume: it refuses rather than
    check a rotated span.  Slices of a 2-D matrix are located by its rows, and slices of the same rows are checked together."""
    ws = torch.zeros(10 * 24 + 5, dtype=torch.float16)
    blk = ws[5:].view(10, 24)
    with pytest.raises(MA.AuditError, match="cannot be located"):
        MA.SliceGuard([(blk[:, 8:16], 8)])
    parent = torch.zeros(12, 24, dtype=torch.float16)
    rows = parent[2:11]
    guard = MA.SliceGuard([(rows[:, 0:8], 8), (rows[:, 16:24], 8)])
    parent[2:11, 0:8], parent[2:11, 16:24] = 1.0, 2.0
    parent[0, 9] = parent[11, 9] = 3.0                                            # rows outside the slices' rows
    assert guard.check()[0] == 0.0
    parent[10, 8] = 4.0
    r, where = guard.check()
    assert r == INF and "row 8 col 8" in where                                    # rows count from the slices' first row


def test_every_launching_entry_of_ops_is_in_the_audit_tables():
    """Every function of pretorched_x_b200/ops.py whose body calls ``_lib.check(`` is audited, recorded as unaudited or a
    composite: a launching entry added later cannot slip past the audit.  The pack constructors (wrapped separately) and
    ``_conv_grouped`` (reached through ``conv``) are the exceptions."""
    import ast
    from pretorched_x_b200 import ops
    with open(ops.__file__) as f:
        tree = ast.parse(f.read())
    launching = set()
    for node in ast.walk(tree):
        if isinstance(node, ast.FunctionDef):
            for call in ast.walk(node):
                if (isinstance(call, ast.Call) and isinstance(call.func, ast.Attribute) and call.func.attr == "check"
                        and isinstance(call.func.value, ast.Name) and call.func.value.id == "_lib"):
                    launching.add(node.name)
                    break
    launching -= {"__init__", "_conv_grouped"}
    assert {"conv", "gemm", "gemm_preact", "se_excite"} <= launching
    tables = set(MA.ENTRIES) | set(MA.UNAUDITED) | set(MA.PASS_THROUGH)
    assert not launching - tables, "launching entries the audit does not wrap: %s" % sorted(launching - tables)
    assert set(MA.KNOWN) == set(MA.ENTRIES)
