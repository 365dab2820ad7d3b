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
    with pytest.raises(MA.AuditError, match="no check"):
        aud.wrap("se_excite", mystery)(0)

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
    for name in list(MA.UNAUDITED) + list(MA.PASS_THROUGH) + list(MA.PASS_THROUGH.values()) + list(MA.NO_CHECK) + list(MA.ENTRIES):
        assert callable(getattr(ops, name)), name
    assert not set(MA.UNAUDITED) & set(MA.ENTRIES)
