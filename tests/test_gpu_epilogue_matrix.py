"""GPU (-m gpu): the generator epilogues of the convolution / GEMM kernels against fp64, element by element, with the kernel that
ran pinned -- per-sample affine, fused upsample, upsampled and pre-affine residuals, second output, input affine, the two-operand
GEMM -- and the output pitch contract of every fp16 family: columns [K, ldy) of y are written as zero whatever the residual holds
past its K columns, and a residual pitch narrower than y's is never read past its row.

Same conventions as tests/test_gpu_kernel_matrix.py (whose helpers and knob-restoring fixture this file uses): references from
exactly the operands the kernel reads (tests/kernel_ref.py), the bound of that file, rows outside ``out=`` keep a NaN sentinel,
two identical calls are bitwise equal.  Worst err / bound ratios are printed per case (pytest -s)."""
import ctypes
import os

import pytest
import torch
import torch.nn as nn

from oracle import functional as OF
from tests.conftest import has_h100
from tests.kernel_ref import (conv_acc, conv_ref, epilogue, gemm_acc, in_affine_acc, nearest_up2, per_row, second_output,
                              upconv_acc, upconv_fold)
from tests.test_gpu_kernel_matrix import (DENSEM, IGEMM, KIND, KNOB_ENV, PGEMM, SLAB, TSTACK, Problem, _lib, assert_within, dev,
                                          last_kernel, lib, plan_info, rup, seed_of)

pytestmark = [
    pytest.mark.gpu,
    pytest.mark.skipif(not has_h100(), reason="needs an H100"),
    pytest.mark.skipif(any(os.environ.get(e) for e in KNOB_ENV),
                       reason="a dispatch override is set in the environment (%s)" % ", ".join(KNOB_ENV)),
]
__all__ = ["dev", "lib"]          # the fixtures of the kernel matrix, used here under the same names

GROUPCONV = 10                    # KID_GROUPCONV of csrc/b2_host.h
PAD = 3                           # NaN sentinel rows on either side of an out= row range


def ops():
    from pretorched_x_b200 import ops as O
    return O


def gen(name):
    return torch.Generator().manual_seed(seed_of(name))


def affine_views(dev, g, N, K):
    """Per-sample (scale, shift) as views into ONE fp32 buffer [N][2 P] (P = round_up(K, 4) + 4), the way biggan_engine._aff
    slices its table: scale = [:, 0:K], shift = [:, P:P + K], pitch 2 P > K.  [K, P) and [P + K, 2 P) hold NaN: never read."""
    P = rup(K, 4) + 4
    buf = torch.full((N, 2 * P), float("nan"))
    buf[:, :K] = torch.rand(N, K, generator=g) + 0.5
    buf[:, P:P + K] = torch.randn(N, K, generator=g) * 0.3
    d = buf.to(dev)
    return d[:, :K], d[:, P:P + K]


def sentinel_buf(dev, M, ld, dtype=torch.float16):
    buf = torch.full((M + 2 * PAD, ld), float("nan"), dtype=dtype, device=dev)
    return buf, buf[PAD:PAD + M]


def check_rows(name, buf, out, M, K, ref, A, f16=True):
    """Bound on [:, :K], exact zeros in [K, ldy), NaN sentinel rows untouched."""
    assert_within(name, out[:, :K], ref, A, f16)
    if out.shape[1] > K:
        pad = out[:, K:].float().cpu()
        assert torch.all(pad == 0), "%s: padding columns [K, ldy) not zero (%d non-zero)" % (name, int((pad != 0).sum()))
    assert torch.isnan(buf[:PAD].float()).all() and torch.isnan(buf[PAD + M:].float()).all(), "%s: rows outside out= written" % name


def same_bits(a, b):
    return torch.equal(a.contiguous().view(torch.int16), b.contiguous().view(torch.int16))


def slab_plan_of(lib, pb_or_shape, ldy, aff_ld=0, upsample=0):
    """b2_debug_slab_plan (host only) of a convolution under the current knobs, with the per-sample / upsample fields set."""
    N, T, H, W, C, K, k, s, p = pb_or_shape
    a = _lib().ConvArgs()
    a.N, a.T, a.H, a.W, a.C, a.K, a.ldy = N, T, H, W, C, K, ldy
    a.kt, a.kh, a.kw = k
    a.st, a.sh, a.sw = s
    a.pt, a.ph, a.pw = p
    a.aff_ld, a.upsample = aff_ld, upsample
    out = (ctypes.c_int * 10)()
    assert lib.b2_debug_slab_plan(ctypes.byref(a), out) == 0
    return tuple(out)


def shape_of(pb):
    return (pb.a.N, pb.a.T, pb.a.H, pb.a.W, pb.a.ld, pb.K, pb.k, pb.s, pb.p)


def run_ops_conv(dev, lib, name, M, ldy, K, call, ref, A, ref2=None, A2=None):
    """``call(out)`` runs ops.conv into ``out`` (a row range of a NaN-filled buffer) and returns its result.  Checks the bound, the
    zero padding, the sentinel rows and a bitwise-equal second call (second output included).  Returns the kernel probe."""
    buf, out = sentinel_buf(dev, M, ldy)
    res = call(out)
    torch.cuda.synchronize()
    probe = last_kernel(lib)
    label = "%s %s" % (KIND[probe[0]], name)
    check_rows(label, buf, out, M, K, ref, A)
    y2 = res[1].data if isinstance(res, tuple) else None
    if ref2 is not None:
        assert_within(label + " y2", y2[:, :K], ref2, A2, True)
        if ldy > K:
            assert torch.all(y2[:, K:].float().cpu() == 0), "y2 padding columns [K, ldy) not zero"
    buf2, out2 = sentinel_buf(dev, M, ldy)
    res2 = call(out2)
    torch.cuda.synchronize()
    assert same_bits(out2, out), "two identical calls differ"
    if y2 is not None:
        assert same_bits(res2[1].data, y2), "two identical calls differ (y2)"
    return probe


# ---------------------------------------------------------------------------------------------
# slab kernel, per-sample affine
# ---------------------------------------------------------------------------------------------
# name, N, Cin, pitch, T, H, W, K, kernel, stride, padding
PS_CASES = [
    ("ps_fixed64", 2, 64, 64, 1, 12, 14, 64, (1, 3, 3), (1, 1, 1), (0, 1, 1)),
    ("ps_fixed128", 2, 64, 64, 1, 12, 14, 128, (1, 3, 3), (1, 1, 1), (0, 1, 1)),
    ("ps_flex_k144", 2, 64, 64, 1, 10, 12, 144, (1, 3, 3), (1, 1, 1), (0, 1, 1)),
    ("ps_n16_k3", 2, 64, 64, 1, 20, 20, 3, (1, 3, 3), (1, 1, 1), (0, 1, 1)),
    ("ps_n16_k6", 3, 32, 32, 1, 16, 16, 6, (1, 3, 3), (1, 1, 1), (0, 1, 1)),
    ("ps_wchunks_w256", 1, 64, 64, 1, 4, 256, 64, (1, 3, 3), (1, 1, 1), (0, 1, 1)),
    ("ps_300_samples_8x8", 300, 64, 64, 1, 8, 8, 64, (1, 3, 3), (1, 1, 1), (0, 1, 1)),
    ("ps_3x3x3_t3", 2, 32, 32, 3, 6, 7, 40, (3, 3, 3), (1, 1, 1), (1, 1, 1)),
]
PS_EXPECT = {"ps_fixed64": ("bn", 64), "ps_fixed128": ("bn", 128), "ps_flex_k144": ("flex", 1), "ps_n16_k3": ("bn", 16),
             "ps_n16_k6": ("bn", 16), "ps_wchunks_w256": ("wchunks", 2)}
PLAN_AT = {"bn": 1, "mt": 2, "wchunks": 6, "flex": 8}


def make_ps(dev, case):
    name, N, Cin, pitch, T, H, W, K, k, s, p = case
    return Problem(dev, name, N, Cin, T, H, W, K, k, s, p, pitch=pitch)


def run_per_sample(dev, lib, pb, relu, residual, tag=""):
    O = ops()
    M, K, ldy = pb.M, pb.K, pb.ldy
    sc, sh = affine_views(dev, pb.gen, pb.a.N, K)
    r = pb.residual(dev, ldy + 16) if residual else None
    ract = O.Act(r, pb.a.N, pb.To, pb.Ho, pb.Wo, K) if residual else None
    acc, mag = conv_acc(pb.x, pb.w, pb.k, pb.s, pb.p)
    rows = pb.To * pb.Ho * pb.Wo
    ref, A = epilogue(acc, mag, per_row(sc.cpu(), rows, M, K), per_row(sh.cpu(), rows, M, K),
                      residual=None if r is None else r[:, :K].cpu().double(), relu=relu)
    name = "%s per-sample%s%s%s" % (pb.name, " relu" if relu else "", " res" if residual else "", tag)
    return run_ops_conv(dev, lib, name, M, ldy, K,
                        lambda out: O.conv(pb.a, pb.pc, residual=ract, relu=relu, sample_affine=(sc, sh), out=out), ref, A)


@pytest.mark.parametrize("residual", [False, True], ids=["nores", "res"])
@pytest.mark.parametrize("relu", [False, True], ids=["linear", "relu"])
@pytest.mark.parametrize("case", PS_CASES, ids=[c[0] for c in PS_CASES])
def test_slab_per_sample_affine_against_fp64(dev, lib, case, relu, residual):
    lib.b2_debug_set_densem(0, 0)
    pb = make_ps(dev, case)
    aff_ld = 2 * (rup(pb.K, 4) + 4)
    plan = slab_plan_of(lib, shape_of(pb), pb.ldy, aff_ld=aff_ld)
    if case[0] in PS_EXPECT:
        key, want = PS_EXPECT[case[0]]
        assert plan[PLAN_AT[key]] >= want if key == "wchunks" else plan[PLAN_AT[key]] == want, plan
    kid, info = run_per_sample(dev, lib, pb, relu, residual)
    assert kid == SLAB and info == plan_info(plan)


def _mt_params():
    """ps_fixed64 under a forced MT of 1 and of the largest value set_slab_mt admits on it (from the host plan)."""
    lib = _lib().load()
    case = PS_CASES[0]
    shape = (case[1], case[4], case[5], case[6], case[3], case[7], case[8], case[9], case[10])
    aff_ld = 2 * (rup(case[7], 4) + 4)
    out = []
    try:
        admissible = []
        for mt in (1, 2, 3, 4):
            lib.b2_debug_set_slab_mt(mt)
            if slab_plan_of(lib, shape, rup(case[7], 8), aff_ld=aff_ld)[2] == mt:
                admissible.append(mt)
    finally:
        lib.b2_debug_set_slab_mt(0)
    for mt in sorted({1, max(admissible)}):
        out.append(pytest.param(mt, id="mt%d" % mt))
    return out


@pytest.mark.parametrize("mt", _mt_params())
def test_slab_per_sample_affine_forced_mt(dev, lib, mt):
    lib.b2_debug_set_densem(0, 0)
    lib.b2_debug_set_slab_mt(mt)
    pb = make_ps(dev, PS_CASES[0])
    plan = slab_plan_of(lib, shape_of(pb), pb.ldy, aff_ld=2 * (rup(pb.K, 4) + 4))
    assert plan[2] == mt
    kid, info = run_per_sample(dev, lib, pb, True, True, " mt%d" % mt)
    assert kid == SLAB and info == plan_info(plan)


# ---------------------------------------------------------------------------------------------
# slab kernel, fused nearest-2x upsample (conv3x3 of the upsampled image from the low-res tensor)
# ---------------------------------------------------------------------------------------------
# N, C, H, W, K (low-res input): the shapes of tests/test_gpu_biggan.py (among them a 128-wide low-res row, which is cut into W
# chunks), two N tiles (K = 200) and the runtime-N (flex) tile: 152 columns on a 160-wide tile
UP_CASES = [(3, 64, 12, 20, 64), (2, 128, 16, 16, 128), (5, 512, 4, 4, 512), (2, 16, 40, 40, 8), (2, 64, 10, 128, 64),
            (1, 256, 32, 32, 256), (3, 32, 7, 9, 24), (2, 64, 8, 8, 200), (2, 64, 8, 8, 152)]


def up_problem(dev, N, C, H, W, K):
    O = ops()
    name = "up_%dx%dx%dx%d_k%d" % (N, C, H, W, K)
    g = gen(name)
    x = torch.randn(N, H, W, C, generator=g).half()
    w = torch.randn(K, C, 3, 3, generator=g) / (3 * C ** 0.5)
    bn = OF.randomize_bn_(nn.BatchNorm2d(K), seed_of(name) + 1).eval()
    pc = O.PackedConv(w.to(dev), None, bn.to(dev), (1, 1, 1), (0, 1, 1), in_pitch=C, upsample=True)
    a = O.Act(x.reshape(-1, C).to(dev), N, 1, H, W, C)
    return name, g, x, w, pc, a


@pytest.mark.parametrize("affine", ["sample", "channel"])
@pytest.mark.parametrize("shape", UP_CASES, ids=["%dx%dx%dx%d_k%d" % s for s in UP_CASES])
def test_slab_upsample_against_fp64(dev, lib, shape, affine):
    O = ops()
    N, C, H, W, K = shape
    name, g, x, w, pc, a = up_problem(dev, N, C, H, W, K)
    M, ldy = N * 4 * H * W, rup(K, 8)
    acc, mag = upconv_acc(x, pc.w.view(K, 16, C).cpu())
    kw = {}
    if affine == "sample":
        sc, sh = affine_views(dev, g, N, K)
        kw["sample_affine"] = (sc, sh)
        ref, A = epilogue(acc, mag, per_row(sc.cpu(), 4 * H * W, M, K), per_row(sh.cpu(), 4 * H * W, M, K), relu=True)
    else:
        ref, A = epilogue(acc, mag, pc.scale.cpu(), pc.shift.cpu(), relu=True)
    plan = slab_plan_of(lib, (N, 1, H, W, C, K, (1, 3, 3), (1, 1, 1), (0, 1, 1)), ldy,
                        aff_ld=sc.stride(0) if affine == "sample" else 0, upsample=1)
    kid, info = run_ops_conv(dev, lib, "%s %s" % (name, affine), M, ldy, K,
                             lambda out: O.conv(a, pc, relu=True, out=out, **kw), ref, A)
    assert kid == SLAB and info == plan_info(plan)
    if K == 152:
        assert info[:3:2] == (160, 1), "K = 152 must take the 160-wide runtime-N (flex) tile"
    if W == 128:
        assert info[3] > 1, "a 128-wide low-res row must be cut into W chunks"


@pytest.mark.parametrize("shape", [(64, 64), (200, 24), (8, 16)], ids=["k64_c64", "k200_c24", "k8_c16"])
def test_pack_upconv3x3_weight_against_fp64_fold(dev, shape):
    O = ops()
    K, Cin = shape
    C = rup(Cin, 8) + 8
    w = torch.randn(K, Cin, 3, 3, generator=gen("fold%d" % K)) * 3
    pc = O.PackedConv(w.to(dev), None, None, (1, 1, 1), (0, 1, 1), in_pitch=C, upsample=True)
    got = pc.w.view(K, 16, C).cpu()
    fold, wsum = upconv_fold(w)
    bnd = 2.0 ** -11 * fold.abs() + 2.0 ** -22 * wsum
    ratio = float(((got[:, :, :Cin].double() - fold).abs() / bnd).max())
    print("[epilogue-matrix] pack_upconv3x3 K%d Cin%d worst err/bound %.4f" % (K, Cin, ratio))
    assert ratio <= 1.0
    assert torch.all(got[:, :, Cin:] == 0), "channels [Cin, C) of the phase filter not zero"


# ---------------------------------------------------------------------------------------------
# persistent GEMM, generator instance (1x1 convolutions of the GBlock)
# ---------------------------------------------------------------------------------------------
def pw_problem(dev, name, N, C, H, W, K):
    """1x1 2-D convolution C -> K over N images of H x W (the input already at the output resolution)."""
    return Problem(dev, name, N, C, 1, H, W, K, (1, 1, 1), (1, 1, 1), (0, 0, 0), pitch=C)


def skip_tensor(dev, g, rows, ld, poison_rows=0):
    """Low-res skip tensor [rows][ld] with data in EVERY column (the channels past K are the GBlock's channel drop), as a view
    into a buffer whose ``poison_rows`` following rows are NaN."""
    buf = torch.full((rows + poison_rows, ld), float("nan"), dtype=torch.float16)
    buf[:rows] = torch.randn(rows, ld, generator=g).half()
    d = buf.to(dev)
    return d[:rows], buf[:rows]


def gan_bn(ldy):
    return 64 if ldy <= 64 else 128


# N, C, H, W (output), K, skip pitch: every admissible output width, several images per tile, a channel drop, a ragged M, K = 60
RES_UP_CASES = [(3, 64, 4, 4, 64, 72), (2, 64, 8, 8, 60, 72), (1, 64, 6, 8, 64, 64), (2, 64, 6, 32, 64, 128),
                (1, 128, 4, 64, 128, 136), (1, 64, 2, 128, 64, 64), (1, 64, 2, 256, 200, 208), (1, 64, 6, 64, 60, 64)]


@pytest.mark.parametrize("case", RES_UP_CASES, ids=["n%d_c%d_%dx%d_k%d_ldr%d" % c for c in RES_UP_CASES])
def test_pgemm_residual_up_against_fp64(dev, lib, case):
    O = ops()
    N, C, H, W, K, ldr = case
    pb = pw_problem(dev, "resup_%d_%d_%d_%d_%d_%d" % case, N, C, H, W, K)
    skip, skip_h = skip_tensor(dev, pb.gen, N * (H // 2) * (W // 2), ldr)
    sact = O.Act(skip, N, 1, H // 2, W // 2, K)
    acc, mag = conv_acc(pb.x, pb.w, pb.k, pb.s, pb.p)
    ref, A = epilogue(acc, mag, pb.pc.scale.cpu(), pb.pc.shift.cpu(), residual=nearest_up2(skip_h, N, H, W, K))
    kid, info = run_ops_conv(dev, lib, pb.name + " residual_up", pb.M, pb.ldy, K,
                             lambda out: O.conv(pb.a, pb.pc, residual=sact, residual_up=True, out=out), ref, A)
    assert (kid, info[:3]) == (PGEMM, (gan_bn(pb.ldy), 0, 1))


@pytest.mark.parametrize("case", [(2, 64, 8, 16, 64, 64), (1, 128, 4, 64, 60, 64)], ids=["k64", "k60"])
def test_pgemm_residual_pre_relu_against_fp64(dev, lib, case):
    O = ops()
    N, C, H, W, K, ldr = case
    pb = pw_problem(dev, "respre_%d_%d_%d_%d_%d_%d" % case, N, C, H, W, K)
    r = torch.randn(pb.M, ldr, generator=pb.gen).half()
    ract = O.Act(r.to(dev), N, 1, H, W, K)
    acc, mag = conv_acc(pb.x, pb.w, pb.k, pb.s, pb.p)
    ref, A = epilogue(acc, mag, pb.pc.scale.cpu(), pb.pc.shift.cpu(), residual=r[:, :K].double(), pre=True, relu=True)
    kid, info = run_ops_conv(dev, lib, pb.name + " residual_pre relu", pb.M, pb.ldy, K,
                             lambda out: O.conv(pb.a, pb.pc, residual=ract, residual_pre=True, relu=True, out=out), ref, A)
    assert (kid, info[:3]) == (PGEMM, (gan_bn(pb.ldy), 0, 1))


@pytest.mark.parametrize("K", [64, 200])
def test_pgemm_second_output_against_fp64(dev, lib, K):
    """y2 = relu(s2 * y + t2) from the fp32 first output, one N tile (K = 64) and two (K = 200); the aff2 pitch gap is NaN."""
    O = ops()
    pb = pw_problem(dev, "y2_k%d" % K, 2, 64, 8, 16, K)
    sc2, sh2 = affine_views(dev, pb.gen, 2, K)
    acc, mag = conv_acc(pb.x, pb.w, pb.k, pb.s, pb.p)
    v, A = epilogue(acc, mag, pb.pc.scale.cpu(), pb.pc.shift.cpu(), relu=True)
    ref2, A2 = second_output(v, A, per_row(sc2.cpu(), 128, pb.M, K), per_row(sh2.cpu(), 128, pb.M, K))
    kid, info = run_ops_conv(dev, lib, pb.name + " +y2", pb.M, pb.ldy, K,
                             lambda out: O.conv(pb.a, pb.pc, relu=True, next_affine=(sc2, sh2), out=out), v, A, ref2, A2)
    assert (kid, info[:3]) == (PGEMM, (gan_bn(pb.ldy), 0, 1))


@pytest.mark.parametrize("C", [64, 256])
def test_pgemm_input_affine_against_fp64(dev, lib, C):
    O = ops()
    pb = pw_problem(dev, "inaff_c%d" % C, 2, C, 8, 16, 96)
    isc, ish = affine_views(dev, pb.gen, 2, C)
    acc, mag = in_affine_acc(pb.x.reshape(-1, C), pb.w[:, 0], isc.cpu(), ish.cpu(), 128)
    ref, A = epilogue(acc, mag, pb.pc.scale.cpu(), pb.pc.shift.cpu())
    kid, info = run_ops_conv(dev, lib, pb.name + " in_affine", pb.M, pb.ldy, pb.K,
                             lambda out: O.conv(pb.a, pb.pc, in_affine=(isc, ish), out=out), ref, A)
    assert (kid, info[:3]) == (PGEMM, (gan_bn(pb.ldy), 0, 1))


def test_pgemm_gblock_conv1_in_affine_sample_affine_relu(dev, lib):
    """conv1 of biggan_engine._gblock_body: relu(bn2(conv1(relu(bn1(x))))) -- input affine, per-sample output affine, ReLU."""
    O = ops()
    pb = pw_problem(dev, "gblock_conv1", 2, 128, 16, 16, 64)
    isc, ish = affine_views(dev, pb.gen, 2, 128)
    sc, sh = affine_views(dev, pb.gen, 2, 64)
    acc, mag = in_affine_acc(pb.x.reshape(-1, 128), pb.w[:, 0], isc.cpu(), ish.cpu(), 256)
    ref, A = epilogue(acc, mag, per_row(sc.cpu(), 256, pb.M, 64), per_row(sh.cpu(), 256, pb.M, 64), relu=True)
    kid, info = run_ops_conv(dev, lib, pb.name, pb.M, pb.ldy, 64,
                             lambda out: O.conv(pb.a, pb.pc, relu=True, sample_affine=(sc, sh), in_affine=(isc, ish), out=out),
                             ref, A)
    assert (kid, info[:3]) == (PGEMM, (64, 0, 1))


@pytest.mark.parametrize("last", [False, True], ids=["conv4_next_affine", "last_conv4_residual_pre_relu"])
def test_pgemm_gblock_conv4(dev, lib, last):
    """conv4 + the upsampled skip with a channel drop (256 -> 128): with the next block's ccbn + ReLU as a second output, or (last
    block) the output BN folded in front of the residual, + ReLU."""
    O = ops()
    N, H, W, K = 2, 16, 16, 128
    pb = pw_problem(dev, "gblock_conv4_%d" % last, N, 64, H, W, K)
    skip, skip_h = skip_tensor(dev, pb.gen, N * (H // 2) * (W // 2), 256)
    sact = O.Act(skip, N, 1, H // 2, W // 2, K)
    acc, mag = conv_acc(pb.x, pb.w, pb.k, pb.s, pb.p)
    r = nearest_up2(skip_h, N, H, W, K)
    if last:
        ref, A = epilogue(acc, mag, pb.pc.scale.cpu(), pb.pc.shift.cpu(), residual=r, pre=True, relu=True)
        call = lambda out: O.conv(pb.a, pb.pc, residual=sact, relu=True, residual_up=True, residual_pre=True, out=out)
        kid, info = run_ops_conv(dev, lib, pb.name, pb.M, pb.ldy, K, call, ref, A)
    else:
        sc2, sh2 = affine_views(dev, pb.gen, N, K)
        v, A = epilogue(acc, mag, pb.pc.scale.cpu(), pb.pc.shift.cpu(), residual=r)
        ref2, A2 = second_output(v, A, per_row(sc2.cpu(), H * W, pb.M, K), per_row(sh2.cpu(), H * W, pb.M, K))
        call = lambda out: O.conv(pb.a, pb.pc, residual=sact, residual_up=True, next_affine=(sc2, sh2), out=out)
        kid, info = run_ops_conv(dev, lib, pb.name, pb.M, pb.ldy, K, call, v, A, ref2, A2)
    assert (kid, info[:3]) == (PGEMM, (128, 0, 1))


# ---------------------------------------------------------------------------------------------
# GEMM entry points: per-sample affine rows, second output, the two-operand GEMM
# ---------------------------------------------------------------------------------------------
def gemm_operands(name, M, N, Kd):
    g = gen(name)
    Kp = rup(Kd, 8)
    A = torch.zeros(M, Kp, dtype=torch.float16)
    A[:, :Kd] = torch.randn(M, Kd, generator=g).half()
    B = torch.zeros(N, Kp, dtype=torch.float16)
    B[:, :Kd] = (torch.randn(N, Kd, generator=g) / Kd ** 0.5).half()
    return g, A, B


@pytest.mark.parametrize("rows", [128, 256])
@pytest.mark.parametrize("dual", [False, True], ids=["d", "d_d2"])
def test_gemm_per_sample_rows_against_fp64(dev, lib, rows, dual):
    O = ops()
    M, N, Kd = 3 * 256, 96, 136
    g, A, B = gemm_operands("gemm_aff%d" % rows, M, N, Kd)
    sc, sh = affine_views(dev, g, M // rows, N)
    R = torch.randn(M, N + 8, generator=g).half()
    acc, mag = gemm_acc(A, B)
    v, Av = epilogue(acc, mag, per_row(sc.cpu(), rows, M, N), per_row(sh.cpu(), rows, M, N), residual=R[:, :N].double(), relu=True)
    ldd = rup(N, 8)
    buf, out = sentinel_buf(dev, M, ldd)
    kw = dict(residual=R.to(dev), relu=True, aff_rows=rows, out=out)
    if dual:
        sc2, sh2 = affine_views(dev, g, M // rows, N)
        kw["next_affine"] = (sc2, sh2, rows)
    res = O.gemm(A.to(dev), B.to(dev), sc, sh, M, N, Kd, **kw)
    torch.cuda.synchronize()
    kid, info = last_kernel(lib)
    assert (kid, info[:3]) == (PGEMM, (128, 0, int(dual)))
    name = "pgemm gemm aff_rows %d%s" % (rows, " +d2" if dual else "")
    check_rows(name, buf, out, M, N, v, Av)
    if dual:
        ref2, A2 = second_output(v, Av, per_row(sc2.cpu(), rows, M, N), per_row(sh2.cpu(), rows, M, N))
        assert_within(name + " d2", res[1][:, :N], ref2, A2, True)
    buf2, out2 = sentinel_buf(dev, M, ldd)
    kw["out"] = out2
    O.gemm(A.to(dev), B.to(dev), sc, sh, M, N, Kd, **kw)
    torch.cuda.synchronize()
    assert same_bits(out2, out)


@pytest.mark.parametrize("kd,k2", [(64, 64), (128, 256), (200, 72)])
def test_gemm2_against_fp64(dev, lib, kd, k2):
    """b2_gemm2_f16: the type-B shortcut projection accumulated into the block-closing 1x1 GEMM."""
    O = ops()
    M, N = 384, 200
    g, A, B = gemm_operands("gemm2_%d_%d" % (kd, k2), M, N, kd)
    _, A2, B2 = gemm_operands("gemm2b_%d_%d" % (kd, k2), M, N, k2)
    sc, sh = torch.rand(N, generator=g) + 0.5, torch.randn(N, generator=g)
    R = torch.randn(M, rup(N, 8), generator=g).half()
    acc1, mag1 = gemm_acc(A, B)
    acc2, mag2 = gemm_acc(A2, B2)
    ref, Aref = epilogue(acc1 + acc2, mag1 + mag2, sc, sh, residual=R[:, :N].double(), relu=True)
    ldd = rup(N, 8)
    buf, out = sentinel_buf(dev, M, ldd)
    args = (A.to(dev), B.to(dev), sc.to(dev), sh.to(dev), M, N, kd)
    second = (A2.to(dev), B2.to(dev), k2)
    O.gemm(*args, residual=R.to(dev), relu=True, out=out, second=second)
    torch.cuda.synchronize()
    kid, info = last_kernel(lib)
    assert (kid, info[:3]) == (PGEMM, (128, 0, 0))
    check_rows("pgemm gemm2 Kd%d K2%d" % (kd, k2), buf, out, M, N, ref, Aref)
    buf2, out2 = sentinel_buf(dev, M, ldd)
    O.gemm(*args, residual=R.to(dev), relu=True, out=out2, second=second)
    torch.cuda.synchronize()
    assert same_bits(out2, out)


# ---------------------------------------------------------------------------------------------
# pitch contract: columns [K, ldy) of an fp16 y are zero whatever the residual holds past K; ldr < ldy reads nothing past a row
# ---------------------------------------------------------------------------------------------
# family: (shape N, Cin, T, H, W, kernel, padding, K of (a) / (b) / (c), knobs, expected kernel id)
S33, P33 = (1, 3, 3), (0, 1, 1)
FAMILIES = {
    "slab64": dict(shape=(1, 64, 1, 12, 14), k=S33, p=P33, Ks=(60, 60, 64), kid=SLAB),
    "slab128": dict(shape=(1, 64, 1, 12, 14), k=S33, p=P33, Ks=(124, 124, 128), kid=SLAB),
    "flex": dict(shape=(1, 64, 1, 10, 12), k=S33, p=P33, Ks=(140, 132, 144), kid=SLAB),
    "n16": dict(shape=(1, 64, 1, 20, 20), k=S33, p=P33, Ks=(12, 4, 8), kid=SLAB),
    "tstack": dict(shape=(2, 64, 5, 6, 6), k=(3, 1, 1), p=(1, 0, 0), Ks=(60, 36, 32), kid=TSTACK),
    "igemm_gather": dict(shape=(1, 64, 1, 12, 14), k=S33, p=P33, Ks=(60, 60, 64), kid=IGEMM),
    "igemm_tma": dict(shape=(2, 64, 1, 8, 16), k=(1, 1, 1), p=(0, 0, 0), Ks=(60, 60, 64), kid=IGEMM),
    "pgemm": dict(shape=(2, 64, 1, 8, 16), k=(1, 1, 1), p=(0, 0, 0), Ks=(60, 60, 64), kid=PGEMM),
    "pgemm_gan": dict(shape=(2, 64, 1, 8, 16), k=(1, 1, 1), p=(0, 0, 0), Ks=(60, 60, 64), kid=PGEMM),
    "densem": dict(shape=(1, 64, 1, 6, 6), k=S33, p=P33, Ks=(60, 60, 64), kid=DENSEM),
}


def pitches(fam, sub, K):
    """(ldy, ldr) of sub-case a / b / c: (a) ldy = round_up(K, 8), a skip 12 columns wider than K with data in [K, ldr);
    (b) ldr = round_up(K, 8) < ldy (80 / 64 for K = 60); (c) K a multiple of 8 written with a wider pitch (96 for K = 64), the
    residual 8 columns wider than K.  The N = 16 tile needs ldy <= 16 and the temporal stack ldy <= 64: their wide pitch is that;
    the flex tiles whose weight stages and accumulators fit in shared memory here are at most 160 columns wide."""
    wide = {"n16": 16, "tstack": 64, "flex": 160}.get(fam)
    if sub == "a":
        return rup(K, 8), K + 12
    if sub == "b":
        return wide or rup(K, 8) + 16, rup(K, 8)
    return wide or K + 32, K + 8


def set_family_knobs(lib, fam):
    lib.b2_debug_set_densem(-1 if fam == "densem" else 0, 0)
    if fam == "tstack":
        lib.b2_debug_set_tstack(1)
    if fam == "igemm_gather":
        lib.b2_debug_set_conv_algo(1)
    if fam in ("igemm_gather", "igemm_tma"):
        lib.b2_debug_set_gemm_algo(1)


@pytest.mark.parametrize("sub", ["a", "b", "c"])
@pytest.mark.parametrize("fam", list(FAMILIES))
def test_pitch_contract(dev, lib, fam, sub):
    f = FAMILIES[fam]
    N, Cin, T, H, W = f["shape"]
    K = f["Ks"]["abc".index(sub)]
    pb = Problem(dev, "pitch_%s_%s" % (fam, sub), N, Cin, T, H, W, K, f["k"], (1, 1, 1), f["p"], pitch=Cin)
    ldy, ldr = pitches(fam, sub, K)
    set_family_knobs(lib, fam)
    up = fam == "pgemm_gan"
    rrows = pb.M // 4 if up else pb.M
    # the residual: data in every column of its rows (past K too), followed inside the same allocation by poisoned rows
    rbuf = torch.full((rrows + 8, ldr), float("nan"), dtype=torch.float16)
    rbuf[:rrows] = torch.randn(rrows, ldr, generator=pb.gen).half()
    rd = rbuf.to(dev)
    res = rd[:rrows]
    buf, y = sentinel_buf(dev, pb.M, ldy)
    args = pb.args(y, res, relu=True)
    args.residual_up = int(up)
    rc = lib.b2_conv_ndhwc_fprop(ctypes.byref(args), None)
    assert rc == 0, _lib().last_error()
    torch.cuda.synchronize()
    kid, info = last_kernel(lib)
    if up:
        acc, mag = conv_acc(pb.x, pb.w, pb.k, pb.s, pb.p)
        ref, A = epilogue(acc, mag, pb.pc.scale.cpu(), pb.pc.shift.cpu(), residual=nearest_up2(rbuf[:rrows], N, H, W, K), relu=True)
    else:
        ref, A = conv_ref(pb.x, pb.w, pb.pc.scale, pb.pc.shift, pb.k, pb.s, pb.p, residual=rbuf[:rrows], relu=True)
    check_rows("%s pitch(%s) K%d ldy%d ldr%d" % (KIND[kid], sub, K, ldy, ldr), buf, y, pb.M, K, ref, A)
    assert kid == f["kid"], (fam, KIND[kid])
    if f["kid"] == SLAB:
        plan = slab_plan_of(lib, shape_of(pb), ldy)
        assert info == plan_info(plan)
        if fam == "n16":
            assert info[0] == 16
    if fam.startswith("pgemm"):
        assert info[:3] == (64 if ldy <= 64 else 128, 0, int(up))
    buf2, y2 = sentinel_buf(dev, pb.M, ldy)
    args2 = pb.args(y2, res, relu=True)
    args2.residual_up = int(up)
    assert lib.b2_conv_ndhwc_fprop(ctypes.byref(args2), None) == 0
    torch.cuda.synchronize()
    assert same_bits(y2, y)


def test_grouped_conv_leaves_columns_past_k_untouched(dev, lib):
    """The grouped kernel's own contract: y columns [K, ldy) are left as they were (NaN here), residual columns past K unread."""
    O = ops()
    L = _lib()
    N, T, H, W, C, groups = 1, 3, 8, 10, 64, 16
    g = gen("grouped_pitch")
    x = torch.randn(N, T, H, W, C, generator=g).half()
    wg = torch.randn(C, C // groups, 3, 3, 3, generator=g) / (27 * C // groups) ** 0.5
    bn = OF.randomize_bn_(nn.BatchNorm3d(C), 7).eval()
    pc = O.PackedGroupedConv(wg.to(dev), groups, bn=bn.to(dev), stride=(1, 1, 1), padding=(1, 1, 1))
    M, ldy, ldr = N * T * H * W, C + 32, C + 16
    rbuf = torch.full((M + 8, ldr), float("nan"), dtype=torch.float16)
    rbuf[:M] = torch.randn(M, ldr, generator=g).half()
    res = rbuf.to(dev)[:M]
    buf, y = sentinel_buf(dev, M, ldy)
    xd = x.reshape(-1, C).to(dev)
    a = L.ConvArgs()
    a.x, a.w, a.scale, a.shift, a.residual, a.y = xd.data_ptr(), pc.w.data_ptr(), pc.scale.data_ptr(), pc.shift.data_ptr(), \
        res.data_ptr(), y.data_ptr()
    a.N, a.T, a.H, a.W, a.C, a.K, a.ldy, a.ldr = N, T, H, W, C, C, ldy, ldr
    a.kt, a.kh, a.kw = 3, 3, 3
    a.st, a.sh, a.sw = 1, 1, 1
    a.pt, a.ph, a.pw = 1, 1, 1
    a.relu = 1
    assert lib.b2_conv_grouped_ndhwc_fprop(ctypes.byref(a), groups, None) == 0, L.last_error()
    torch.cuda.synchronize()
    assert last_kernel(lib)[0] == GROUPCONV
    dense = O.dense_from_grouped(wg, groups).half()
    wpk = dense.permute(0, 2, 3, 4, 1).reshape(C, 27, C)
    ref, A = conv_ref(x, wpk, pc.scale, pc.shift, (3, 3, 3), (1, 1, 1), (1, 1, 1), residual=rbuf[:M], relu=True)
    assert_within("groupconv pitch K%d ldy%d ldr%d" % (C, ldy, ldr), y[:, :C], ref, A, True)
    assert torch.isnan(y[:, C:].float()).all(), "grouped convolution wrote columns [K, ldy)"
    assert torch.isnan(buf[:PAD].float()).all() and torch.isnan(buf[PAD + M:].float()).all()
