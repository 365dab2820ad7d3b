"""GPU (-m gpu): every convolution / GEMM kernel variant, the attention kernels and the fine-tuning backward helpers against fp64,
with the kernel that ran pinned by b2_debug_last_kernel.

Variants are forced only through the library's admissibility-checked debug knobs; every case asserts which kernel (and which
tile plan) produced its result, so a change of the dispatch rules cannot silently move a case to another kernel.  The reference
is computed from exactly the operands the kernel sees (fp16 activation, packed fp16 filter read back from PackedConv.w, folded
fp32 scale / shift, fp16 residual) and every element is held to the bound of tests/kernel_ref.py.  Worst err / bound ratios are
printed per case (pytest -s)."""
import ctypes
import os
import zlib

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import functional as OF
from tests.conftest import has_h100
from tests.kernel_ref import att_bound, att_ref, conv_ref, where_worst, worst_ratio

KNOB_ENV = ("B2_CONV_ALGO", "B2_GEMM_ALGO", "B2_DENSEM_MAXM", "B2_DENSEM_S", "B2_TSTACK", "B2_SLABTS")

pytestmark = [
    pytest.mark.gpu,
    pytest.mark.skipif(not has_h100(), reason="needs an H100"),
    pytest.mark.skipif(any(os.environ.get(e) for e in KNOB_ENV),
                       reason="a dispatch override is set in the environment (%s)" % ", ".join(KNOB_ENV)),
]

# b2_debug_last_kernel ids (KID_* of csrc/b2_host.h)
STEM, SLAB, SLABTS, TSTACK, DENSEM, PGEMM, IGEMM, SIMT, ATTENTION = range(1, 10)
KIND = ["none", "stem", "slab", "slabts", "tstack", "densem", "pgemm", "igemm", "simt", "attention"]


def _lib():
    from pretorched_x_b200 import _lib as L
    return L


@pytest.fixture(autouse=True)
def lib():
    """The knobs are process-global and the other GPU files run in the same process: put every one back to its rule."""
    lib = _lib().load()
    try:
        yield lib
    finally:
        lib.b2_debug_set_conv_algo(0)
        lib.b2_debug_set_gemm_algo(0)
        lib.b2_debug_set_densem(-1, 0)
        lib.b2_debug_set_slab_mt(0)
        lib.b2_debug_set_slab_wide(-1)
        lib.b2_debug_set_tstack(-1)
        lib.b2_debug_set_slabts(-1)
        lib.b2_debug_set_attention_algo(0)


@pytest.fixture(scope="module")
def dev():
    return torch.device("cuda:0")


def last_kernel(lib):
    info = (ctypes.c_int * 5)()
    kid = lib.b2_debug_last_kernel(info)
    return kid, tuple(info)


def seed_of(name):
    return zlib.crc32(name.encode()) % 100000


def rup(v, m):
    return (v + m - 1) // m * m


def report(name, ratio):
    print("[kernel-matrix] %-60s worst err/bound %.4f" % (name, ratio))


def assert_within(name, got, ref, A, f16):
    r = worst_ratio(got, ref, A, f16)
    report(name, r)
    assert r <= 1.0, "%s: err/bound %.3f at %s" % (name, r, where_worst(got, ref, A, f16))


# ---------------------------------------------------------------------------------------------
# convolution problems
# ---------------------------------------------------------------------------------------------
class Problem:
    """One convolution with random operands: fp16 NDHWC input (pitch C, channels [Cin, C) zero), a PackedConv with a
    non-trivial folded BatchNorm (or a bias without BN), and the geometry of its output."""

    def __init__(self, dev, name, N, Cin, T, H, W, K, k, s, p, pitch=None, bias_only=False):
        from pretorched_x_b200 import ops
        self.name, self.K, self.k, self.s, self.p = name, K, k, s, p
        g = torch.Generator().manual_seed(seed_of(name))
        C = pitch or rup(Cin, 8)
        x = torch.zeros(N, T, H, W, C, dtype=torch.float16)
        x[..., :Cin] = torch.randn(N, T, H, W, Cin, generator=g).half()
        taps = k[0] * k[1] * k[2]
        wt = torch.randn((K, Cin) + tuple(k), generator=g) / (Cin * taps) ** 0.5
        if bias_only:
            bias, bn = torch.randn(K, generator=g), None
        else:
            bias, bn = None, OF.randomize_bn_(nn.BatchNorm3d(K), seed_of(name) + 1).eval()
        self.pc = ops.PackedConv(wt.to(dev), bias.to(dev) if bias is not None else None, bn.to(dev) if bn is not None else None,
                                 stride=s, padding=p, in_pitch=C)
        self.x = x
        self.a = ops.Act(x.reshape(-1, C).to(dev), N, T, H, W, Cin)
        self.To, self.Ho, self.Wo = (ops._out_dim(i, kk, ss, pp) for i, kk, ss, pp in zip((T, H, W), k, s, p))
        self.M = N * self.To * self.Ho * self.Wo
        self.ldy = rup(K, 8)
        self.w = self.pc.w.view(K, taps, C).cpu()
        self.gen = g

    def residual(self, dev, ld):
        r = torch.zeros(self.M, ld, dtype=torch.float16)
        r[:, :self.K] = torch.randn(self.M, self.K, generator=self.gen).half()
        return r.to(dev)

    def ref(self, residual=None, relu=False, base=None):
        return conv_ref(self.x, self.w, self.pc.scale, self.pc.shift, self.k, self.s, self.p,
                        residual=None if residual is None else residual.cpu(), relu=relu, base=base)

    def args(self, y, residual=None, relu=False, out_f32=False, accumulate=False):
        """b2_conv_args for an output y ([M][ldy], fp16 or fp32) -- the fp32 epilogue is only reachable this way."""
        L = _lib()
        a = L.ConvArgs()
        a.x, a.w, a.scale, a.shift = self.a.data.data_ptr(), self.pc.w.data_ptr(), self.pc.scale.data_ptr(), self.pc.shift.data_ptr()
        a.residual = residual.data_ptr() if residual is not None else None
        a.y = y.data_ptr()
        a.N, a.T, a.H, a.W, a.C = self.a.N, self.a.T, self.a.H, self.a.W, self.a.ld
        a.K, a.ldy, a.ldr = self.K, y.stride(0), residual.stride(0) if residual is not None else 0
        a.kt, a.kh, a.kw = self.k
        a.st, a.sh, a.sw = self.s
        a.pt, a.ph, a.pw = self.p
        a.relu, a.out_f32, a.accumulate, a.mode = int(relu), int(out_f32), int(accumulate), L.B2_CONV_AUTO
        return a


def call(lib, fn, args):
    rc = fn(ctypes.byref(args), None)
    assert rc == 0, _lib().last_error()
    torch.cuda.synchronize()


def run_f16(dev, lib, pb, residual=False, relu=True, mask=False, simt=False):
    """fp16 output through ops.conv, written into a row range of a NaN-filled buffer.  Checks the bound, the zero padding
    columns, the untouched sentinel rows, exact zeros where mask <= 0 and a bitwise-identical second call.  Returns the
    (kernel id, info) of the launch."""
    from pretorched_x_b200 import ops
    M, K, ldy = pb.M, pb.K, pb.ldy
    r = pb.residual(dev, ldy + 16) if residual else None
    ract = ops.Act(r, pb.a.N, pb.To, pb.Ho, pb.Wo, K) if residual else None
    mk = None
    if mask:
        mv = torch.randn(M, ldy + 24, generator=pb.gen).half()
        flat = mv.view(-1)
        flat[0::7] = -0.0
        flat[1::7] = torch.tensor(2.0 ** -24).half()          # smallest positive subnormal: counts as > 0
        flat[2::7] = float("nan")
        mk = ops.Act(mv.to(dev), pb.a.N, pb.To, pb.Ho, pb.Wo, K)
    pad = 3
    buf = torch.full((M + 2 * pad, ldy), float("nan"), dtype=torch.float16, device=dev)
    out = buf[pad:pad + M]
    ops.conv(pb.a, pb.pc, residual=ract, relu=relu, simt=simt, out=out, mask=mk)
    torch.cuda.synchronize()
    probe = last_kernel(lib)
    ref, A = pb.ref(residual=r, relu=relu)
    if mask:
        keep = mk.data[:, :K].cpu().float() > 0
        ref = torch.where(keep, ref, torch.zeros_like(ref))
        assert torch.all(out[:, :K].cpu()[~keep] == 0), "output not zero where mask <= 0"
    assert_within("%s %s" % (KIND[probe[0]], pb.name), out[:, :K], ref, A, True)
    if ldy > K:
        assert torch.all(out[:, K:].cpu() == 0), "padding columns [K, ldy) not zero"
    assert torch.isnan(buf[:pad].float()).all() and torch.isnan(buf[pad + M:].float()).all(), "rows outside out= were written"
    again = torch.empty_like(out)
    ops.conv(pb.a, pb.pc, residual=ract, relu=relu, simt=simt, out=again, mask=mk)
    torch.cuda.synchronize()
    assert torch.equal(again.view(torch.int16), out.view(torch.int16)), "two identical calls differ"
    return probe


def run_f32(dev, lib, pb, ldy, accumulate, residual=False, relu=False, simt=False):
    """fp32 output through b2_conv_args (out_f32, accumulate): columns [K, ldy) are left untouched (NaN sentinel)."""
    M, K = pb.M, pb.K
    r = pb.residual(dev, rup(K, 8) + 8) if residual else None
    base = torch.randn(M, K, generator=pb.gen) if accumulate else None
    y0 = torch.full((M, ldy), float("nan"), dtype=torch.float32)
    if accumulate:
        y0[:, :K] = base
    y = y0.to(dev)
    fn = lib.b2_conv_ndhwc_fprop_simt if simt else lib.b2_conv_ndhwc_fprop
    call(lib, fn, pb.args(y, r, relu, out_f32=True, accumulate=accumulate))
    probe = last_kernel(lib)
    ref, A = pb.ref(residual=r, relu=relu, base=base)
    assert_within("%s %s f32%s" % (KIND[probe[0]], pb.name, " acc" if accumulate else ""), y[:, :K], ref, A, False)
    if ldy > K:
        assert torch.isnan(y[:, K:]).all(), "fp32 columns [K, ldy) must be left untouched"
    y2 = y0.to(dev)
    call(lib, fn, pb.args(y2, r, relu, out_f32=True, accumulate=accumulate))
    assert torch.equal(y2.view(torch.int32), y.view(torch.int32)), "two identical calls differ"
    return probe


# ---------------------------------------------------------------------------------------------
# implicit GEMM (gather and 1x1 TMA modes) and the CUDA-core cross-check
# ---------------------------------------------------------------------------------------------
# name, N, Cin, pitch, T, H, W, K, kernel, stride, padding
IGEMM_CASES = [
    ("3x3x3_s1_c72_k40", 1, 72, 72, 3, 5, 7, 40, (3, 3, 3), (1, 1, 1), (1, 1, 1)),
    ("3x3x3_s2_c200_k200", 1, 200, 200, 4, 9, 9, 200, (3, 3, 3), (2, 2, 2), (1, 1, 1)),
    ("1x3x3_s1_c256_k130_m256", 2, 256, 256, 2, 8, 8, 130, (1, 3, 3), (1, 1, 1), (0, 1, 1)),
    ("1x3x3_s2_c8_k64", 3, 8, 8, 1, 15, 17, 64, (1, 3, 3), (1, 2, 2), (0, 1, 1)),
    ("3x1x1_c72_k72_m129", 1, 72, 72, 3, 43, 1, 72, (3, 1, 1), (1, 1, 1), (1, 0, 0)),
    ("7x1x1_c200_k64_m127", 1, 200, 200, 127, 1, 1, 64, (7, 1, 1), (1, 1, 1), (3, 0, 0)),
    ("3x3_s2_3ch_pitch8_k64", 2, 3, 8, 2, 33, 31, 64, (1, 3, 3), (1, 2, 2), (0, 1, 1)),
    ("1x1_s2_c256_k96", 2, 256, 256, 3, 9, 9, 96, (1, 1, 1), (2, 2, 2), (0, 0, 0)),
    ("T1_kt3_c72_k64", 2, 72, 72, 1, 6, 6, 64, (3, 3, 3), (1, 1, 1), (1, 1, 1)),
    ("one_output_pixel_c256_k200", 1, 256, 256, 1, 1, 1, 200, (3, 3, 3), (1, 1, 1), (1, 1, 1)),
    ("three_clips_c8_k24", 3, 8, 8, 2, 5, 5, 24, (3, 3, 3), (1, 1, 1), (1, 1, 1)),
]
EPILOGUES = ["f16_res_relu", "f16_mask_res", "f32_res", "f32_acc_pad"]


def make(dev, case, **kw):
    name, N, Cin, pitch, T, H, W, K, k, s, p = case
    return Problem(dev, name, N, Cin, T, H, W, K, k, s, p, pitch=pitch, **kw)


def run_epilogue(dev, lib, pb, epi, simt=False):
    if epi == "f16_res_relu":
        return run_f16(dev, lib, pb, residual=True, relu=True, simt=simt), pb.ldy, 0
    if epi == "f16_mask_res":
        return run_f16(dev, lib, pb, residual=True, relu=False, mask=True), pb.ldy, 1
    if epi == "f32_res":                       # ldy == K (odd K included)
        return run_f32(dev, lib, pb, pb.K, False, residual=True, relu=True, simt=simt), pb.K, 0
    return run_f32(dev, lib, pb, pb.K + 3, True, residual=True, simt=simt), pb.K, 0


@pytest.mark.parametrize("epi", EPILOGUES)
@pytest.mark.parametrize("case", IGEMM_CASES, ids=[c[0] for c in IGEMM_CASES])
def test_igemm_against_fp64(dev, lib, case, epi):
    lib.b2_debug_set_conv_algo(1)
    lib.b2_debug_set_gemm_algo(1)
    pb = make(dev, case)
    (kid, info), width, masked = run_epilogue(dev, lib, pb, epi)
    assert kid == IGEMM and info[:2] == (64 if width <= 64 else 128, masked)


# 1x1x1 stride-1 convolutions: A is the activation matrix itself (TMA operand)
TMA_CASES = [
    ("1x1_tma_c72_k200_m189", 1, 72, 72, 3, 7, 9, 200, (1, 1, 1), (1, 1, 1), (0, 0, 0)),
    ("1x1_tma_c256_k64_m256", 2, 256, 256, 2, 8, 8, 64, (1, 1, 1), (1, 1, 1), (0, 0, 0)),
    ("1x1_tma_c8_k33_m1", 1, 8, 8, 1, 1, 1, 33, (1, 1, 1), (1, 1, 1), (0, 0, 0)),
]


@pytest.mark.parametrize("case", TMA_CASES, ids=[c[0] for c in TMA_CASES])
def test_pointwise_pgemm_and_tma_igemm_against_fp64(dev, lib, case):
    pb = make(dev, case)
    bn = 64 if pb.ldy <= 64 else 128
    assert run_f16(dev, lib, pb, residual=True, relu=True) == (PGEMM, (bn, 0, 0, 0, 0))
    assert run_f16(dev, lib, pb, residual=True, relu=False, mask=True) == (PGEMM, (64, 1, 0, 0, 0))
    assert run_f32(dev, lib, pb, pb.K + 1, True, residual=True)[0] == IGEMM      # fp32 output never takes the persistent GEMM
    lib.b2_debug_set_gemm_algo(1)
    assert run_f16(dev, lib, pb, residual=True, relu=True) == (IGEMM, (bn, 0, 0, 0, 0))
    assert run_f16(dev, lib, pb, residual=True, relu=False, mask=True) == (IGEMM, (bn, 1, 0, 0, 0))
    assert run_f32(dev, lib, pb, pb.K, False, residual=True, relu=True) == (IGEMM, (64 if pb.K <= 64 else 128, 0, 0, 0, 0))


SIMT_CASES = [IGEMM_CASES[i] for i in (0, 1, 3, 6, 9)]


@pytest.mark.parametrize("epi", ["f16_res_relu", "f32_res", "f32_acc_pad"])
@pytest.mark.parametrize("case", SIMT_CASES, ids=[c[0] for c in SIMT_CASES])
def test_simt_crosscheck_against_fp64(dev, lib, case, epi):
    pb = make(dev, case)
    (kid, info), _, _ = run_epilogue(dev, lib, pb, epi, simt=True)
    assert kid == SIMT


# ---------------------------------------------------------------------------------------------
# dense-M split-K cluster kernel: every admissible cluster split S of every N tile
# ---------------------------------------------------------------------------------------------
def densem_bn(width):
    """N tile of densem_plan (b2_conv_api.cu): least padding among 128 / 96 / 64 (ties: the widest), 32 for <= 32 columns."""
    best, waste = 128, 1 << 30
    for bn in (128, 96, 64):
        w = -(-width // bn) * bn - width
        if w < waste:
            best, waste = bn, w
    return 32 if width <= 32 else best


def densem_splits(bn, nkb):
    out = []
    for S in range(1, 9):
        per = -(-nkb // S)
        if bn % (32 * S) == 0 and S <= nkb and (S - 1) * per < nkb and (S == 1 or nkb // S >= 2):
            out.append(S)
    return out


# name, N, Cin, pitch, T, H, W, K, kernel, stride, padding, residual, relu, bias_only
DENSEM_CASES = [
    ("dm_m1_3x3x3_k32", 1, 128, 128, 1, 1, 1, 32, (3, 3, 3), (1, 1, 1), (1, 1, 1), False, True, False),
    ("dm_m3_1x3x3_k128_bias", 3, 256, 256, 1, 1, 1, 128, (1, 3, 3), (1, 1, 1), (0, 1, 1), False, False, True),
    ("dm_m127_3x3x3_s2_k96", 1, 72, 72, 1, 1, 253, 96, (3, 3, 3), (2, 2, 2), (1, 1, 1), True, True, False),
    ("dm_m129_1x1_k328", 1, 200, 200, 1, 3, 43, 328, (1, 1, 1), (1, 1, 1), (0, 0, 0), True, True, False),
    ("dm_m129_1x3x3_k64", 1, 64, 64, 1, 3, 43, 64, (1, 3, 3), (1, 1, 1), (0, 1, 1), False, True, False),
    ("dm_m1000_3x1x1_k1152_res", 5, 192, 192, 2, 10, 10, 1152, (3, 1, 1), (1, 1, 1), (1, 0, 0), True, True, False),
]


def _densem_params():
    out = []
    for c in DENSEM_CASES:
        taps = c[8][0] * c[8][1] * c[8][2]
        nkb = taps * -(-c[3] // 64)
        bn = densem_bn(rup(c[7], 8))
        for S in densem_splits(bn, nkb):
            out.append(pytest.param(c, bn, S, id="%s-S%d" % (c[0], S)))
    return out


@pytest.mark.parametrize("case,bn,S", _densem_params())
def test_densem_every_split_against_fp64(dev, lib, case, bn, S):
    pb = Problem(dev, case[0], *case[1:3], *case[4:11], pitch=case[3], bias_only=case[13])
    lib.b2_debug_set_densem(pb.M, S)
    assert run_f16(dev, lib, pb, residual=case[11], relu=case[12]) == (DENSEM, (bn, S, 0, 0, 0))


@pytest.mark.parametrize("M,N,Kd,S", [(3, 339, 2048, 4), (127, 96, 640, 3), (1, 40, 200, 1)])
def test_densem_fp32_gemm_against_fp64(dev, lib, M, N, Kd, S):
    """fp32 output through b2_gemm_f16 (the classifier heads): N tile from Ncols, forced split S."""
    from pretorched_x_b200 import ops
    g = torch.Generator().manual_seed(M * 7 + N)
    Kp = rup(Kd, 8)
    A = torch.zeros(M, Kp, dtype=torch.float16); A[:, :Kd] = torch.randn(M, Kd, generator=g).half()
    B = torch.zeros(N, Kp, dtype=torch.float16); B[:, :Kd] = (torch.randn(N, Kd, generator=g) / Kd ** 0.5).half()
    sc, sh = torch.rand(N, generator=g) + 0.5, torch.randn(N, generator=g)
    lib.b2_debug_set_densem(M, S)
    got = ops.gemm(A.to(dev), B.to(dev), sc.to(dev), sh.to(dev), M, N, Kd, out_f32=True)
    torch.cuda.synchronize()
    kid, info = last_kernel(lib)
    assert (kid, info[:2]) == (DENSEM, (densem_bn(N), S))
    Ad, Bd = A.double(), B.double()
    ref = Ad @ Bd.t() * sc.double() + sh.double()
    mag = Ad.abs() @ Bd.abs().t() * sc.double() + sh.double().abs()
    assert_within("densem gemm f32 M%d N%d K%d S%d" % (M, N, Kd, S), got, ref, mag, False)


# ---------------------------------------------------------------------------------------------
# slab kernel: rule plans, every admissible MT, the wide-N request; the temporal-group slab kernel against the slab kernel
# ---------------------------------------------------------------------------------------------
# name, N, Cin, pitch, T, H, W, K, kernel, stride, padding, residual, what the rule's plan must be (key, value)
SLAB_CASES = [
    ("slab_fixed64_3x3x3", 1, 64, 64, 3, 9, 11, 64, (3, 3, 3), (1, 1, 1), (1, 1, 1), True, ("bn", 64)),
    ("slab_fixed128_s2_c72", 1, 72, 72, 3, 13, 13, 128, (3, 3, 3), (2, 2, 2), (1, 1, 1), False, ("bn", 128)),
    ("slab_flex_144", 1, 64, 64, 2, 12, 14, 144, (1, 3, 3), (1, 1, 1), (0, 1, 1), True, ("flex", 1)),
    ("slab_flex_n16_k3", 1, 64, 64, 1, 20, 20, 3, (1, 3, 3), (1, 1, 1), (0, 1, 1), False, ("bn", 16)),
    ("slab_multiplane_7x7_192", 5, 128, 128, 3, 7, 7, 192, (1, 3, 3), (1, 1, 1), (0, 1, 1), True, ("flex", 1)),
    ("slab_wchunks_300", 1, 64, 64, 1, 5, 300, 64, (1, 3, 3), (1, 1, 1), (0, 1, 1), False, ("wchunks", 2)),
    ("slab_remapped_temporal", 2, 144, 144, 6, 10, 10, 128, (3, 1, 1), (1, 1, 1), (1, 0, 0), True, ("remapped", 1)),
    # 256 output channels: set_slab_wide(1) asks for one 256-column N tile, which the register accumulators (192 columns)
    # refuse, so the plan must stay on the fixed 128-column tile
    ("slab_wide_256", 2, 64, 64, 1, 10, 12, 256, (1, 3, 3), (1, 1, 1), (0, 1, 1), False, ("bn", 128)),
]
PLAN_KEYS = {"bn": 1, "mt": 2, "wchunks": 6, "flex": 8, "remapped": 9}


def slab_plan(lib, case):
    """b2_debug_slab_plan (host only: no launch, no GPU) of a SLAB_CASES / SLABTS_CASES convolution under the current knobs."""
    L = _lib()
    a = L.ConvArgs()
    _, N, _, pitch, T, H, W, K, k, s, p = case[:11]
    a.N, a.T, a.H, a.W, a.C, a.K, a.ldy = N, T, H, W, pitch, K, rup(K, 8)
    a.kt, a.kh, a.kw = k
    a.st, a.sh, a.sw = s
    a.pt, a.ph, a.pw = p
    out = (ctypes.c_int * 10)()
    assert lib.b2_debug_slab_plan(ctypes.byref(a), out) == 0
    return tuple(out)


def plan_info(plan):
    """The b2_debug_last_kernel info of a slab launch: {BN, MT, flex, wchunks, remapped}."""
    return (plan[1], plan[2], plan[8], plan[6], plan[9])


def _slab_params():
    """Each shape under its rule plan, under every MT that set_slab_mt can actually force on it, and (256 channels) with the
    wide-N request.  The admissible MTs come from the host-side plan, so no case is collected that would only skip."""
    lib = _lib().load()
    out = []
    try:
        for c in SLAB_CASES:
            out.append(pytest.param(c, 0, id=c[0] + "-rule"))
            for mt in (1, 2, 3, 4):
                lib.b2_debug_set_slab_mt(mt)
                if slab_plan(lib, c)[2] == mt:
                    out.append(pytest.param(c, mt, id="%s-mt%d" % (c[0], mt)))
            lib.b2_debug_set_slab_mt(0)
            if c[7] % 256 == 0:
                out.append(pytest.param(c, -1, id=c[0] + "-wide"))
    finally:
        lib.b2_debug_set_slab_mt(0)
    return out


@pytest.mark.parametrize("case,knob", _slab_params())
def test_slab_against_fp64(dev, lib, case, knob):
    lib.b2_debug_set_densem(0, 0)                         # small planes: keep them off the dense-M kernel
    lib.b2_debug_set_slabts(0)
    rule = slab_plan(lib, case)
    key, want = case[12]
    assert rule[0] == 1 and (rule[PLAN_KEYS[key]] >= want if key == "wchunks" else rule[PLAN_KEYS[key]] == want), rule
    if knob > 0:
        lib.b2_debug_set_slab_mt(knob)
    elif knob < 0:
        lib.b2_debug_set_slab_wide(1)
    plan = slab_plan(lib, case)
    assert knob <= 0 or plan[2] == knob
    pb = make(dev, case[:11])
    kid, info = run_f16(dev, lib, pb, residual=case[11], relu=True)
    assert kid == SLAB and info == plan_info(plan)


SLABTS_CASES = [
    ("slabts_c64_t5", 1, 64, 64, 5, 12, 12, 64, (3, 3, 3), (1, 1, 1), (1, 1, 1)),
    ("slabts_c32_to_48_t7_odd", 1, 32, 32, 7, 13, 19, 48, (3, 3, 3), (1, 1, 1), (1, 1, 1)),
    ("slabts_c128_to_40_t3_two_clips", 2, 128, 128, 3, 9, 10, 40, (3, 3, 3), (1, 1, 1), (1, 1, 1)),
]


@pytest.mark.parametrize("case", SLABTS_CASES, ids=[c[0] for c in SLABTS_CASES])
def test_slabts_and_slab_against_fp64(dev, lib, case):
    """The temporal-group slab kernel is asked for on shapes its rule admits (3 x kh x kw, stride 1, <= 64 output channels, no
    residual), then the plain slab kernel.  Its shared-memory budget declines every shape today: the 192-column accumulator
    staging tile (98 KB) and four 24 KB weight stages leave 29 KB for two slab stages, and a slab that covers one 128-position
    M tile plus its halo needs more than 112 positions x 128 B each.  So the slab kernel runs both times; when slabts becomes
    reachable again this test fails on the first kernel id and must be switched to expect it."""
    lib.b2_debug_set_densem(0, 0)
    pb = make(dev, case)
    lib.b2_debug_set_slabts(1)
    kid, info = run_f16(dev, lib, pb, relu=True)
    assert kid == SLAB and info == plan_info(slab_plan(lib, case))
    lib.b2_debug_set_slabts(0)
    kid, info = run_f16(dev, lib, pb, relu=True)
    assert kid == SLAB and info == plan_info(slab_plan(lib, case))


def test_tstack_and_stem_probes(dev, lib):
    from pretorched_x_b200 import engine, ops
    lib.b2_debug_set_densem(0, 0)
    lib.b2_debug_set_tstack(1)
    pb = Problem(dev, "tstack_probe", 2, 64, 5, 6, 6, 64, (3, 1, 1), (1, 1, 1), (1, 0, 0))
    assert run_f16(dev, lib, pb, relu=True)[0] == TSTACK
    conv = nn.Conv3d(3, 64, 7, stride=(1, 2, 2), padding=3, bias=False).to(dev)
    engine.conv_bn_act(conv, None, ops.from_ncdhw(torch.randn(1, 3, 4, 32, 32, device=dev)), relu=True)
    torch.cuda.synchronize()
    kid, info = last_kernel(lib)
    assert kid == STEM and info[0] == lib.b2_debug_last_stem_rows()


# ---------------------------------------------------------------------------------------------
# non-local attention
# ---------------------------------------------------------------------------------------------
# mode, two_pass knob, B, Nq, Nk, d, dv
ATT_CASES = [
    (0, 0, 1, 128, 128, 64, 64), (0, 0, 3, 200, 50, 128, 192), (0, 0, 1, 65, 17, 256, 128), (0, 0, 3, 300, 129, 192, 256),
    (0, 0, 1, 129, 129, 512, 64), (0, 1, 3, 200, 64, 64, 192), (0, 1, 1, 70, 65, 256, 256), (0, 1, 3, 260, 65, 128, 128),
    (1, 0, 1, 128, 128, 64, 64), (1, 0, 3, 260, 65, 128, 192), (1, 0, 1, 100, 17, 512, 256),
    (2, 0, 3, 129, 129, 64, 128), (2, 0, 1, 256, 64, 256, 64), (2, 0, 3, 99, 17, 192, 192),
]


def att_operands(dev, B, Nq, Nk, d, dv, seed):
    """q in one wide matrix, k | v in another (the sub-sampled phi | g projection), both with a pitch wider than their use."""
    g = torch.Generator().manual_seed(seed)
    qm = (torch.randn(B * Nq, d + 40, generator=g) * 0.3).half()
    kv = torch.randn(B * Nk, d + dv + 24, generator=g).half()
    kv[:, :d] = (kv[:, :d].float() * 0.3).half()
    return qm, kv


@pytest.mark.parametrize("case", ATT_CASES, ids=["m%d%s_B%d_q%d_k%d_d%d_dv%d" % (c[0], "tp" if c[1] else "", *c[2:]) for c in ATT_CASES])
def test_attention_against_fp64(dev, lib, case):
    from pretorched_x_b200 import ops
    mode, two_pass, B, Nq, Nk, d, dv = case
    qm, kv = att_operands(dev, B, Nq, Nk, d, dv, seed_of(str(case)))
    lib.b2_debug_set_attention_algo(two_pass)
    qd, kvd = qm.to(dev), kv.to(dev)
    o = ops.attention(qd, kvd, kvd[:, d:], d, dv, B, Nq, Nk, mode=mode)
    torch.cuda.synchronize()
    kid, info = last_kernel(lib)
    online = int(mode == 0 and d <= 256 and not two_pass)
    assert (kid, info[:2]) == (ATTENTION, (online, 128 if online and dv % 128 == 0 else 64))
    ref, pv = att_ref(qm[:, :d], kv[:, :d], kv[:, d:d + dv], B, Nq, Nk, mode)
    err = (o[:, :dv].cpu().double() - ref).abs()
    ratio = float((err / att_bound(ref, pv, kv[:, d:d + dv], B, Nq, Nk, mode)).max())
    report("attention %s" % (case,), ratio)
    assert ratio <= 1.0
    o2 = ops.attention(qd, kvd, kvd[:, d:], d, dv, B, Nq, Nk, mode=mode)
    assert torch.equal(o2.view(torch.int16), o.view(torch.int16))


def test_attention_concat_mode_row_without_positive_logits_is_zero(dev, lib):
    from pretorched_x_b200 import ops
    B, Nq, Nk, d, dv = 2, 130, 33, 64, 64
    qm, kv = att_operands(dev, B, Nq, Nk, d, dv, 9)
    kv[:Nk, :d] = kv[:Nk, :d].abs()              # sample 0: keys >= 0 ...
    qm[5, :d] = -qm[5, :d].abs()                 # ... and a query <= 0: every logit of row 5 is <= 0
    kvd = kv.to(dev)
    o = ops.attention(qm.to(dev), kvd, kvd[:, d:], d, dv, B, Nq, Nk, mode=2)
    torch.cuda.synchronize()
    assert last_kernel(lib)[0] == ATTENTION
    assert torch.all(o[5, :dv].cpu() == 0)
    assert o[6, :dv].abs().max() > 0


# ---------------------------------------------------------------------------------------------
# fine-tuning backward helpers
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows,C,ld,inv", [(100, 40, 48, None), (129, 72, 72, 2.0 ** -9), (3 * 2 ** 20 + 1, 24, 32, 2.0 ** -7),
                                           (257, 8, 16, None)])
def test_colsum_against_fp64(dev, rows, C, ld, inv):
    from pretorched_x_b200 import ops
    g = torch.Generator(device=dev).manual_seed(rows)
    data = torch.zeros(rows, ld, dtype=torch.float16, device=dev)
    data[:, :C] = (torch.randn(rows, C, generator=g, device=dev) * 30).half()
    data[:, C:] = float("nan")                   # columns past C must not be read
    act = ops.Act(data, rows, 1, 1, 1, C)
    inv_t = torch.tensor([inv], dtype=torch.float32, device=dev) if inv is not None else None
    got = ops.colsum(act, inv_t).double().cpu()
    s = 1.0 if inv is None else inv
    ref = data[:, :C].double().sum(dim=0).cpu() * s
    mag = data[:, :C].double().abs().sum(dim=0).cpu() * s
    chain = rows / (128 * 8) + 8 + 128 + 2        # longest fp32 addition chain of the two-pass reduction
    err = (got - ref).abs()
    assert float((err / (chain * 2.0 ** -24 * mag + 2.0 ** -24)).max()) <= 1.0


@pytest.mark.parametrize("peak,want_k", [(2.0 ** 7, 0), (255.99, 0), (2.0 ** -60, 67), (2.0 ** 120, -113), (0.0, 0),
                                         (float("nan"), 0), (float("inf"), 0)])
def test_loss_scale_exact(dev, peak, want_k):
    from pretorched_x_b200 import ops
    gf = torch.zeros(3, 50, dtype=torch.float32)
    finite = peak == peak and peak not in (0.0, float("inf"))
    if finite:
        gf[1, 7] = -peak
        gf[2, 3] = peak / 3
    elif peak != 0.0:                            # a non-finite entry among ordinary ones
        gf[0, 0] = 1.0
        gf[2, 49] = peak
    pair = torch.empty(2, dtype=torch.float32, device=dev)
    ops.loss_scale_(gf.to(dev), pair)
    got = pair.cpu().tolist()
    assert got == [2.0 ** want_k, 2.0 ** -want_k]
    if finite:                                   # the scaled peak sits in [2^7, 2^8): finite in fp16
        assert 2.0 ** 7 <= peak * got[0] < 2.0 ** 8


@pytest.mark.parametrize("N,S,C,ld", [(2, 7, 40, 48), (3, 49, 24, 24), (1, 100, 8, 16)])
def test_avgpool_global_backward_against_fp64(dev, lib, N, S, C, ld):
    g = torch.Generator().manual_seed(N * S)
    gf = torch.randn(N, C + 5, generator=g)                # ldf > C
    out = torch.randn(N * S, ld, generator=g).half()
    flat = out.view(-1)
    flat[0::5] = -0.0
    flat[1::5] = torch.tensor(2.0 ** -24).half()           # positive subnormal: the ReLU let it through
    out[:, C:] = 1.0
    pair = torch.tensor([2.0 ** 5, 2.0 ** -5], dtype=torch.float32)
    gfd, paird, outd = gf.to(dev), pair.to(dev), out.to(dev)
    y = torch.full_like(outd, float("nan"))
    rc = lib.b2_avgpool_global_backward(gfd.data_ptr(), gfd.stride(0), paird.data_ptr(), outd.data_ptr(), y.data_ptr(), N, S, C, ld,
                                        None)
    assert rc == 0, _lib().last_error()
    got = y.cpu()
    keep = out[:, :C].float() > 0
    ref = gf[:, :C].double().repeat_interleave(S, dim=0) * 2.0 ** 5 / S
    ref = torch.where(keep, ref, torch.zeros_like(ref))
    assert torch.all(got[:, :C][~keep] == 0) and torch.all(got[:, C:] == 0)
    err = (got[:, :C].double() - ref).abs()
    assert float((err / (2.0 ** -11 * ref.abs() + 2.0 ** -24)).max()) <= 1.0


@pytest.mark.parametrize("size,stride,C,channels,ld", [((3, 7, 9), 2, 16, 8, 24), ((5, 5, 5), 1, 24, 24, 24), ((1, 9, 7), 2, 40, 40, 48),
                                                      ((4, 6, 10), 2, 8, 8, 8)])
def test_zero_insert_bit_exact(dev, size, stride, C, channels, ld):
    from pretorched_x_b200 import ops
    from tests.test_finetune_cpu import zero_insert as zero_insert_ref
    N = 2
    lo = tuple((n - 1) // stride + 1 for n in size)
    gen = torch.Generator().manual_seed(sum(size) + C)
    gl = torch.randn(N, C, *lo, generator=gen).half()
    ldg = C + 8
    data = torch.zeros(N, *lo, ldg, dtype=torch.float16)
    data[..., :C] = gl.permute(0, 2, 3, 4, 1)
    data[..., C:] = float("nan")                   # past C: never read
    act = ops.Act(data.reshape(-1, ldg).to(dev), N, *lo, C)
    y = ops.zero_insert(act, *size, stride, channels=channels, ld=ld)
    want = zero_insert_ref(gl.float(), size, stride, channels=channels).permute(0, 2, 3, 4, 1).reshape(-1, channels)
    got = y.data.cpu()
    assert torch.equal(got[:, :channels].float(), want) and torch.all(got[:, channels:] == 0)
