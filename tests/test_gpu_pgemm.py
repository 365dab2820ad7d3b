"""GPU (-m gpu): the persistent GEMM (pgemm_kernel, b2_pgemm.cuh) that runs every 1x1x1 convolution, against a CPU fp32
reference on the same fp16-rounded operands.  Tolerance 2e-3 of max|reference| (fp32 accumulate, one fp16 rounding).

Each case pins the kernel with b2_debug_last_gemm_path() == 2 and picks shapes for one property of it: the 64- and 128-wide
N tiles (64 when the output pitch is <= 64), ragged M, output pitches that are not a multiple of the N tile, padding columns,
K from one to 32 blocks, more tiles than SMs (ring, residual and staging buffer phases wrap), the fused second operand pair,
and every epilogue variant (residual, ReLU, per-sample affines, upsampled / pre-affine residual, second output, input affine,
ReLU-derivative mask)."""
import ctypes

import pytest
import torch
import torch.nn.functional as F

from pretorched_x_b200 import _lib, ops
from pretorched_x_b200.ops import Act

pytestmark = pytest.mark.gpu
TOL = 2e-3


@pytest.fixture(scope="module")
def lib():
    assert torch.cuda.is_available(), "GPU tests need an H100"
    lib = _lib.load()
    lib.b2_debug_last_gemm_path.restype = ctypes.c_int
    return lib


def h(x):
    return x.half().float()


def rel(got, ref):
    return (got.double().cpu() - ref.double()).abs().max().item() / max(ref.abs().max().item(), 1e-12)


def operands(g, M, N, K):
    return h(torch.randn(M, K, generator=g)), h(torch.randn(N, K, generator=g) / K ** 0.5)


# M, N, K, ldd (output pitch, >= N), residual, relu
GEMM_CASES = [
    (1000, 64, 64, 64, True, True),          # BN = 64, ragged M, one K block
    (1000, 256, 2048, 256, False, True),     # BN = 128, 32 K blocks
    (777, 192, 256, 192, True, False),       # pitch 192: the second N tile is half outside the output
    (300, 320, 64, 320, False, False),       # pitch 320
    (513, 200, 128, 256, True, True),        # Ncols 200 < pitch 256: columns [200, 256) are written as zero
    (40000, 256, 64, 256, True, True),       # 626 tiles over the SMs: buffer parities wrap many times (layer1 conv3)
    (40000, 64, 256, 64, True, True),        # 313 tiles of the 64-wide instance (layer1 conv1 shape)
]


@pytest.mark.parametrize("M,N,K,ldd,res,relu", GEMM_CASES)
def test_gemm(lib, M, N, K, ldd, res, relu):
    g = torch.Generator().manual_seed(M + N + K)
    A, B = operands(g, M, N, K)
    sc, sh = torch.rand(N, generator=g) + 0.5, torch.randn(N, generator=g)
    R = h(torch.randn(M, N, generator=g)) if res else None
    want = A @ B.t() * sc + sh + (R if res else 0.0)
    want = F.relu(want) if relu else want
    out = torch.full((M, ldd), float("nan"), dtype=torch.float16, device="cuda")
    got = ops.gemm(A.half().cuda(), B.half().cuda(), sc.cuda(), sh.cuda(), M, N, K, relu=relu, out=out,
                   residual=R.half().cuda() if res else None)
    assert lib.b2_debug_last_gemm_path() == 2
    assert rel(got[:, :N].float(), want) <= TOL
    if ldd > N:
        assert float(got[:, N:].float().abs().max()) == 0.0


@pytest.mark.parametrize("M,N,K1,K2", [(5000, 256, 64, 64), (3000, 512, 128, 256), (700, 64, 256, 512)])
def test_two_operand_gemm(lib, M, N, K1, K2):
    """conv3 + type-B projection: both operand pairs into one accumulator."""
    g = torch.Generator().manual_seed(K1 + K2)
    A1, B1 = operands(g, M, N, K1)
    A2, B2 = operands(g, M, N, K2)
    sh = torch.randn(N, generator=g)
    want = F.relu(A1 @ B1.t() + A2 @ B2.t() + sh)
    got = ops.gemm(A1.half().cuda(), B1.half().cuda(), torch.ones(N, device="cuda"), sh.cuda(), M, N, K1, relu=True,
                   second=(A2.half().cuda(), B2.half().cuda(), K2))
    assert lib.b2_debug_last_gemm_path() == 2
    assert rel(got.float(), want) <= TOL


@pytest.mark.parametrize("N", [64, 200])
def test_per_sample_affine_and_second_output(lib, N):
    """Per-sample scale/shift (aff_rows) and the second output relu(y * scale2 + shift2) with its own per-sample rows."""
    g = torch.Generator().manual_seed(N)
    S, rows, K = 5, 256, 192
    M = S * rows
    A, B = operands(g, M, N, K)
    R = h(torch.randn(M, N, generator=g))
    pitch = N + 8
    aff = torch.randn(S, 4 * pitch, generator=g)
    sc, sh, sc2, sh2 = (aff[:, i * pitch:i * pitch + N] for i in range(4))
    want = F.relu((A @ B.t()).view(S, rows, N) * sc[:, None] + sh[:, None] + R.view(S, rows, N))
    want2 = F.relu(want * sc2[:, None] + sh2[:, None])
    affd = aff.cuda()
    scd, shd, sc2d, sh2d = (affd[:, i * pitch:i * pitch + N] for i in range(4))
    got, got2 = ops.gemm(A.half().cuda(), B.half().cuda(), scd, shd, M, N, K, relu=True, residual=R.half().cuda(),
                         aff_rows=rows, next_affine=(sc2d, sh2d, rows))
    assert lib.b2_debug_last_gemm_path() == 2
    assert rel(got[:, :N].float(), want.view(M, N)) <= TOL
    assert rel(got2[:, :N].float(), want2.view(M, N)) <= TOL


@pytest.mark.parametrize("N", [64, 512])
def test_masked_gemm(lib, N):
    """ReLU-derivative mask of the fine-tuning backward: zero where mask <= 0, ragged M."""
    g = torch.Generator().manual_seed(3 * N)
    M, K = 2000, 1024
    A, B = operands(g, M, N, K)
    R = h(torch.randn(M, N, generator=g))
    mask = torch.randn(M, N, generator=g).half()
    one, zero = torch.ones(N, device="cuda"), torch.zeros(N, device="cuda")
    got = ops.gemm(A.half().cuda(), B.half().cuda(), one, zero, M, N, K, residual=R.half().cuda(), mask=mask.cuda())
    assert lib.b2_debug_last_gemm_path() == 2
    want = (A @ B.t() + R) * (mask.float() > 0)
    assert rel(got.float(), want) <= TOL
    assert bool((got.cpu()[mask <= 0] == 0).all())


def nhwc(x16):
    N, C, H, W = x16.shape
    return Act(x16.permute(0, 2, 3, 1).contiguous().view(N * H * W, C).cuda(), N, 1, H, W, C)


def to_nchw(a):
    return a.data[:, :a.C].float().view(a.N, a.H, a.W, a.C).permute(0, 3, 1, 2).cpu()


# N, C, H, W, K: output width W >= 128 (a tile is half an image row of sources) and W <= 64 (whole row pairs); K 64 and 128+
@pytest.mark.parametrize("shape", [(2, 64, 4, 256, 128), (3, 128, 16, 32, 200), (2, 64, 8, 64, 64)])
@pytest.mark.parametrize("pre", [False, True])
def test_upsampled_residual_with_second_output(lib, shape, pre):
    """GBlock close: conv1x1(t) + nearest-2x(x) read at low resolution (res_up), before (res_pre) or after the affine, and the
    next block's ccbn + ReLU as a second output."""
    N, C, H, W, K = shape
    g = torch.Generator().manual_seed(H * W + K)
    t = torch.randn(N, C, H, W, generator=g).half()
    x = torch.randn(N, K + 8, H // 2, W // 2, generator=g).half()
    w = torch.randn(K, C, 1, 1, generator=g) / C ** 0.5
    pc = ops.PackedConv(w.cuda(), None, None, (1, 1, 1), (0, 0, 0), in_pitch=C)
    pc.scale = (torch.rand(K, generator=g) + 0.5).cuda()
    pc.shift = torch.randn(K, generator=g).cuda()
    aff = torch.randn(N, 2 * K + 8, generator=g)
    sc2, sh2 = aff[:, :K], aff[:, K + 8:]
    affd = aff.cuda()
    out, nxt = ops.conv(nhwc(t), pc, residual=nhwc(x), relu=True, residual_up=True, residual_pre=pre,
                        next_affine=(affd[:, :K], affd[:, K + 8:]))
    assert lib.b2_debug_last_gemm_path() == 2
    acc = F.conv2d(t.float(), w.half().float())
    skip = F.interpolate(x.float()[:, :K], scale_factor=2)
    s_, b_ = pc.scale.cpu().view(1, K, 1, 1), pc.shift.cpu().view(1, K, 1, 1)
    want = F.relu((acc + skip) * s_ + b_) if pre else F.relu(acc * s_ + b_ + skip)
    want2 = F.relu(want * sc2.view(N, K, 1, 1) + sh2.view(N, K, 1, 1))
    assert rel(to_nchw(out), want) <= TOL and rel(to_nchw(nxt), want2) <= TOL


@pytest.mark.parametrize("K", [64, 256])
def test_input_affine(lib, K):
    """relu(x * in_scale[n] + in_shift[n]) applied to the A operand in shared memory (GBlock bn1 + ReLU), per sample."""
    N, C, H, W = 3, 192, 16, 16
    g = torch.Generator().manual_seed(K)
    x = torch.randn(N, C, H, W, generator=g).half()
    w = torch.randn(K, C, 1, 1, generator=g) / C ** 0.5
    iaff = torch.randn(N, 2 * C, generator=g)
    isc, ish = iaff[:, :C], iaff[:, C:]
    pc = ops.PackedConv(w.cuda(), None, None, (1, 1, 1), (0, 0, 0), in_pitch=C)
    iaffd = iaff.cuda()
    out = ops.conv(nhwc(x), pc, relu=False, in_affine=(iaffd[:, :C], iaffd[:, C:]))
    assert lib.b2_debug_last_gemm_path() == 2
    xin = h(F.relu(x.float() * isc.view(N, C, 1, 1) + ish.view(N, C, 1, 1)))
    want = F.conv2d(xin, w.half().float())
    assert rel(to_nchw(out), want) <= TOL
