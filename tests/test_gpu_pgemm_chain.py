"""GPU (-m gpu): the chained persistent GEMM (pgemm_chain_kernel, b2_gemm_chain_f16) -- a bottleneck's closing 1x1x1 GEMM with
the next block's conv1 computed from the on-chip block output.

Every case pins the chained kernel (b2_debug_last_kernel) and holds both outputs to two references: bit equality with the two
stand-alone launches it replaces (b2_gemm_f16 / b2_gemm2_f16, then b2_gemm_f16 on the stored y), and the fp64 bound of
tests/kernel_ref.py (y from the operands, h1 from the y the kernel stored).  The resnet3d50 forward test checks the engine's
pairing: chained and unchained trunks agree bit for bit, eagerly and under GraphedForward replay."""
import ctypes

import pytest
import torch

from pretorched_x_b200 import _lib, engine, ops
from pretorched_x_b200._lib import GemmArgs

from tests import kernel_ref as R

pytestmark = pytest.mark.gpu
KID_PGEMM = 6
KID_PGEMM_CHAIN = 11
B2_ERR_UNSUPPORTED = -3


@pytest.fixture(scope="module")
def lib():
    assert torch.cuda.is_available(), "GPU tests need an H100"
    lib = _lib.load()
    lib.b2_debug_last_kernel.restype = ctypes.c_int
    lib.b2_debug_last_kernel.argtypes = [ctypes.c_void_p]
    return lib


def last_kernel(lib):
    info = (ctypes.c_int * 5)()
    kid = lib.b2_debug_last_kernel(ctypes.cast(info, ctypes.c_void_p))
    return kid, list(info)


def case(seed, M, N, K, N1, K2=0, res=True):
    """fp16 operands on the GPU: closing GEMM A[M][K] . B[N][K]^T (+ A2 . B2^T) + residual, chained W1[N1][N]."""
    g = torch.Generator().manual_seed(seed)
    d = {"A": torch.randn(M, K, generator=g), "B": torch.randn(N, K, generator=g) / K ** 0.5,
         "sc": torch.rand(N, generator=g) + 0.5, "sh": torch.randn(N, generator=g) * 0.5,
         "W1": torch.randn(N1, N, generator=g) / N ** 0.5, "sc1": torch.rand(N1, generator=g) + 0.5,
         "sh1": torch.randn(N1, generator=g) * 0.5}
    if res:
        d["R"] = torch.randn(M, N, generator=g)
    if K2:
        d["A2"], d["B2"] = torch.randn(M, K2, generator=g), torch.randn(N, K2, generator=g) / K2 ** 0.5
    return {k: (v.half() if v.dim() == 2 else v).cuda() for k, v in d.items()}


def run_chain(c, M, N, K, N1, K2=0, out=None):
    second = (c["A2"], c["B2"], K2) if K2 else None
    return ops.gemm_chain(c["A"], c["B"], c["sc"], c["sh"], M, N, K, c["W1"], c["sc1"], c["sh1"], N1, residual=c.get("R"), relu=True,
                          second=second, out=out)


def run_separate(c, M, N, K, N1, K2=0):
    second = (c["A2"], c["B2"], K2) if K2 else None
    y = ops.gemm(c["A"], c["B"], c["sc"], c["sh"], M, N, K, residual=c.get("R"), relu=True, second=second)
    h1 = ops.gemm(y, c["W1"], c["sc1"], c["sh1"], M, N1, N, relu=True)
    return y, h1


def check_bound(c, y, h1, M, N, N1, K2=0):
    acc, mag = R.gemm_acc(c["A"], c["B"])
    if K2:
        acc2, mag2 = R.gemm_acc(c["A2"], c["B2"])
        acc, mag = acc + acc2, mag + mag2
    res = c["R"].double().cpu() if "R" in c else None
    ref, A = R.epilogue(acc, mag, c["sc"], c["sh"], residual=res, relu=True)
    assert R.worst_ratio(y[:, :N].float(), ref, A, True) <= 1.0, R.where_worst(y[:, :N].float(), ref, A, True)
    acc1, mag1 = R.gemm_acc(y[:, :N], c["W1"])
    ref1, A1 = R.epilogue(acc1, mag1, c["sc1"], c["sh1"], relu=True)
    assert R.worst_ratio(h1[:, :N1].float(), ref1, A1, True) <= 1.0, R.where_worst(h1[:, :N1].float(), ref1, A1, True)


# M (ragged: a multiple of 128 plus 40), N, K, N1, K2 (second operand pair), residual
CASES = [
    (128 * 9 + 40, 64, 64, 64, 0, True),
    (128 * 9 + 40, 128, 64, 128, 0, True),
    (128 * 9 + 40, 192, 128, 64, 0, False),
    (128 * 9 + 40, 256, 64, 64, 0, True),          # layer1.1 -> layer1.2
    (128 * 9 + 40, 256, 64, 128, 0, True),         # layer1.2 -> layer2.0
    (128 * 9 + 40, 256, 64, 64, 64, False),        # layer1.0 (projection pair) -> layer1.1
    (128 * 300 + 40, 256, 64, 64, 0, True),        # 301 tiles: ring, residual and tile parities wrap
    (128 * 300 + 40, 256, 64, 64, 64, False),
    (128 * 4 + 40, 128, 64, 40, 0, True),          # n1 = 40: a 40-wide chained output on the 64-wide instance
    (128 * 4 + 40, 64, 64, 100, 0, False),         # n1 = 100 in a 104-wide pitch: columns [100, 104) written as zero
]


@pytest.mark.parametrize("M,N,K,N1,K2,res", CASES)
def test_chain_matches_two_launches(lib, M, N, K, N1, K2, res):
    c = case(M + N + N1 + K2, M, N, K, N1, K2, res)
    y_ref, h1_ref = run_separate(c, M, N, K, N1, K2)
    assert last_kernel(lib)[0] == KID_PGEMM
    y, h1 = run_chain(c, M, N, K, N1, K2)
    kid, info = last_kernel(lib)
    assert kid == KID_PGEMM_CHAIN and info[:2] == [64 if N <= 64 else 128, 64 if ops._round_up(N1, 8) <= 64 else 128]
    torch.cuda.synchronize()
    assert torch.equal(y.view(torch.int16), y_ref.view(torch.int16))
    assert torch.equal(h1.view(torch.int16), h1_ref.view(torch.int16))
    if h1.shape[1] > N1:
        assert float(h1[:, N1:].float().abs().max()) == 0.0
    check_bound(c, y, h1, M, N, N1, K2)
    y2, h12 = run_chain(c, M, N, K, N1, K2)                          # repeat call: bitwise equal
    assert torch.equal(y2.view(torch.int16), y.view(torch.int16)) and torch.equal(h12.view(torch.int16), h1.view(torch.int16))


def test_chain_out_rows(lib):
    """y into a row range of a larger buffer: the NaN sentinel rows around it stay untouched."""
    M, N, K, N1 = 128 * 5 + 40, 256, 64, 64
    c = case(7, M, N, K, N1)
    buf = torch.full((M + 300, N), float("nan"), dtype=torch.float16, device="cuda")
    y, h1 = run_chain(c, M, N, K, N1, out=buf[100:100 + M])
    y_ref, h1_ref = run_separate(c, M, N, K, N1)
    torch.cuda.synchronize()
    assert y.data_ptr() == buf[100].data_ptr()
    assert torch.equal(buf[100:100 + M].view(torch.int16), y_ref.view(torch.int16))
    assert torch.equal(h1.view(torch.int16), h1_ref.view(torch.int16))
    assert bool(buf[:100].isnan().all()) and bool(buf[100 + M:].isnan().all())


def _args(c, M, N, K, ldd):
    g = GemmArgs()
    g.a, g.b, g.scale, g.shift = c["A"].data_ptr(), c["B"].data_ptr(), c["sc"].data_ptr(), c["sh"].data_ptr()
    g.d = torch.empty((M, ldd), dtype=torch.float16, device="cuda").data_ptr()
    g.M, g.N, g.Kd = M, N, K
    g.lda, g.ldb, g.ldd = K, K, ldd
    g.relu = 1
    return g


def test_chain_unsupported(lib):
    """Everything outside the contract returns B2_ERR_UNSUPPORTED (the caller then runs the two launches)."""
    M, K = 1000, 64
    c = case(3, M, 320, K, 200)
    h1 = torch.empty((M, 256), dtype=torch.float16, device="cuda")
    keep = []

    def call(N, ldd, ld1=64, n1=64, **fields):
        g = _args(c, M, N, K, ldd)
        for name, v in fields.items():
            if isinstance(v, torch.Tensor):
                keep.append(v)
                v = v.data_ptr()
            setattr(g, name, v)
        return lib.b2_gemm_chain_f16(ctypes.byref(g), None, 0, None, 0, 0, c["W1"].data_ptr(), 320, n1, c["sc1"].data_ptr(),
                                     c["sh1"].data_ptr(), h1.data_ptr(), ld1, None)

    aff = torch.ones((8, 256), device="cuda")
    unsupported = [
        call(256, 256, out_f32=1),
        call(256, 256, per_row=1),
        call(256, 256, aff_ld=256, aff_rows=128, scale=aff, shift=aff),
        call(256, 256, d2=torch.empty((M, 256), dtype=torch.float16, device="cuda"), scale2=aff, shift2=aff, aff2_ld=256, aff2_rows=128),
        call(256, 256, mask=torch.ones((M, 256), dtype=torch.float16, device="cuda"), ldm=256),
        call(200, 200),                               # N % 64 != 0
        call(320, 320),                               # N > 256
        call(128, 136),                               # ldd != N
        call(256, 256, ld1=136, n1=136),              # chained pitch > 128
    ]
    assert unsupported == [B2_ERR_UNSUPPORTED] * len(unsupported), unsupported
    assert last_kernel(lib)[0] == 0


# ---------------------------------------------------------------------------------------------------------------------------
# the engine's pairing on a resnet3d50 forward
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def r3d50():
    import pretorched_x_b200 as P
    from oracle import functional as OF
    torch.manual_seed(0)
    model = P.resnet3d50(num_classes=400, pretrained=None)
    OF.randomize_bn_(model, 1)
    return model.eval().cuda()


def _forward_counting(model, x, lib, monkeypatch):
    """Forward with every b2_gemm_chain_f16 call recorded by the kernel id it left behind."""
    kids = []
    real = ops.gemm_chain

    def spy(*a, **k):
        out = real(*a, **k)
        kids.append(last_kernel(lib)[0])
        return out

    monkeypatch.setattr(ops, "gemm_chain", spy)
    with torch.no_grad():
        y = model(x)
    torch.cuda.synchronize()
    monkeypatch.setattr(ops, "gemm_chain", real)
    return y, kids


def test_resnet3d50_chained_forward_is_bitwise(lib, r3d50, monkeypatch):
    x = torch.randn(2, 3, 16, 224, 224, generator=torch.Generator().manual_seed(5)).cuda()
    got, kids = _forward_counting(r3d50, x, lib, monkeypatch)
    assert kids == [KID_PGEMM_CHAIN] * 3                             # layer1.0 -> 1.1 -> 1.2 -> layer2.0
    monkeypatch.setattr(engine, "_chains", lambda *a, **k: False)
    want, kids = _forward_counting(r3d50, x, lib, monkeypatch)
    assert kids == []
    assert torch.equal(got, want)


def test_resnet3d50_chained_graph_replay(lib, r3d50, monkeypatch):
    from pretorched_x_b200.graph import GraphedForward
    x = torch.randn(2, 3, 16, 224, 224, generator=torch.Generator().manual_seed(6)).cuda()
    with torch.no_grad():
        want = r3d50(x)
        gf = GraphedForward(r3d50, x)
        got = gf(x).clone()
        got2 = gf(x).clone()
    torch.cuda.synchronize()
    assert torch.equal(got, want) and torch.equal(got2, want)
    monkeypatch.setattr(engine, "_chains", lambda *a, **k: False)
    with torch.no_grad():
        plain = r3d50(x)
    torch.cuda.synchronize()
    assert torch.equal(got, plain)
