"""GPU (-m gpu): BNInception and TRN on it.

1. b2_gemm_split_f16 for every block's 1x1 heads and pool projection (B = 2 at 224^2, and an M that does not fill a 128-row tile):
   every destination element within the kernel-matrix bound of tests/kernel_ref.py against fp64, the kernel pinned, sentinel columns
   around each slice bit-for-bit unchanged, and each destination bitwise equal to its stand-alone b2_gemm_f16 when the two use the
   same N tile.
2. b2_conv_ndhwc_fprop_slice for every 3x3 shape of the network (stride 1 and 2): the same bound, sentinel and pinning checks.
3. b2_pool_ndhwc_slice: max bit-exact against F.max_pool2d on the fp16 input, average within one fp16 rounding of the fp64 average,
   columns outside the slices untouched.
4. Each block kind (stride-1 with the average pool, 5b's max pool, stride 2) against the fp64 oracle block on the engine's fp16
   input: 5e-3 of max |ref|.
5. bninception and TRN-MSTRN against the reference's fixtures, CUDA-graph replay bit-identical to the eager forward, a trainable
   last_linear on the frozen trunk, and the refusal of a final map other than 7x7.
"""
import ctypes
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import pretorched_x_b200 as P
from pretorched_x_b200 import _lib, engine, ops
from pretorched_x_b200 import functions as Fn
from pretorched_x_b200.graph import GraphedForward
from pretorched_x_b200.models import bninception as PB
from pretorched_x_b200.ops import Act
from oracle import bninception as OB
from oracle import functional as OF
from oracle.make_golden import sample_of
from tests import kernel_ref as KR
from tests.conftest import has_h100

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_h100(), reason="needs an H100")]

dev = torch.device("cuda:0")
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
KID_PGEMM_SPLIT, KID_SLAB_SLICE, KID_POOL = 12, 13, 14      # csrc/b2_host.h
SENTINEL = -12345                                            # int16 bit pattern around every slice (an fp16 NaN is not used:
                                                             # a bit-for-bit check needs a pattern the kernels never produce)


def _load(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


def _last_kernel():
    info = (ctypes.c_int * 5)()
    kid = _lib.load().b2_debug_last_kernel(info)
    return kid, list(info)


def _sentinel(M, width):
    return torch.full((M, width), SENTINEL, dtype=torch.int16, device=dev).view(torch.float16)


def _outside_untouched(buf, c0, c1):
    b = buf.view(torch.int16)
    return bool((b[:, :c0] == SENTINEL).all()) and bool((b[:, c1:] == SENTINEL).all())


# ---------------------------------------------------------------------------------------------
# 1. split GEMM
# ---------------------------------------------------------------------------------------------
def _split_cases():
    cases = []
    for n, cin, c1, (c3r, _), (cdr, _), (_, proj) in PB.BLOCKS:
        hw = {'3': 28, '4': 14, '5': 7}[n[0]]
        heads = ([c1] if c1 is not None else []) + [c3r, cdr]
        for M in (2 * hw * hw, 100):
            cases.append(("%s_heads_M%d" % (n, M), cin, heads, M))
            if proj is not None and M != 100:
                cases.append(("%s_proj_M%d" % (n, M), cin, [proj], M))
    return cases


SPLIT_CASES = _split_cases()


@pytest.mark.parametrize("name,Kd,cols,M", SPLIT_CASES, ids=[c[0] for c in SPLIT_CASES])
def test_split_gemm(name, Kd, cols, M):
    g = torch.Generator().manual_seed(M + Kd + len(cols))
    npad, box0 = ops.split_plan(cols)
    a = (torch.rand((M, Kd), generator=g) - 0.3).to(torch.float16).to(dev)
    w = torch.zeros((npad, Kd), dtype=torch.float16)
    scale, shift = torch.zeros(npad), torch.zeros(npad)
    for d, K in enumerate(cols):
        r0 = 64 * box0[d]
        w[r0:r0 + K] = ((torch.rand((K, Kd), generator=g) - 0.5) / Kd ** 0.5).to(torch.float16)
        scale[r0:r0 + K] = torch.rand(K, generator=g) + 0.5
        shift[r0:r0 + K] = torch.rand(K, generator=g) - 0.5
    w, scale, shift = w.to(dev), scale.to(dev), shift.to(dev)
    # destination 0 sits at column 32 of a wider sentinel matrix (a block output), the others at column 8 of their own
    offs = [32] + [8] * (len(cols) - 1)
    bufs = [_sentinel(M, off + K + 24) for off, K in zip(offs, cols)]
    dests = [b[:, off:off + K] for b, off, K in zip(bufs, offs, cols)]
    ops.gemm_split(a, w, scale, shift, M, Kd, dests, relu=True)
    torch.cuda.synchronize()
    kid, info = _last_kernel()
    bn = 64 if npad <= 64 else 128
    assert kid == KID_PGEMM_SPLIT and info[:3] == [bn, len(cols), npad]
    for d, K in enumerate(cols):
        r0 = 64 * box0[d]
        acc, mag = KR.gemm_acc(a, w[r0:r0 + K])
        sc, sh = scale[r0:r0 + K].double().cpu(), shift[r0:r0 + K].double().cpu()
        ref = (acc * sc + sh).clamp_min(0.0)
        A = mag * sc.abs() + sh.abs()
        ratio = KR.worst_ratio(dests[d], ref, A, True)
        assert ratio <= 1.0, "%s dest %d: %s" % (name, d, KR.where_worst(dests[d], ref, A, True))
        assert _outside_untouched(bufs[d], offs[d], offs[d] + K), "%s dest %d wrote outside its slice" % (name, d)
        if (K <= 64) == (npad <= 64):                 # b2_gemm_f16 picks the same N tile: bit for bit
            alone = ops.gemm(a, w[r0:r0 + K], scale[r0:r0 + K].contiguous(), shift[r0:r0 + K].contiguous(), M, K, Kd, relu=True)
            assert torch.equal(alone, dests[d]), "%s dest %d differs from the stand-alone GEMM" % (name, d)


# ---------------------------------------------------------------------------------------------
# 2. slice convolution
# ---------------------------------------------------------------------------------------------
def _conv_cases():
    seen = []
    for n, cin, c1, (c3r, c3), (cdr, cd), (pk, _) in PB.BLOCKS:
        hw = {'3': 28, '4': 14, '5': 7}[n[0]]
        s = 2 if pk == 'max2' else 1
        for c in ((c3r, c3, s, hw), (cdr, cd, 1, hw), (cd, cd, s, hw)):
            if c not in seen:
                seen.append(c)
    return seen


CONV_CASES = _conv_cases()


@pytest.mark.parametrize("C,K,s,H", CONV_CASES, ids=["%d-%d_s%d_%d" % c for c in CONV_CASES])
def test_slice_conv(C, K, s, H):
    g = torch.Generator().manual_seed(C * K + s + H)
    N = 2
    conv = torch.nn.Conv2d(C, K, 3, stride=s, padding=1)
    with torch.no_grad():
        conv.weight.mul_(2.0)
    conv = conv.to(dev)
    pc = ops.PackedConv(conv.weight.detach(), conv.bias, None, (1, s, s), (0, 1, 1), in_pitch=C)
    pc.scale.copy_((torch.rand(K, generator=g) + 0.5).to(dev))
    x = torch.rand((N, 1, H, H, C), generator=g).to(torch.float16)
    a = Act(x.reshape(-1, C).to(dev), N, 1, H, H, C)
    Ho = (H - 1) // s + 1
    M = N * Ho * Ho
    off = 40
    buf = _sentinel(M, off + K + 16)
    out = ops.conv_slice(a, pc, buf[:, off:off + K])
    torch.cuda.synchronize()
    kid, _ = _last_kernel()
    assert kid == KID_SLAB_SLICE and (out.H, out.W) == (Ho, Ho)
    ref, A = KR.conv_ref(x, pc.w.view(K, 9, C), pc.scale, pc.shift, (1, 3, 3), (1, s, s), (0, 1, 1), relu=True)
    got = buf[:, off:off + K]
    assert KR.worst_ratio(got, ref, A, True) <= 1.0, KR.where_worst(got, ref, A, True)
    assert _outside_untouched(buf, off, off + K)


# ---------------------------------------------------------------------------------------------
# 3. slice pooling
# ---------------------------------------------------------------------------------------------
POOL_CASES = [
    # k, stride, padding, H, avg
    (3, 1, 1, 7, False),        # 5b's pool branch
    (3, 2, 0, 28, False),       # 3c pass-through, 28 -> 14
    (3, 2, 0, 14, False),       # 4e pass-through, 14 -> 7
    (3, 1, 1, 28, True),        # the pool branches of 3a .. 5a
    (3, 1, 1, 14, True),
    (3, 1, 1, 7, True),
]


@pytest.mark.parametrize("k,s,p,H,avg", POOL_CASES)
def test_slice_pool(k, s, p, H, avg):
    g = torch.Generator().manual_seed(H * 7 + s + int(avg))
    N, C, ldx, xoff, yoff = 2, 96, 136, 16, 24
    x = (torch.rand((N, C, H, H), generator=g) * 4 - 1).to(torch.float16)
    src = torch.full((N * H * H, ldx), 7.0, dtype=torch.float16)
    src[:, xoff:xoff + C] = x.permute(0, 2, 3, 1).reshape(-1, C)
    src = src.to(dev)
    Ho = ops.ceil_pool_dim(H, k, s, p)
    buf = _sentinel(N * Ho * Ho, yoff + C + 8)
    a = Act(src[:, xoff:xoff + C], N, 1, H, H, C)
    y = ops.pool_slice(a, k, s, p, avg, buf[:, yoff:yoff + C])
    torch.cuda.synchronize()
    assert _last_kernel() == (KID_POOL, [int(avg), 0, 0, 0, 0]) and (y.H, y.W) == (Ho, Ho)
    got = buf[:, yoff:yoff + C].float().cpu().view(N, Ho, Ho, C).permute(0, 3, 1, 2)
    if avg:
        want = F.avg_pool2d(x.double(), k, s, p, ceil_mode=True, count_include_pad=True)
        bnd = KR.U_F16 * want.abs() + 2.0 ** -20 * F.avg_pool2d(x.double().abs(), k, s, p, ceil_mode=True) + KR.FLOOR
        assert float(((got.double() - want).abs() / bnd).max()) <= 1.0
    else:
        assert torch.equal(got, F.max_pool2d(x.float(), k, s, p, ceil_mode=True))
    assert _outside_untouched(buf, yoff, yoff + C)


# ---------------------------------------------------------------------------------------------
# 4. blocks against the fp64 oracle block
# ---------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def model():
    torch.manual_seed(0)
    m = P.bninception(pretrained=None)
    OF.randomize_bn_(m, 3)
    return m.eval().to(dev)


@pytest.mark.parametrize("name", ["3a", "4d", "5b", "3c", "4e"])
def test_block_matches_oracle(model, name):
    spec = [b for b in PB.BLOCKS if b[0] == name][0]
    H = {'3': 28, '4': 14, '5': 7}[name[0]]
    H = 28 if name == "3c" else H
    cin = spec[1]
    x = torch.rand((2, cin, H, H), generator=torch.Generator().manual_seed(9)).to(torch.float16)
    a = ops.from_ncdhw(x.to(dev))
    with torch.no_grad():
        y = engine.run_inception(model, spec, a)
    assert y.ld == y.C == PB.block_out_channels(spec)
    got = ops.to_ncdhw(y).squeeze(2).double().cpu()
    sd = {k: v.detach().double().cpu() for k, v in model.state_dict().items()}
    want = OB.block(x.double(), sd, spec)
    err = (got - want).abs().max().item() / want.abs().max().item()
    assert err <= 5e-3, "%s: rel err %.3e" % (name, err)


# ---------------------------------------------------------------------------------------------
# 5. models against the reference fixtures
# ---------------------------------------------------------------------------------------------
def _stages(m, x):
    a = Fn.frozen(lambda t, o: engine._bninception_stem_body(m, t, o), ops.from_ncdhw(x))
    out = {"stem": a}
    for spec in PB.BLOCKS:
        a = engine.run_inception(m, spec, a)
        out[spec[0]] = a
    return out, m.logits(a)


def test_model_stages_match_reference_fixture():
    fx = _load("bninception_b2_224.pt")
    m = OB.build_package_model(P, fx).to(dev)
    x = OF.seeded_input(fx["input_shape"], fx["seeds"]["input"]).to(dev)
    with torch.no_grad():
        stages, logits = _stages(m, x)
        whole = m(x)
        feats = m.features(x)
    torch.cuda.synchronize()
    assert tuple(feats.shape) == (2, 1024, 7, 7) and feats.dtype == torch.float32
    for name, summ in fx["stages"].items():
        t = ops.to_ncdhw(stages[name]).squeeze(2).cpu()
        assert tuple(t.shape) == tuple(summ["shape"]), name
        s, step = sample_of(t)
        assert step == summ["step"]
        err = (s.double() - summ["sample"].double()).abs().max().item() / summ["absmax"]
        assert err <= 1e-2, "%s: rel err %.3e" % (name, err)
    want = fx["logits"].double()
    err = (logits.cpu().double() - want).abs().max().item() / want.abs().max().item()
    assert err <= 5e-3, "logits: rel err %.3e" % err
    assert torch.equal(logits.argmax(1).cpu(), want.argmax(1))
    assert torch.equal(whole, logits)
    g = GraphedForward(m, x)
    assert torch.equal(g(x).clone(), whole), "graph replay differs from the eager forward"


def test_trn_mstrn_matches_reference_fixture():
    fx = _load("trn_bninception_MSTRN.pt")
    m = OB.build_package_model(P, fx).to(dev)
    x = OF.seeded_input(fx["input_shape"], fx["seeds"]["input"]).to(dev)
    with torch.no_grad():
        np.random.seed(fx["seeds"]["tuples"])
        feats = m.features(x)
        logits = m.logits(feats)
    for got, want, tol in ((feats, fx["features"], 1e-2), (logits, fx["logits"], 5e-3)):
        want = want.double()
        err = (got.cpu().double() - want).abs().max().item() / want.abs().max().item()
        assert err <= tol, "rel err %.3e" % err
    assert int(logits.argmax()) == int(fx["logits"].argmax())
    # graph replay: the relation's tuples are drawn on the host at capture (the second draw after seeding: warm-up, capture)
    np.random.seed(fx["seeds"]["tuples"])
    with torch.no_grad():
        m(x)
        eager = m(x)
    np.random.seed(fx["seeds"]["tuples"])
    g = GraphedForward(m, x, warmup=1)
    assert torch.equal(g(x).clone(), eager), "graph replay differs from the eager forward"


def test_trainable_last_linear_on_frozen_trunk(model):
    head = torch.nn.Linear(1024, 7).to(dev)
    model.last_linear = head
    try:
        x = torch.rand((2, 3, 224, 224), generator=torch.Generator().manual_seed(4)).to(dev)
        loss = model(x).square().sum()
        loss.backward()
        assert head.weight.grad is not None and float(head.weight.grad.abs().sum()) > 0
        assert all(p.grad is None for n, p in model.named_parameters() if not n.startswith("last_linear"))
    finally:
        model.last_linear = torch.nn.Linear(1024, 1000).to(dev)


def test_final_map_other_than_7x7_is_refused(model):
    x = torch.rand((1, 3, 192, 192), device=dev)
    with torch.no_grad(), pytest.raises(ValueError, match="7x7"):
        model(x)
