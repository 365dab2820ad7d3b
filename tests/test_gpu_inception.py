"""GPU (-m gpu): Inception-v4, Inception-ResNet-v2 and TRN on them.

1. b2_conv_ndhwc_fprop_slice for every valid-padded convolution of both networks and every 1xn / nx1 / 5x5 one: every element
   within the kernel-matrix bound of tests/kernel_ref.py against fp64, the kernel pinned, sentinel columns around the slice
   bit-for-bit unchanged, a second call bitwise equal; each valid-padded shape also through the gather kernel (forced with
   b2_debug_set_conv_algo(1)) within the same bound.
2. The plain entry b2_conv_ndhwc_fprop on every valid-padded shape, unforced, at a batch above the small-M rule: the kernel the
   host plan views name is the one that ran (the slab kernel, its 128-wide transposed form, or the gather kernel where no slab
   tiling fits), within the fp64 bound.
   Where the transposed form's geometry applies it is also forced (b2_debug_set_slab_t128(1)): pinned, within the bound, and
   bitwise equal to the slab kernel with the form off.
3. b2_avgpool_ndhwc_slice_exclude_pad within one fp16 rounding of the fp64 F.avg_pool2d(count_include_pad=False), corners and
   edges included, columns outside the slices untouched.
4. Each block kind against the fp64 oracle block on the engine's fp16 input: 5e-3 of max |ref|.
5. Both networks and TRN-MSTRN on each against the reference's fixtures, CUDA-graph replay bit-identical to the eager forward, a
   trainable last_linear on the frozen trunk, and the refusal of a final map other than 8x8.
"""
import ctypes
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import pretorched_x_b200 as P
from pretorched_x_b200 import _lib, engine, ops
from pretorched_x_b200.graph import GraphedForward
from pretorched_x_b200.ops import Act
from oracle import functional as OF
from oracle import inception as OI
from oracle.inception import ONE_BY_N, VALID
from oracle.make_golden import sample_of
from tests import kernel_ref as KR
from tests.conftest import has_h100

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_h100(), reason="needs an H100")]

dev = torch.device("cuda:0")
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
KID_SLAB, KID_IGEMM, KID_SLAB_SLICE, KID_POOL, KID_SLAB_T128 = 2, 7, 13, 14, 15   # csrc/b2_host.h
SENTINEL = -12345


def _load(name):
    return torch.load(os.path.join(GOLDEN, name), weights_only=False)


def _last_kernel():
    info = (ctypes.c_int * 5)()
    return _lib.load().b2_debug_last_kernel(info), list(info)


def _sentinel(M, width):
    return torch.full((M, width), SENTINEL, dtype=torch.int16, device=dev).view(torch.float16)


def _outside_untouched(buf, c0, c1):
    b = buf.view(torch.int16)
    return bool((b[:, :c0] == SENTINEL).all()) and bool((b[:, c1:] == SENTINEL).all())


# ---------------------------------------------------------------------------------------------
# 1. slice convolution
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("C,H,K,kh,kw,s,ph,pw", VALID + ONE_BY_N, ids=lambda *a: None)
def test_slice_conv(C, H, K, kh, kw, s, ph, pw):
    g = torch.Generator().manual_seed(C * K + kh * 7 + kw + s + H)
    N = 2
    conv = torch.nn.Conv2d(C, K, (kh, kw), stride=s, padding=(ph, pw))
    with torch.no_grad():
        conv.weight.mul_(2.0)
    conv = conv.to(dev)
    pc = ops.PackedConv(conv.weight.detach(), conv.bias, None, (1, s, s), (0, ph, pw), in_pitch=C)
    pc.scale.copy_((torch.rand(K, generator=g) + 0.5).to(dev))
    x = torch.rand((N, 1, H, H, C), generator=g).to(torch.float16)
    a = Act(x.reshape(-1, C).to(dev), N, 1, H, H, C)
    Ho, Wo = (H + 2 * ph - kh) // s + 1, (H + 2 * pw - kw) // s + 1
    M = N * Ho * Wo
    off = 40
    buf = _sentinel(M, off + K + 16)
    out = ops.conv_slice(a, pc, buf[:, off:off + K])
    torch.cuda.synchronize()
    kid, _ = _last_kernel()
    assert kid == KID_SLAB_SLICE and (out.H, out.W) == (Ho, Wo)
    ref, A = KR.conv_ref(x, pc.w.view(K, kh * kw, C), pc.scale, pc.shift, (1, kh, kw), (1, s, s), (0, ph, pw), relu=True)
    got = buf[:, off:off + K].clone()
    assert KR.worst_ratio(got, ref, A, True) <= 1.0, KR.where_worst(got, ref, A, True)
    assert _outside_untouched(buf, off, off + K)
    ops.conv_slice(a, pc, buf[:, off:off + K])
    torch.cuda.synchronize()
    assert torch.equal(buf[:, off:off + K], got), "second call differs"
    if (ph, pw) == (0, 0):
        lib = _lib.load()
        try:
            lib.b2_debug_set_conv_algo(1)
            gather = ops.conv(a, pc, relu=True)
        finally:
            lib.b2_debug_set_conv_algo(0)
        torch.cuda.synchronize()
        assert KR.worst_ratio(gather.data[:, :K], ref, A, True) <= 1.0


# ---------------------------------------------------------------------------------------------
# 2. the plain entry on valid-padded shapes
# ---------------------------------------------------------------------------------------------
def _host_plans(lib, a):
    slab, t128 = (ctypes.c_int * 10)(), (ctypes.c_int * 10)()
    for fn in (lib.b2_debug_slab_plan, lib.b2_debug_slab_t128_plan):
        fn.argtypes = [ctypes.POINTER(_lib.ConvArgs), ctypes.POINTER(ctypes.c_int)]
    assert lib.b2_debug_slab_plan(ctypes.byref(a), slab) == 0 and lib.b2_debug_slab_t128_plan(ctypes.byref(a), t128) == 0
    return list(slab), list(t128)


def _plain_batch(H, kh, s, ph):
    """The smallest batch (>= 2) above the small-M rule (b2_conv_api.cu densem_wanted: at most 8192 output rows strided, 1024
    otherwise, go to the dense-M gather kernel before any slab plan), so the slab planner decides."""
    Ho = (H + 2 * ph - kh) // s + 1
    return max(2, (8192 if s > 1 else 1024) // (Ho * Ho) + 1)


# VALID just above the small-M rule, and at B = 128 a valid 3x3 the transposed form's rule takes unforced
PLAIN_CASES = [(_plain_batch(c[1], c[3], c[5], c[6]),) + c for c in VALID] + [(128, 64, 29, 128, 3, 3, 1, 0, 0),
                                                                          (128, 64, 73, 96, 3, 3, 1, 0, 0)]


@pytest.mark.parametrize("N,C,H,K,kh,kw,s,ph,pw", PLAIN_CASES, ids=lambda *a: None)
def test_plain_conv_valid(N, C, H, K, kh, kw, s, ph, pw):
    lib = _lib.load()
    lib.b2_debug_set_slab_t128.argtypes = [ctypes.c_int]
    g = torch.Generator().manual_seed(C * K + s + H + N)
    conv = torch.nn.Conv2d(C, K, (kh, kw), stride=s, padding=(ph, pw))
    pc = ops.PackedConv(conv.weight.detach().to(dev), None, None, (1, s, s), (0, ph, pw), in_pitch=C)
    pc.scale.copy_((torch.rand(K, generator=g) + 0.5).to(dev))
    pc.shift.copy_((torch.rand(K, generator=g) - 0.5).to(dev))
    x = torch.rand((N, 1, H, H, C), generator=g).to(torch.float16)
    a = Act(x.reshape(-1, C).to(dev), N, 1, H, H, C)
    args = _lib.ConvArgs()
    args.N, args.T, args.H, args.W, args.C, args.K, args.ldy = N, 1, H, H, C, K, K
    args.kt, args.kh, args.kw, args.st, args.sh, args.sw, args.pt, args.ph, args.pw = 1, kh, kw, 1, s, s, 0, ph, pw
    slab, t128 = _host_plans(lib, args)
    want = KID_SLAB_T128 if t128[0] else KID_SLAB if slab[0] else KID_IGEMM      # no slab tiling: the gather kernel
    ref, A = KR.conv_ref(x, pc.w.view(K, kh * kw, C), pc.scale, pc.shift, (1, kh, kw), (1, s, s), (0, ph, pw), relu=True)
    y = ops.conv(a, pc, relu=True)
    torch.cuda.synchronize()
    kid, info = _last_kernel()
    assert kid == want, (kid, info, slab, t128)
    if kid == KID_SLAB:
        assert info[:4] == [slab[1], slab[2], slab[8], slab[6]]
    assert KR.worst_ratio(y.data[:, :K], ref, A, True) <= 1.0, KR.where_worst(y.data[:, :K], ref, A, True)
    if t128[1]:
        try:
            lib.b2_debug_set_slab_t128(0)
            off = ops.conv(a, pc, relu=True).data.clone()
            torch.cuda.synchronize()
            assert _last_kernel()[0] == KID_SLAB
            lib.b2_debug_set_slab_t128(1)
            on = ops.conv(a, pc, relu=True).data
            torch.cuda.synchronize()
            assert _last_kernel()[0] == KID_SLAB_T128
        finally:
            lib.b2_debug_set_slab_t128(-1)
        assert KR.worst_ratio(on[:, :K], ref, A, True) <= 1.0, KR.where_worst(on[:, :K], ref, A, True)
        assert torch.equal(on, off), "the transposed form differs from the slab kernel"


# ---------------------------------------------------------------------------------------------
# 3. exclude-pad average pool
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("H", [35, 17, 8, 3])
def test_avgpool_exclude_pad(H):
    g = torch.Generator().manual_seed(H)
    N, C, ldx, xoff, yoff = 2, 96, 136, 16, 24
    x = (torch.rand((N, C, H, H), generator=g) * 4 - 1).to(torch.float16)
    src = torch.full((N * H * H, ldx), 7.0, dtype=torch.float16)
    src[:, xoff:xoff + C] = x.permute(0, 2, 3, 1).reshape(-1, C)
    src = src.to(dev)
    buf = _sentinel(N * H * H, yoff + C + 8)
    y = ops.pool_slice(Act(src[:, xoff:xoff + C], N, 1, H, H, C), 3, 1, 1, True, buf[:, yoff:yoff + C], count_include_pad=False)
    torch.cuda.synchronize()
    assert _last_kernel() == (KID_POOL, [2, 0, 0, 0, 0]) and (y.H, y.W) == (H, H)
    got = buf[:, yoff:yoff + C].float().cpu().view(N, H, H, C).permute(0, 3, 1, 2)
    want = F.avg_pool2d(x.double(), 3, 1, 1, count_include_pad=False)
    bnd = KR.U_F16 * want.abs() + 2.0 ** -20 * F.avg_pool2d(x.double().abs(), 3, 1, 1, count_include_pad=False) + KR.FLOOR
    assert float(((got.double() - want).abs() / bnd).max()) <= 1.0
    assert _outside_untouched(buf, yoff, yoff + C)


# ---------------------------------------------------------------------------------------------
# 4. blocks against the fp64 oracle block
# ---------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def models():
    out = {}
    for i, arch in enumerate(("inceptionv4", "inceptionresnetv2")):
        torch.manual_seed(i)
        m = P.__dict__[arch](pretrained=None)
        OF.randomize_bn_(m, 3)
        out[arch] = m.eval().to(dev)
    return out


BLOCKS = [("inceptionv4", "features.3", 147), ("inceptionv4", "features.4", 73), ("inceptionv4", "features.5", 71),
          ("inceptionv4", "features.6", 35), ("inceptionv4", "features.10", 35), ("inceptionv4", "features.11", 17),
          ("inceptionv4", "features.18", 17), ("inceptionv4", "features.19", 8),
          ("inceptionresnetv2", "mixed_5b", 35), ("inceptionresnetv2", "repeat.0", 35), ("inceptionresnetv2", "mixed_6a", 35),
          ("inceptionresnetv2", "repeat_1.0", 17), ("inceptionresnetv2", "mixed_7a", 17), ("inceptionresnetv2", "repeat_2.0", 8),
          ("inceptionresnetv2", "block8", 8)]


@pytest.mark.parametrize("arch,name,H", BLOCKS, ids=["%s-%s" % b[:2] for b in BLOCKS])
def test_frozen_block_matches_oracle(models, arch, name, H):
    m = models[arch]
    blk = m.get_submodule(name)
    cin = [mod for mod in blk.modules() if isinstance(mod, torch.nn.Conv2d)][0].in_channels
    x = torch.rand((2, cin, H, H), generator=torch.Generator().manual_seed(9)).to(torch.float16)
    with torch.no_grad():
        y = engine.Fn.frozen(lambda t, o: engine._inception_block_body(blk, t, o), ops.from_ncdhw(x.to(dev)))
    got = ops.to_ncdhw(y).squeeze(2).double().cpu()
    sd = {k: v.detach().double().cpu() for k, v in m.state_dict().items()}
    want = OI.block(x.double(), sd, blk, name + ".")
    assert got.shape == want.shape
    err = (got - want).abs().max().item() / want.abs().max().item()
    assert err <= 5e-3, "%s: rel err %.3e" % (name, err)


# ---------------------------------------------------------------------------------------------
# 5. models against the reference fixtures
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("arch", ["inceptionv4", "inceptionresnetv2"])
def test_model_matches_reference_fixture(arch):
    fx = _load("%s_b2_299.pt" % arch)
    m = OI.build_package_model(P, fx).to(dev)
    x = OF.seeded_input(fx["input_shape"], fx["seeds"]["input"]).to(dev)
    with torch.no_grad():
        feats = m.features(x)
        logits = m.logits(feats)
        whole = m(x)
    torch.cuda.synchronize()
    assert tuple(feats.shape) == (2, 1536, 8, 8) and feats.dtype == torch.float32
    s, step = sample_of(feats.cpu())
    assert step == fx["features"]["step"]
    err = (s.double() - fx["features"]["sample"].double()).abs().max().item() / fx["features"]["absmax"]
    assert err <= 1e-2, "features: rel err %.3e" % err
    want = fx["logits"].double()
    err = (logits.cpu().double() - want).abs().max().item() / want.abs().max().item()
    assert err <= 5e-3, "logits: rel err %.3e" % err
    assert torch.equal(logits.argmax(1).cpu(), want.argmax(1))
    assert torch.equal(whole, logits)
    g = GraphedForward(m, x)
    assert torch.equal(g(x).clone(), whole), "graph replay differs from the eager forward"


@pytest.mark.parametrize("arch", ["inceptionv4", "inceptionresnetv2"])
def test_trn_mstrn_matches_reference_fixture(arch):
    fx = _load("trn_%s_MSTRN.pt" % arch)
    m = OI.build_package_model(P, fx).to(dev)
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
    np.random.seed(fx["seeds"]["tuples"])
    with torch.no_grad():
        m(x)
        eager = m(x)
    np.random.seed(fx["seeds"]["tuples"])
    g = GraphedForward(m, x, warmup=1)
    assert torch.equal(g(x).clone(), eager), "graph replay differs from the eager forward"


@pytest.mark.parametrize("arch", ["inceptionv4", "inceptionresnetv2"])
def test_trainable_last_linear_on_frozen_trunk(models, arch):
    model = models[arch]
    head = torch.nn.Linear(1536, 7).to(dev)
    old = model.last_linear
    model.last_linear = head
    try:
        x = torch.rand((2, 3, 299, 299), generator=torch.Generator().manual_seed(4)).to(dev)
        model(x).square().sum().backward()
        assert head.weight.grad is not None and float(head.weight.grad.abs().sum()) > 0
        assert all(p.grad is None for n, p in model.named_parameters() if not n.startswith("last_linear"))
    finally:
        model.last_linear = old


@pytest.mark.parametrize("arch", ["inceptionv4", "inceptionresnetv2"])
def test_final_map_other_than_8x8_is_refused(models, arch):
    x = torch.rand((1, 3, 320, 320), device=dev)
    with torch.no_grad(), pytest.raises(ValueError, match="8x8"):
        models[arch](x)
