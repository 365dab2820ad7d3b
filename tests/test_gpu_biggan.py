"""GPU (-m gpu): BigGAN-deep generator path (BASELINE.json configs[4]) against oracle/biggan.py.

PARITY UNPINNED: the reference tree holds no GAN code (SURVEY.md section 8a row a14), so the checker is our own CPU
restatement of the published architecture, not an output of the reference.

Stated tolerances (fp16 activations and weights, fp32 accumulation; relative to max|restatement| of the tensor):
  helper kernels 2e-3 (one fp16 rounding), convolutions with a per-sample epilogue 3e-3.
Whole generator: 13 un-normalised residual blocks, 52 BatchNorms that re-scale channels whose mean may dwarf their
spread, and an unscaled softmax make fp16 *storage* itself cost up to 4e-2 of a stage's range at the largest outlier
(RMS ~1e-2) on a random-init ch=128 model -- measured on the CPU with ``oracle.biggan.fp16_storage``, the restatement
run with an fp16 round trip at exactly the points where the engine stores fp16.  The product path is therefore bounded
by that expected-numerics twin, per stage: max error <= 2 x twin + 2e-3, RMS error <= 1.5 x twin + 5e-4 (both relative
to the fp32 restatement), with absolute caps of 2e-2 RMS per stage and 1e-2 RMS / 0.15 max on the images in (-1, 1).
"""
import glob
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import biggan as OB
import pretorched_x_b200 as P
from pretorched_x_b200 import biggan_engine, ops
from pretorched_x_b200.ops import Act

pytestmark = pytest.mark.gpu
FIX = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "biggan_*.pt")))


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need an H100"
    return torch.device("cuda:0")


def nhwc(x16):
    """fp16 NCHW (cpu or cuda) -> Act on cuda."""
    N, C, H, W = x16.shape
    return Act(x16.permute(0, 2, 3, 1).contiguous().view(N * H * W, C).cuda(), N, 1, H, W, C)


def to_nchw(a):
    return a.data[:, :a.C].float().view(a.N, a.H, a.W, a.C).permute(0, 3, 1, 2).cpu()


def rel(got, want):
    return (got.double() - want.double()).abs().max().item() / max(want.abs().max().item(), 1e-12)


@pytest.mark.parametrize("up", [1, 2])
@pytest.mark.parametrize("mode", ["sample", "shared", "copy"])
def test_ccbn_act(dev, up, mode):
    g = torch.Generator().manual_seed(5)
    N, C, H, W = 3, 48, 6, 10
    x = torch.randn(N, C, H, W, generator=g).half()
    a = nhwc(x)
    pitch = 104
    aff = torch.randn(N, 2 * pitch, generator=g).cuda()
    Cs = 24 if mode == "copy" else C
    if mode == "sample":
        sc, sh = aff[:, 8:8 + C], aff[:, pitch + 8:pitch + 8 + C]
        want = F.relu(x.float() * sc.cpu().view(N, C, 1, 1) + sh.cpu().view(N, C, 1, 1))
        out = ops.ccbn_act(a, sc, sh, up=up)
    elif mode == "shared":
        sc, sh = aff[:1, 8:8 + C].contiguous(), aff[:1, pitch + 8:pitch + 8 + C].contiguous()
        want = F.relu(x.float() * sc.cpu().view(1, C, 1, 1) + sh.cpu().view(1, C, 1, 1))
        out = ops.ccbn_act(a, sc, sh, up=up)
    else:
        want = x.float()[:, :Cs]
        out = ops.ccbn_act(a, None, None, channels=Cs, up=up, relu=False)
    if up == 2:
        want = F.interpolate(want, scale_factor=2)
    assert (out.H, out.W, out.C) == (H * up, W * up, Cs)
    assert rel(to_nchw(out), want) <= (0.0 if mode == "copy" else 2e-3)
    assert float(out.data[:, Cs:].abs().max()) == 0.0 if out.ld > Cs else True


def test_embed_concat_and_tanh(dev):
    g = torch.Generator().manual_seed(6)
    z = torch.randn(5, 128, generator=g)
    lab = torch.tensor([0, 9, 3, 3, 7])
    table = torch.randn(10, 128, generator=g)
    y = ops.embed_concat(z.cuda(), lab.cuda(), table.cuda())
    want = torch.cat([table[lab], z], 1)
    assert y.shape == (5, 256) and rel(y.float().cpu(), want) <= 1e-3
    y2 = ops.embed_concat(z.cuda(), table[lab].cuda(), table.cuda())
    assert torch.equal(y, y2)
    y3 = ops.embed_concat(z.cuda(), lab.cuda(), table.cuda(), split=True)
    assert y3.shape == (5, 768) and torch.equal(y3[:, :256], y) and torch.equal(y3[:, 512:], y)
    assert rel(y3[:, :256].float().cpu() + y3[:, 256:512].float().cpu(), want) <= 1e-6
    x = (torch.randn(2, 3, 9, 14, generator=g) * 3).half()
    a = nhwc(F.pad(x, (0, 0, 0, 0, 0, 5)))          # 3 channels in an 8-wide row
    a.C = 3
    for dt in (torch.float32, torch.float16):
        img = ops.tanh_to_nchw(a, dt)
        assert img.dtype == dt and img.shape == (2, 3, 9, 14)
        assert (img.float().cpu() - torch.tanh(x.float())).abs().max().item() <= (1e-5 if dt == torch.float32 else 1e-3)


@pytest.mark.parametrize("shape", [(3, 64, 12, 20, 64), (2, 128, 16, 16, 128), (5, 32, 4, 4, 32), (2, 16, 40, 40, 8),
                                   (2, 64, 20, 256, 64), (1, 128, 9, 256, 3), (2, 128, 12, 128, 128),
                                   # many small planes: items must never span two samples' affine rows
                                   (300, 64, 8, 8, 64), (320, 128, 4, 4, 256)])
def test_conv3x3_with_per_sample_affine(dev, shape):
    N, C, H, W, K = shape
    g = torch.Generator().manual_seed(7)
    x = torch.randn(N, C, H, W, generator=g).half()
    w = (torch.randn(K, C, 3, 3, generator=g) / (3 * C ** 0.5))
    Kp = (K + 7) // 8 * 8                                   # per-sample affine rows: 16-byte aligned, pitch % 4 == 0
    aff = torch.randn(N, 2 * Kp + 16, generator=g).cuda()
    sc, sh = aff[:, :K], aff[:, Kp + 16:Kp + 16 + K]
    pc = ops.PackedConv(w.cuda(), None, None, (1, 1, 1), (0, 1, 1), in_pitch=C)
    out = ops.conv(nhwc(x), pc, relu=True, sample_affine=(sc, sh))
    ref = F.conv2d(x.float(), w.half().float(), None, 1, 1)
    want = F.relu(ref * sc.cpu().view(N, K, 1, 1) + sh.cpu().view(N, K, 1, 1))
    assert rel(to_nchw(out), want) <= 3e-3


@pytest.mark.parametrize("shape", [(3, 64, 12, 20, 64), (2, 128, 16, 16, 128), (5, 512, 4, 4, 512), (2, 16, 40, 40, 8),
                                   (2, 64, 10, 128, 64), (1, 256, 32, 32, 256), (3, 32, 7, 9, 24)])
@pytest.mark.parametrize("affine", ["sample", "channel"])
def test_conv3x3_of_upsampled_image_without_materialising_it(dev, shape, affine):
    """b2_conv_args.upsample: conv3x3(nearest_up2(x)) from the low-res tensor (four folded 2x2 phase filters)."""
    N, C, H, W, K = shape
    g = torch.Generator().manual_seed(9)
    x = torch.randn(N, C, H, W, generator=g).half()
    w = torch.randn(K, C, 3, 3, generator=g) / (3 * C ** 0.5)
    b = torch.randn(K, generator=g)
    pc = ops.PackedConv(w.cuda(), b.cuda(), None, (1, 1, 1), (0, 1, 1), in_pitch=C, upsample=True)
    ref = F.conv2d(F.interpolate(x.float(), scale_factor=2), w, None, 1, 1)
    if affine == "sample":
        aff = torch.randn(N, 2 * K + 16, generator=g).cuda()
        sc, sh = aff[:, :K], aff[:, K + 16:]
        out = ops.conv(nhwc(x), pc, relu=True, sample_affine=(sc, sh))
        want = F.relu(ref * sc.cpu().view(N, K, 1, 1) + sh.cpu().view(N, K, 1, 1))
    else:
        out = ops.conv(nhwc(x), pc, relu=False)
        want = ref + b.view(1, K, 1, 1)
    assert (out.H, out.W, out.C) == (2 * H, 2 * W, K)
    assert rel(to_nchw(out), want) <= 3e-3


@pytest.mark.parametrize("shape", [(2, 64, 16, 16, 128, 200), (3, 32, 8, 8, 64, 64), (1, 128, 64, 128, 32, 96), (2, 16, 6, 10, 24, 24),
                                   (3, 64, 64, 64, 64, 72), (1, 32, 4, 256, 40, 40), (5, 16, 4, 4, 16, 16)])
@pytest.mark.parametrize("pre", [False, True])
def test_conv1x1_with_upsampled_skip(dev, shape, pre):
    """GBlock closing convolution: conv1x1(t) + upsample(x[:, :K]) with x read at low resolution by the epilogue
    (residual_up), optionally with the residual joining before the affine (residual_pre: folded output BatchNorm)."""
    N, C, H, W, K, Cx = shape                              # t: [N, C, H, W]; x: [N, Cx >= K, H/2, W/2]
    g = torch.Generator().manual_seed(10)
    t = torch.randn(N, C, H, W, generator=g).half()
    x = torch.randn(N, Cx, H // 2, W // 2, generator=g).half()
    w = torch.randn(K, C, 1, 1, generator=g) / C ** 0.5
    pc = ops.PackedConv(w.cuda(), None, None, (1, 1, 1), (0, 0, 0), in_pitch=C)
    pc.scale = (torch.rand(K, generator=g) + 0.5).cuda()
    pc.shift = torch.randn(K, generator=g).cuda()
    if W % 128 != 0 and 64 % W != 0:          # a tile's sources must be consecutive low-res rows: refused, not mis-added
        with pytest.raises(RuntimeError, match="multiple of 128 or divides 64"):
            ops.conv(nhwc(t), pc, residual=nhwc(x), relu=True, residual_up=True, residual_pre=pre)
        return
    out = ops.conv(nhwc(t), pc, residual=nhwc(x), relu=True, residual_up=True, residual_pre=pre)
    acc = F.conv2d(t.float(), w.half().float())
    skip = F.interpolate(x.float()[:, :K], scale_factor=2)
    s_, b_ = pc.scale.cpu().view(1, K, 1, 1), pc.shift.cpu().view(1, K, 1, 1)
    want = F.relu((acc + skip) * s_ + b_) if pre else F.relu(acc * s_ + b_ + skip)
    assert rel(to_nchw(out), want) <= 3e-3
    assert out.ld == (K + 7) // 8 * 8 and (out.ld == K or float(out.data[:, K:].abs().max()) == 0.0)


@pytest.mark.parametrize("shape", [(3, 256, 16, 16, 64), (2, 64, 16, 8, 200)])
def test_conv1x1_with_per_sample_affine(dev, shape):
    N, C, H, W, K = shape
    g = torch.Generator().manual_seed(8)
    x = torch.randn(N, C, H, W, generator=g).half()
    w = torch.randn(K, C, 1, 1, generator=g) / C ** 0.5
    aff = torch.randn(N, 2 * K + 8, generator=g).cuda()
    sc, sh = aff[:, :K], aff[:, K + 8:]
    pc = ops.PackedConv(w.cuda(), None, None, (1, 1, 1), (0, 0, 0), in_pitch=C)
    out = ops.conv(nhwc(x), pc, relu=True, sample_affine=(sc, sh))
    want = F.relu(F.conv2d(x.float(), w.half().float()) * sc.cpu().view(N, K, 1, 1) + sh.cpu().view(N, K, 1, 1))
    assert rel(to_nchw(out), want) <= 3e-3
    # a tile that would straddle two samples is refused, not silently mis-scaled
    x2 = torch.randn(2, C, 6, 6, generator=g).half()
    with pytest.raises(RuntimeError, match="128"):
        ops.conv(nhwc(x2), pc, relu=True, sample_affine=(sc[:2], sh[:2]))


@pytest.mark.parametrize("shape", [(2, 128, 24, 40), (1, 64, 9, 300), (3, 16, 5, 7)])
def test_split_rgb_head(dev, shape):
    """3x3 conv to RGB as a 1x1 GEMM to per-tap partial products + gather-sum + bias + tanh (b2_rgb_head_gather_tanh)."""
    N, C, H, W = shape
    g = torch.Generator().manual_seed(11)
    x = torch.randn(N, C, H, W, generator=g).half()
    w = torch.randn(3, C, 3, 3, generator=g) / (3 * C ** 0.5)
    b = torch.randn(3, generator=g)
    hw = torch.zeros(40, C, dtype=torch.float16)
    for tap in range(9):
        hw[tap * 4:tap * 4 + 3] = w[:, :, tap // 3, tap % 3].half()
    a = nhwc(x)
    part = ops.gemm(a.data, hw.cuda(), torch.ones(40).cuda(), torch.zeros(40).cuda(), a.M, 40, a.ld)
    want = torch.tanh(F.conv2d(x.float(), w.half().float(), b, 1, 1))
    for dt in (torch.float32, torch.float16):
        img = ops.rgb_head(part, b.cuda(), N, H, W, 3, dt)
        assert img.shape == (N, 3, H, W) and img.dtype == dt
        assert (img.float().cpu() - want).abs().max().item() <= 3e-3


@pytest.mark.parametrize("shape", [(2, 64, 16, 16, 128), (3, 256, 16, 8, 64), (1, 32, 32, 32, 200)])
@pytest.mark.parametrize("up", [False, True])
def test_conv1x1_with_second_output(dev, shape, up):
    """conv4 of a GBlock writing h + skip AND relu(ccbn1_next(h + skip)) (b2_conv_args.y2) from one accumulator."""
    N, C, H, W, K = shape
    g = torch.Generator().manual_seed(12)
    t = torch.randn(N, C, H, W, generator=g).half()
    x = torch.randn(N, K + 8, H // 2, W // 2, generator=g).half() if up else torch.randn(N, K, H, W, generator=g).half()
    w = torch.randn(K, C, 1, 1, generator=g) / C ** 0.5
    b = torch.randn(K, generator=g)
    aff = torch.randn(N, 2 * K + 8, generator=g).cuda()
    sc2, sh2 = aff[:, :K], aff[:, K + 8:]
    pc = ops.PackedConv(w.cuda(), b.cuda(), None, (1, 1, 1), (0, 0, 0), in_pitch=C)
    out, nxt = ops.conv(nhwc(t), pc, residual=nhwc(x), residual_up=up, next_affine=(sc2, sh2))
    skip = F.interpolate(x.float()[:, :K], scale_factor=2) if up else x.float()
    want = F.conv2d(t.float(), w.half().float(), b) + skip
    want2 = F.relu(want * sc2.cpu().view(N, K, 1, 1) + sh2.cpu().view(N, K, 1, 1))
    assert rel(to_nchw(out), want) <= 3e-3 and rel(to_nchw(nxt), want2) <= 3e-3


def rms(got, want):
    return ((got.double() - want.double()).pow(2).mean().sqrt() / want.double().pow(2).mean().sqrt().clamp_min(1e-12)).item()


def run_case(model, sd, z, labels, res, ch, dev, fuse_output_bn=True):
    want_stages, twin_stages, got_stages = {}, {}, {}
    with torch.no_grad():
        want = OB.generator_forward(z, labels, sd, res, ch, stages=want_stages)
        twin = OB.generator_forward(z, labels, sd, res, ch, stages=twin_stages, storage=OB.fp16_storage)
        got = biggan_engine.generator_forward(model.to(dev), z.to(dev), labels.to(dev), stages=got_stages,
                                              fuse_output_bn=fuse_output_bn, split_head=fuse_output_bn,
                                              dual_output=not fuse_output_bn)
    torch.cuda.synchronize()
    assert got.shape == want.shape and got.dtype == torch.float32
    report = []
    last = "stage%d" % (len(model.blocks) - 1)
    # fused tail: the raw last stage and the pre-tanh tensor never exist (output BN in conv4's epilogue, split RGB head)
    assert set(want_stages) - set(got_stages) == ({last, "pre_tanh"} if fuse_output_bn else set())
    for k in got_stages:
        g = to_nchw(got_stages[k])
        e_max, e_rms = rel(g, want_stages[k]), rms(g, want_stages[k])
        t_max, t_rms = rel(twin_stages[k], want_stages[k]), rms(twin_stages[k], want_stages[k])
        report.append("%s=%.1e/%.1e(twin %.1e/%.1e)" % (k, e_max, e_rms, t_max, t_rms))
        assert e_max <= 2.0 * t_max + 2e-3, (k, e_max, t_max)
        assert e_rms <= 1.5 * t_rms + 5e-4 and e_rms <= 2e-2, (k, e_rms, t_rms)
    i_max, i_rms = (got.cpu() - want).abs().max().item(), (got.cpu() - want).pow(2).mean().sqrt().item()
    t_max, t_rms = (twin - want).abs().max().item(), (twin - want).pow(2).mean().sqrt().item()
    print("biggan %d ch%d B%d%s max/rms:" % (res, ch, z.shape[0], "" if fuse_output_bn else " (unfused tail)"), " ".join(report),
          "image=%.1e/%.1e(twin %.1e/%.1e)" % (i_max, i_rms, t_max, t_rms))
    assert i_max <= min(2.0 * t_max + 5e-3, 0.15) and i_rms <= min(1.5 * t_rms + 5e-4, 1e-2), (i_max, i_rms, t_max, t_rms)
    return got


@pytest.mark.parametrize("path", FIX, ids=[os.path.basename(p)[:-3] for p in FIX])
def test_generator_matches_restatement_on_fixture_cases(dev, path):
    fx = torch.load(path, weights_only=False)
    model, sd, z, labels = OB.build_case(P.biggan_deep, fx["resolution"], fx["ch"], fx["n_classes"], fx["batch"],
                                         fx["seeds"]["init"], fx["seeds"]["input"], fx["init"])
    got = run_case(model, sd, z, labels, fx["resolution"], fx["ch"], dev)
    run_case(model, sd, z, labels, fx["resolution"], fx["ch"], dev, fuse_output_bn=False)
    ref = fx["image"]                                  # the committed samples of the restatement's images
    samp = got.cpu().reshape(-1)[::ref["step"]][:ref["sample"].numel()]
    assert (samp - ref["sample"]).pow(2).mean().sqrt().item() <= 1e-2


def test_full_size_biggan_deep_256(dev):
    """BASELINE configs[4] architecture (ch = 128, 1000 classes, 55.7 M parameters) at a batch the CPU checks in seconds,
    plus size-independent properties: a sample's image does not depend on its batch neighbours, fp16 output is the
    rounding of the fp32 output, images stay inside (-1, 1)."""
    model, sd, z, labels = OB.build_case(P.biggan_deep, 256, 128, 1000, 3, init="ortho")
    got = run_case(model, sd, z, labels, 256, 128, dev)
    assert float(got.abs().max()) <= 1.0
    with torch.no_grad():
        solo = model(z[1:2].to(dev), labels[1:2].to(dev))
        half = model(z.to(dev), labels.to(dev), out_dtype=torch.float16)
    # kernel selection depends on the number of output positions (a batch of one takes the small-M split-K kernel for the
    # 64x64 stages, a batch of three the slab kernel): same arithmetic, different fp32 summation order, and 13 residual
    # blocks of fp16 storage amplify the last-bit differences -- independence holds to rounding, not bit for bit
    assert (solo[0] - got[1]).abs().max().item() <= 1e-2
    assert (solo[0] - got[1]).pow(2).mean().sqrt().item() <= 1e-3
    assert (half.float() - got).abs().max().item() <= 1e-3
    # embedded class vectors in place of class indices give the same images
    with torch.no_grad():
        emb = model(z.to(dev), model.shared.weight[labels.to(dev)])
    assert torch.equal(emb, got)


@pytest.mark.parametrize("res,ch,specs", [(128, 16, ["64:2", "16:3,64:1", "8:2,32:7,128:2"]), (256, 16, ["128:2,256:1", "256:3"])])
def test_depth_first_tail_matches_whole_batch(dev, res, ch, specs):
    """The generator's high-resolution tail walked depth-first on chunks of images (biggan_engine.dfs_plan; ragged last chunk,
    whole-batch level behind a chunked one, fp32 and fp16 images) equals the whole-batch walk to rounding -- a chunk may move a
    layer across a kernel-dispatch boundary (different fp32 summation order), as for a batch of one in the full-size test."""
    from pretorched_x_b200.graph import GraphedForward
    model, sd, z, labels = OB.build_case(P.biggan_deep, res, ch, 10, 5, init="ortho")
    model = model.to(dev)
    z, labels = z.to(dev), labels.to(dev)
    try:
        biggan_engine.set_dfs("off")
        with torch.no_grad():
            want = model(z, labels)
        for spec in specs:
            biggan_engine.set_dfs(spec)
            with torch.no_grad():
                got = model(z, labels)
                half = model(z, labels, out_dtype=torch.float16)
            assert got.shape == want.shape and got.dtype == want.dtype
            assert (got - want).abs().max().item() <= 1e-2, spec
            assert (got - want).pow(2).mean().sqrt().item() <= 1e-3, spec
            assert (half.float() - got).abs().max().item() <= 1e-3, spec
        g = GraphedForward(model, (z, labels))
        with torch.no_grad():
            eager = model(z, labels)
        assert torch.equal(g((z, labels)), eager)
    finally:
        biggan_engine.set_dfs("off")
