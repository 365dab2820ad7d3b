"""GPU: fine-tuning the 2-D ResNets (ResNet2D.fine_tune) and TRN (TRN.fine_tune) -- the (kt, kh, kw) weight-gradient entry point,
the backward of torchvision's BasicBlock / Bottleneck, and end-to-end gradients against fp64 CPU autograd of the oracle
restatement.  Tolerances are those of tests/test_gpu_finetune.py (same fp16 storage, same loss scaling)."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import pretorched_x_b200 as P
from pretorched_x_b200 import _lib, engine, ops
from pretorched_x_b200 import functions as Fn
from oracle import functional as OF
from tests.conftest import has_h100
from tests.test_gpu_finetune import COS_MIN, E2E_COS_MIN, E2E_REL_MAX, REL_MAX, WGRAD_CASES, _check, _fro

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_h100(), reason="needs an H100")]

dev = torch.device("cuda:0")


def _act16(x):
    """fp16-rounded fp32 NCDHW tensor on the CPU and its Act on the GPU."""
    x16 = x.half().float()
    return x16, ops.from_ncdhw(x16.to(dev), pitch=ops._round_up(x.shape[1], 8))


# ---------------------------------------------------------------------------------------------
# 1. weight-gradient kernel: (kt, kh, kw) filters with separate temporal / in-plane geometry
# ---------------------------------------------------------------------------------------------
THW_CASES = [
    # N, T, H, W, Cin, Cout, (kt, kh, kw), (st, s)
    (2, 1, 14, 14, 256, 256, (1, 3, 3), (1, 1)),      # resnet50 layer3 conv2 at T = 1
    (3, 1, 13, 9, 64, 128, (1, 3, 3), (1, 2)),        # odd sizes, stride 2, Cin below the 128-wide tile
    (2, 3, 7, 7, 512, 512, (1, 3, 3), (1, 1)),        # T > 1
    (2, 5, 15, 11, 128, 64, (1, 3, 3), (2, 2)),       # T > 1, temporal stride 2, Cout below the tile
    (4, 1, 14, 14, 1024, 2048, (1, 1, 1), (1, 2)),    # resnet50 layer4 projection at T = 1
    (3, 1, 7, 7, 2048, 512, (1, 1, 1), (1, 1)),
    (2, 4, 9, 9, 64, 96, (1, 1, 1), (2, 2)),          # odd size, temporal stride 2, Cout 96
    (2, 4, 14, 14, 64, 64, (3, 3, 3), (2, 1)),        # cubic filter, temporal stride only
    (2, 3, 13, 13, 64, 128, (3, 3, 3), (1, 2)),       # cubic filter, in-plane stride only
]


@pytest.mark.parametrize("case", THW_CASES, ids=lambda c: "N%dT%dH%dW%d_%d-%d_k%s_s%s" % (c[:6] + ("".join(map(str, c[6])),
                                                                                                   "".join(map(str, c[7])))))
def test_wgrad_thw_matches_conv3d_weight(case):
    N, T, H, W, Cin, Cout, k, (st, s) = case
    pad = tuple(v // 2 for v in k)
    stride = (st, s, s)
    gen = torch.Generator().manual_seed(sum(case[:6]))
    x = torch.randn((N, Cin, T, H, W), generator=gen).relu()
    To, Ho, Wo = ((n + 2 * p - kk) // ss + 1 for n, kk, ss, p in zip((T, H, W), k, stride, pad))
    g = torch.randn((N, Cout, To, Ho, Wo), generator=gen)
    x16, xa = _act16(x)
    g16, ga = _act16(g)
    w = torch.randn((Cout, Cin) + k, generator=gen) * 0.05
    scale = torch.rand(Cout, generator=gen) + 0.5
    inv = torch.tensor([0.25])
    ref = torch.nn.grad.conv3d_weight(x16.double(), (Cout, Cin) + k, g16.double(), stride=stride, padding=pad)
    want_dw = ref * scale.double()[:, None, None, None, None] * 0.25
    want_dot = (ref * w.double()).sum((1, 2, 3, 4)) * 0.25
    args = dict(weight=w.to(dev), scale=scale.to(dev), inv_loss_scale=inv.to(dev))
    dw, dot = ops.conv_wgrad(ga, xa, k, stride, pad, **args)
    dw2, dot2 = ops.conv_wgrad(ga, xa, k, stride, pad, **args)
    torch.cuda.synchronize()
    assert tuple(dw.shape) == (Cout, Cin) + k
    assert torch.equal(dw, dw2) and torch.equal(dot, dot2), "weight gradient is not bitwise repeatable"
    _check("wgrad_thw dW %s" % (case,), dw, want_dw, 1e-3, 0.999999)
    _check("wgrad_thw <W,G> %s" % (case,), dot, want_dot, 1e-3, 0.999999)


@pytest.mark.parametrize("case", WGRAD_CASES, ids=lambda c: "N%dT%dH%dW%d_%d-%d_k%ds%d" % c)
def test_cubic_filters_through_new_entry_equal_b2_conv_wgrad(case):
    """b2_conv_wgrad(k, stride, pad) and b2_conv_wgrad_thw((k, k, k), (stride, stride), (pad, pad)) are bitwise equal."""
    N, T, H, W, Cin, Cout, k, s = case
    pad = k // 2
    gen = torch.Generator().manual_seed(hash(case) % 1000)
    _, xa = _act16(torch.randn((N, Cin, T, H, W), generator=gen).relu())
    To, Ho, Wo = ((n + 2 * pad - k) // s + 1 for n in (T, H, W))
    _, ga = _act16(torch.randn((N, Cout, To, Ho, Wo), generator=gen))
    w = (torch.randn((Cout, Cin, k, k, k), generator=gen) * 0.05).to(dev)
    scale = (torch.rand(Cout, generator=gen) + 0.5).to(dev)
    inv = torch.tensor([0.25], device=dev)
    dw_new, dot_new = ops.conv_wgrad(ga, xa, (k, k, k), (s, s, s), (pad, pad, pad), weight=w, scale=scale, inv_loss_scale=inv)
    lib = _lib.load()
    n = lib.b2_conv_wgrad_workspace_elems(xa.N, xa.T, xa.H, xa.W, Cin, Cout, k, s, pad)
    ws = torch.empty(max(int(n), 1), dtype=torch.float32, device=dev)
    dw_old = torch.empty_like(dw_new)
    dot_old = torch.empty_like(dot_new)
    p = lambda t: ctypes.c_void_p(t.data_ptr())
    _lib.check(lib.b2_conv_wgrad(p(ga.data), ga.ld, p(xa.data), xa.ld, p(w), p(scale), p(inv), p(dw_old), p(dot_old), p(ws), ws.numel(),
                                 xa.N, xa.T, xa.H, xa.W, Cin, Cout, k, s, pad, ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)),
               "b2_conv_wgrad")
    torch.cuda.synchronize()
    assert torch.equal(dw_new, dw_old) and torch.equal(dot_new, dot_old)


def test_masked_dgrad_dispatch_for_2d_filters():
    """The input gradient of a 2-D 3x3 convolution is a (1, 3, 3) convolution with padding (0, 1, 1) on the masked
    implicit-GEMM kernel; the 1x1 ones run on the persistent GEMM."""
    lib = _lib.load()
    lib.b2_debug_last_gemm_path.restype = ctypes.c_int
    lib.b2_debug_last_conv_path.restype = ctypes.c_int
    gen = torch.Generator().manual_seed(12)
    N, H, W, C = 16, 14, 14, 256
    conv = torch.nn.Conv2d(C, C, 3, padding=1, bias=False)
    with torch.no_grad():
        conv.weight.copy_(torch.randn(conv.weight.shape, generator=gen) * 0.02)
    s = torch.rand(C, generator=gen) + 0.5
    g16, ga = _act16(torch.randn((N, C, 1, H, W), generator=gen))
    m16, ma = _act16(torch.randn((N, C, 1, H, W), generator=gen))
    want = torch.nn.grad.conv2d_input((N, C, H, W), conv.weight.detach().double() * s.double()[:, None, None, None],
                                      g16[:, :, 0].double(), padding=1)
    pc = engine._dgrad_3x3(conv.to(dev), s.to(dev), ga.ld)
    y = ops.to_ncdhw(ops.conv(ga, pc, mask=ma)).cpu()
    assert lib.b2_debug_last_gemm_path() == 3 and lib.b2_debug_last_conv_path() == 0
    _check("masked 1x3x3 dgrad", y[:, :, 0], want * (m16[:, :, 0] > 0), 5e-3, 0.99999)


# ---------------------------------------------------------------------------------------------
# 2. block backward of torchvision blocks
# ---------------------------------------------------------------------------------------------
BLOCK_CASES = [
    # arch, layer, index, input (H, W)  -- kind
    ("resnet18", "layer1", 1, (15, 15)),     # BasicBlock, identity, stride 1
    ("resnet18", "layer2", 0, (15, 13)),     # BasicBlock, stride-2 projection, odd sizes
    ("resnet50", "layer4", 1, (7, 7)),       # Bottleneck, identity
    ("resnet50", "layer1", 0, (14, 14)),     # Bottleneck, stride-1 projection
    ("resnet50", "layer3", 0, (13, 13)),     # Bottleneck, stride-2 projection, odd size
]


def _masked_block_2d(x, sd, block, masks):
    """fp64 torchvision BasicBlock / Bottleneck whose ReLUs multiply by the given 0/1 masks instead of testing the sign."""
    ds = block.downsample
    stride = block.conv2.stride[0] if hasattr(block, "conv3") else block.conv1.stride[0]
    res = x if ds is None else OF._bn(OF._conv(x, sd, "b.downsample.0", stride, 0), sd, "b.downsample.1")
    if hasattr(block, "conv3"):
        out = OF._bn(OF._conv(x, sd, "b.conv1"), sd, "b.bn1") * masks[0]
        out = OF._bn(OF._conv(out, sd, "b.conv2", stride, 1), sd, "b.bn2") * masks[1]
        out = OF._bn(OF._conv(out, sd, "b.conv3"), sd, "b.bn3") + res
    else:
        out = OF._bn(OF._conv(x, sd, "b.conv1", stride, 1), sd, "b.bn1") * masks[0]
        out = OF._bn(OF._conv(out, sd, "b.conv2", 1, 1), sd, "b.bn2") + res
    return out * masks[-1]


@pytest.mark.parametrize("case", BLOCK_CASES, ids=lambda c: "%s_%s_%d" % c[:3])
def test_block_backward_2d(case):
    arch, layer, idx, (H, W) = case
    torch.manual_seed(0)
    model = OF.randomize_bn_(getattr(P, arch)(num_classes=10, pretrained=None), 1).eval()
    block = getattr(model, layer)[idx]
    engine.check_trainable_block(block)
    sd = {"b." + k: v.detach().clone().double().requires_grad_(v.is_floating_point() and not k.endswith(("running_mean", "running_var", "num_batches_tracked")))
          for k, v in block.state_dict().items()}
    Cin = block.conv1.weight.shape[1]
    gen = torch.Generator().manual_seed(3)
    x = torch.randn((4, Cin, 1, H, W), generator=gen).relu()
    x16, xa = _act16(x)
    block = block.to(dev)
    ls = torch.tensor([64.0, 1.0 / 64.0], device=dev)
    x2d = xa.data.clone().requires_grad_(True)
    y2d, geom = Fn.BlockTrainFunction.apply(x2d, (xa.N, xa.T, xa.H, xa.W, xa.C), block, ls, *engine.train_params(block))
    ya = ops.Act(y2d.detach(), *geom)
    y = ops.to_ncdhw(ya).cpu()[:, :, 0]
    G = torch.randn(y.shape, generator=gen) * (y > 0)
    gy = ops.from_ncdhw((G.unsqueeze(2) * 64.0).to(dev), pitch=ya.ld).data
    torch.autograd.backward(y2d, gy)
    with torch.no_grad():
        keep = []
        (engine._bottleneck_body if hasattr(block, "conv3") else engine._basic_body)(block, xa, keep=keep)
        masks = [(ops.to_ncdhw(h).cpu()[:, :, 0] > 0).double() for h in keep] + [(y > 0).double()]
    xr = x16[:, :, 0].double().requires_grad_(True)
    yr = _masked_block_2d(xr, sd, block, masks)
    (yr * G.double()).sum().backward()
    bad = []
    _check("%s y" % (case,), y, yr, 1e-2, 0.9999, bad)
    dx = ops.to_ncdhw(ops.Act(x2d.grad, xa.N, xa.T, xa.H, xa.W, xa.C)).cpu()[:, :, 0] / 64.0
    _check("%s dx" % (case,), dx, xr.grad * (x16[:, :, 0] > 0), REL_MAX, COS_MIN, bad)
    for name, p in block.named_parameters():
        assert p.grad.shape == p.shape, name
        _check("%s d%s" % (case, name), p.grad, sd["b." + name].grad, REL_MAX, COS_MIN, bad)
    assert not bad, bad


# ---------------------------------------------------------------------------------------------
# 3. end to end
# ---------------------------------------------------------------------------------------------
E2E_CASES = [
    ("resnet18", 112, 3),
    ("resnet18", 64, 4),
    ("resnet50", 64, 4),
    ("resnet50", 112, 3),
]


@pytest.mark.parametrize("case", E2E_CASES, ids=lambda c: "%s_%d_k%d" % c)
def test_end_to_end_gradients_2d(case):
    arch, hw, k = case
    torch.manual_seed(0)
    model = OF.randomize_bn_(getattr(P, arch)(num_classes=10, pretrained=None), 1).eval()
    model.fine_tune(k)
    x = OF.seeded_input((4, 3, hw, hw), 5)
    target = torch.tensor([1, 7, 3, 0])
    sd = {n: v.detach().clone().double() for n, v in model.state_dict().items()}
    ref_names = [n for n, p in model.named_parameters() if p.requires_grad]
    for n in ref_names:
        sd[n].requires_grad_(True)
    ref_loss_t = F.cross_entropy(OF.forward(x.double(), sd, arch), target)
    ref_loss_t.backward()
    ref_loss, ref = ref_loss_t.item(), {n: sd[n].grad for n in ref_names}
    model = model.to(dev)
    xg = x.to(dev).requires_grad_(True)
    worst, bad = {}, []
    for mult in (1.0, 1e-3):
        model.zero_grad(set_to_none=True)
        loss = F.cross_entropy(model(xg), target.to(dev)) * mult
        loss.backward()
        assert abs(loss.item() / mult - ref_loss) <= 5e-3 * max(1.0, abs(ref_loss))
        assert xg.grad is None
        for n, p in model.named_parameters():
            if n in ref:
                _check("%s x%g %s" % (arch, mult, n), p.grad / mult, ref[n], E2E_REL_MAX, E2E_COS_MIN, bad)
                worst[(n, mult)] = _fro(p.grad / mult, ref[n])
            else:
                assert p.grad is None, n
    assert not bad, bad
    worse = [(n, worst[(n, 1e-3)], worst[(n, 1.0)]) for n in ref if worst[(n, 1e-3)] > 1.05 * worst[(n, 1.0)] + 1e-3]
    assert not worse, worse


def test_features_refuses_grad_mode_in_fine_tune_mode_2d():
    model = P.resnet18(num_classes=10, pretrained=None).eval().to(dev).fine_tune(4)
    x = OF.seeded_input((2, 3, 64, 64), 1).to(dev)
    with pytest.raises(NotImplementedError, match="logits"):
        model.features(x)
    with torch.no_grad():
        assert tuple(model.features(x).shape) == (2, 512, 2, 2)


# ---------------------------------------------------------------------------------------------
# 4. TRN
# ---------------------------------------------------------------------------------------------
TRN_FIXTURES = ["trn_resnet18_TRN", "trn_resnet18_HTRN", "trn_resnet18_MSTRN"]


def _trn_from_fixture(golden_dir, name):
    fx = torch.load("%s/%s.pt" % (golden_dir, name), weights_only=False)
    torch.manual_seed(fx["seeds"]["init"])
    model = P.TRN(10, num_segments=fx["segments"], arch=fx["arch"], consensus=fx["consensus"], pretrained=None, **fx["kwargs"])
    OF.randomize_bn_(model, fx["seeds"]["bn"])
    x = OF.seeded_input(fx["input_shape"], fx["seeds"]["input"])
    return fx, model.eval(), x


@pytest.mark.parametrize("name", TRN_FIXTURES)
def test_trn_fine_tune_gradients(golden_dir, name):
    fx, model, x = _trn_from_fixture(golden_dir, name)
    model.fine_tune(4)
    target = torch.arange(x.shape[0]) % 10
    sd = {n: v.detach().clone().double() for n, v in model.state_dict().items()}
    trainable = [n for n, p in model.named_parameters() if p.requires_grad]
    for n in trainable:
        sd[n].requires_grad_(True)
    if fx["np_seed"] is not None:
        np.random.seed(fx["np_seed"])
    ref_loss = F.cross_entropy(OF.trn_forward(x.double(), sd, fx["arch"], fx["consensus"], fx["segments"]), target)
    ref_loss.backward()
    model = model.to(dev)
    if fx["np_seed"] is not None:
        np.random.seed(fx["np_seed"])                     # the same frame tuples as the reference draw
    logits = model(x.to(dev))
    _check("%s logits" % name, logits, fx["logits"], 2e-2, 0.999)
    loss = F.cross_entropy(logits, target.to(dev))
    loss.backward()
    assert abs(loss.item() - ref_loss.item()) <= 5e-3 * max(1.0, abs(ref_loss.item()))
    bad = []
    for n, p in model.named_parameters():
        if n in trainable:
            assert n.startswith(("base_model.layer4.", "temporal_relation.", "last_linear.")), n
            if n.startswith("temporal_relation.") and sd[n].grad is None:    # HTRN's unused final_linear
                assert p.grad is None, n
                continue
            _check("%s %s" % (name, n), p.grad, sd[n].grad, E2E_REL_MAX, E2E_COS_MIN, bad)
        else:
            assert p.grad is None, n
    assert any(n.startswith("base_model.layer4.") and p.grad is not None for n, p in model.named_parameters())
    assert not bad, bad


def test_trn_backbone_dropout_in_training_mode(golden_dir):
    """The backbone's Dropout head receives the fp32 pooled features: in training mode it drops and rescales them like
    torch's Dropout does in the reference."""
    _, model, x = _trn_from_fixture(golden_dir, "trn_resnet18_TRN")
    model = model.to(dev).fine_tune(4)
    frames = x.to(dev).view((-1, 3) + tuple(x.shape[-2:]))
    with torch.no_grad():
        ref = model.base_model.logits(model.base_model.features_act(frames))
    drop = model.base_model.last_linear
    drop.train()
    torch.manual_seed(0)
    out = model.base_model(frames)
    assert out.dtype == torch.float32 and out.requires_grad
    kept = out != 0
    share = kept.double().mean().item()
    assert 0.4 < share < 0.6, share
    torch.testing.assert_close(out[kept], ref[kept] / (1 - drop.p), rtol=1e-5, atol=1e-6)
    out.sum().backward()
    g = model.base_model.layer4[1].bn2.bias.grad
    assert g is not None and torch.isfinite(g).all()


# ---------------------------------------------------------------------------------------------
# 5. training
# ---------------------------------------------------------------------------------------------
def _sgd_run(model, x, target, groups, lr, momentum=0.9, steps=5):
    opt = torch.optim.SGD(groups, lr=lr, momentum=momentum)
    frozen = {n: p.detach().clone() for n, p in model.named_parameters() if not p.requires_grad}
    losses = []
    for _ in range(steps):
        opt.zero_grad(set_to_none=True)
        loss = F.cross_entropy(model(x), target)
        loss.backward()
        opt.step()
        losses.append(loss.item())
    print("losses", losses)
    assert losses[-1] < losses[0]
    for n, p in model.named_parameters():
        if n in frozen:
            assert torch.equal(p.detach(), frozen[n]), n


def test_sgd_steps_2d():
    torch.manual_seed(0)
    model = OF.randomize_bn_(P.resnet50(num_classes=10, pretrained=None), 1).eval().to(dev)
    groups = P.models.resnet3d.get_fine_tuning_parameters(model, 3)
    x = OF.seeded_input((8, 3, 96, 96), 9).to(dev)
    # random init: the loss starts near 220 and the gradients are large; plain SGD at this step size lowers the fp32 CPU
    # reference's loss at every step (momentum 0.9 overshoots from the second step on)
    _sgd_run(model, x, torch.tensor([0, 3, 5, 9, 1, 2, 4, 8], device=dev), groups, 3e-7, momentum=0.0)


def test_sgd_steps_trn(golden_dir):
    _, model, x = _trn_from_fixture(golden_dir, "trn_resnet18_TRN")
    model = model.to(dev).fine_tune(3)
    _sgd_run(model, x.to(dev), torch.tensor([1, 4], device=dev), [p for p in model.parameters() if p.requires_grad], 1e-3)


def test_models_without_fine_tune_get_no_trunk_gradients(golden_dir):
    model = P.resnet50(num_classes=10, pretrained=None).eval().to(dev)
    x = OF.seeded_input((2, 3, 64, 64), 2).to(dev)
    F.cross_entropy(model(x), torch.tensor([1, 2], device=dev)).backward()
    assert all(p.grad is None for n, p in model.named_parameters() if not n.startswith("last_linear"))
    assert model.last_linear.weight.grad is not None
    _, trn, x = _trn_from_fixture(golden_dir, "trn_resnet18_TRN")
    trn = trn.to(dev)
    F.cross_entropy(trn(x.to(dev)), torch.tensor([1, 2], device=dev)).backward()
    assert all(p.grad is None for p in trn.base_model.parameters())
    assert trn.last_linear.weight.grad is not None and trn.temporal_relation.relate[1].weight.grad is not None
