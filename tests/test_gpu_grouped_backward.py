"""GPU (-m gpu): the backward of grouped 1x3x3 convolutions (C == K) and ResNeXt-101 fine-tuning on it.

1. b2_conv_grouped_ndhwc_dgrad (through engine._conv_dgrad_masked) against fp64 autograd of F.conv2d, masked by [x > 0], for
   cg in {4, 8, 16, 32}, stride 1 and 2, ragged H x W; the group-aware kernel pinned through the launch record.
2. b2_conv_wgrad_grouped against fp64 for the same cases and a split-K case: dw in nn.Conv2d's grouped layout, wdot, the kernel
   (KID 18) and its split count pinned, the executed-MAC ratio of the plan at most 64 / cg (position blocks aside), and the dense
   block-diagonal gradient of fp64 autograd agreeing with ours on the diagonal blocks only -- off-diagonal entries get nothing.
3. One fine-tuning step of resnext101_32x4d at k = 3 and k = 4, and of TRN-MSTRN on it, against fp64 autograd on the same
   weights within the end-to-end bound of tests/test_gpu_finetune.py; a graphed step's replays equal the eager steps bit for bit.
"""
import copy
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import pretorched_x_b200 as P
from pretorched_x_b200 import _lib, engine, ops, ops_grouped
from pretorched_x_b200.graph import GraphedFineTuneStep
from oracle import functional as OF
from oracle import resnext as OX
from tests.conftest import has_h100
from tests.test_gpu_finetune import E2E_COS_MIN, E2E_REL_MAX, _check

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not has_h100(), reason="needs an H100")]

dev = torch.device("cuda:0")
KID_GROUPCONV, KID_WGRAD_GROUPED = 10, 18

# N, H, W, C, cg, stride
CASES = [(2, 14, 14, 128, 4, 1), (2, 13, 9, 256, 8, 2), (3, 7, 7, 512, 16, 1), (2, 15, 11, 1024, 32, 2), (2, 28, 28, 256, 8, 1),
         (1, 9, 13, 64, 4, 2), (16, 14, 14, 512, 16, 1)]        # last: many position blocks, several splits


def _last_kernel():
    info = (ctypes.c_int * 5)()
    return _lib.load().b2_debug_last_kernel(info), list(info)


def _case(N, H, W, C, cg, stride, seed=0):
    g = torch.Generator().manual_seed(seed)
    G = C // cg
    conv = torch.nn.Conv2d(C, C, 3, stride, 1, groups=G, bias=False)
    with torch.no_grad():
        conv.weight.copy_(torch.randn(conv.weight.shape, generator=g) / (3 * cg ** 0.5))
    s = torch.rand(C, generator=g) + 0.5
    x = torch.randn((N, C, H, W), generator=g).half().float()
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    gy = torch.randn((N, C, Ho, Wo), generator=g).half().float()
    return conv, s, x, gy


def _act(t):
    return ops.from_ncdhw(t.to(dev), pitch=t.shape[1])


def _nchw(a):
    return ops.to_ncdhw(a).squeeze(2).float().cpu()


@pytest.mark.parametrize("case", CASES, ids=lambda c: "N%dH%dW%d_C%d_cg%d_s%d" % c)
def test_grouped_dgrad_against_fp64(case):
    N, H, W, C, cg, stride = case
    conv, s, x, gy = _case(*case)
    xd = x.double().requires_grad_(True)
    y = F.conv2d(xd, conv.weight.double() * s.double().view(-1, 1, 1, 1), None, stride, 1, 1, C // cg)
    y.backward(gy.double())
    want = xd.grad * (x > 0)
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    A = F.conv_transpose2d(gy.double().abs(), (conv.weight.double() * s.double().view(-1, 1, 1, 1)).abs(), None, stride, 1,
                           (H - (stride * Ho - 1), W - (stride * Wo - 1)) if stride > 1 else 0, C // cg)
    got = engine._conv_dgrad_masked(conv.to(dev), s.to(dev), _act(gy), _act(x))
    kid, info = _last_kernel()
    assert kid == KID_GROUPCONV and info[0] == (32 if cg == 32 else 16)
    got = _nchw(got).double()
    assert tuple(got.shape) == tuple(want.shape)
    assert bool((got[x <= 0] == 0).all())
    ratio = ((got - want).abs() / (2 ** -10 * (want.abs() + A) + 2 ** -24)).max().item()
    assert ratio <= 1.0, ratio


@pytest.mark.parametrize("case", CASES, ids=lambda c: "N%dH%dW%d_C%d_cg%d_s%d" % c)
def test_grouped_wgrad_against_fp64(case):
    N, H, W, C, cg, stride = case
    conv, s, x, gy = _case(*case)
    G = C // cg
    wd = conv.weight.detach().double().clone().requires_grad_(True)
    F.conv2d(x.double(), wd, None, stride, 1, 1, G).backward(gy.double())
    want = wd.grad * s.double().view(-1, 1, 1, 1)
    A = F.conv2d(x.double().abs(), torch.ones_like(wd), None, stride, 1, 1, G)          # magnitude scale per output
    inv = torch.tensor([0.25], device=dev)
    dw, wdot = ops_grouped.conv_wgrad_grouped(_act(gy * 4), _act(x), G, stride, weight=conv.weight.to(dev), scale=s.to(dev),
                                      inv_loss_scale=inv)
    kid, info = _last_kernel()
    exe, alg, splits = ops_grouped.wgrad_grouped_plan(N, 1, H, W, C, G, stride)
    assert kid == KID_WGRAD_GROUPED and info[0] == cg and info[1] == splits
    nbox = N * ((H - 1) // stride // 8 + 1) * ((W - 1) // stride // 8 + 1)
    assert info[2] == nbox
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    assert exe == nbox * 64 * 9 * C * 64 and alg == N * Ho * Wo * 9 * C * cg
    assert exe / alg <= 64 / cg * (nbox * 64) / (N * Ho * Wo) + 1e-12
    print("cg %d: executed / algorithmic MACs %.3f (64 / cg = %.1f), splits %d" % (cg, exe / alg, 64 / cg, splits))
    dw = dw.view(conv.weight.shape).double().cpu()
    mag = torch.einsum("nchw,nchw->c", gy.double().abs(), A).view(-1, 1, 1, 1) * s.double().view(-1, 1, 1, 1)
    ratio = ((dw - want).abs() / (2 ** -10 * (want.abs() + mag / (cg * 9)) + 2 ** -24)).max().item()
    assert ratio <= 1.0, ratio
    wdot_want = (want / s.double().view(-1, 1, 1, 1) * conv.weight.double()).sum((1, 2, 3))
    torch.testing.assert_close(wdot.double().cpu(), wdot_want, rtol=1e-2, atol=1e-3 * wdot_want.abs().max().item())
    # the dense block-diagonal equivalent: fp64 autograd gives its off-diagonal entries a gradient; ours has none
    dense = ops.dense_from_grouped(wd.detach(), G).requires_grad_(True)
    F.conv2d(x.double(), dense, None, stride, 1).backward(gy.double())
    ours = ops.dense_from_grouped(dw / s.double().view(-1, 1, 1, 1), G)
    diag = ops.dense_from_grouped(torch.ones_like(wd), G) != 0
    assert bool((ours[~diag] == 0).all()) and dense.grad[~diag].abs().max() > 0
    torch.testing.assert_close(ours[diag], dense.grad[diag], rtol=1e-2, atol=1e-2 * dense.grad.abs().max().item())


# ---------------------------------------------------------------------------------------------
# 3. fine-tuning steps against fp64 autograd, and the graphed step
# ---------------------------------------------------------------------------------------------
def _model(k):
    torch.manual_seed(0)
    return OF.randomize_bn_(P.resnext101_32x4d(num_classes=10, pretrained=None), 1).eval().fine_tune(k)


@pytest.mark.parametrize("k", [3, 4])
def test_fine_tune_step_against_fp64(k):
    model = _model(k)
    x = OF.seeded_input((2, 3, 224, 224), 5)
    target = torch.tensor([1, 7])
    sd = {n: v.detach().clone().double().to(dev) for n, v in model.state_dict().items()}
    names = [n for n, p in model.named_parameters() if p.requires_grad]
    assert names and all(n.startswith(tuple("features.%d." % (3 + i) for i in range(k, 5)) + ("last_linear.",)) for n in names)
    for n in names:
        sd[n].requires_grad_(True)
    ref_loss = F.cross_entropy(OX.forward(x.double().to(dev), sd, "resnext101_32x4d"), target.to(dev))
    ref_loss.backward()
    model = model.to(dev)
    loss = F.cross_entropy(model(x.to(dev)), target.to(dev))
    loss.backward()
    assert abs(loss.item() - ref_loss.item()) <= 5e-3 * max(1.0, abs(ref_loss.item()))
    bad = []
    for n, p in model.named_parameters():
        if n in names:
            _check("resnext101_32x4d k%d %s" % (k, n), p.grad, sd[n].grad, E2E_REL_MAX, E2E_COS_MIN, bad)
        else:
            assert p.grad is None, n
    assert not bad, bad


def test_trn_mstrn_fine_tune_step_against_fp64():
    torch.manual_seed(0)
    m = P.TRN(10, num_segments=4, arch="resnext101_32x4d", consensus="MSTRN", pretrained=None, frame_bottleneck_dim=128,
              video_feature_dim=64)
    OF.randomize_bn_(m, 1)
    m = m.eval().fine_tune(4)
    assert m.frame_feature_dim == 2048
    x = OF.seeded_input((2, 4, 3, 224, 224), 5)
    target = torch.tensor([3, 8])
    sd = {n: v.detach().clone().double().to(dev) for n, v in m.state_dict().items()}
    names = [n for n, p in m.named_parameters() if p.requires_grad]
    for n in names:
        sd[n].requires_grad_(True)
    np.random.seed(3)
    ref_loss = F.cross_entropy(OX.trn_forward(x.double().to(dev), sd, "resnext101_32x4d", 4), target.to(dev))
    ref_loss.backward()
    m = m.to(dev)
    np.random.seed(3)
    loss = F.cross_entropy(m(x.to(dev)), target.to(dev))
    loss.backward()
    assert abs(loss.item() - ref_loss.item()) <= 5e-3 * max(1.0, abs(ref_loss.item()))
    bad = []
    for n in names:
        _check("trn k4 %s" % n, dict(m.named_parameters())[n].grad, sd[n].grad, E2E_REL_MAX, E2E_COS_MIN, bad)
    assert not bad, bad


def test_graphed_fine_tune_step_replays_eager_bitwise():
    eager = _model(4).to(dev)
    graphed = copy.deepcopy(eager)
    e_opt = torch.optim.SGD([p for p in eager.parameters() if p.requires_grad], lr=1e-3, momentum=0.9)
    g_opt = torch.optim.SGD([p for p in graphed.parameters() if p.requires_grad], lr=1e-3, momentum=0.9)
    x = OF.seeded_input((4, 3, 224, 224), 6).to(dev)
    t = torch.tensor([0, 3, 5, 9], device=dev)
    step = GraphedFineTuneStep(graphed, g_opt, F.cross_entropy, x, t)
    losses = []
    for _ in range(3):
        e_opt.zero_grad(set_to_none=False)
        want = F.cross_entropy(eager(x), t)
        want.backward()
        e_opt.step()
        got = step(x, t).clone()
        assert torch.equal(got, want.detach()), (got.item(), want.item())
        losses.append(got.item())
    assert len(set(losses)) == 3, losses
    for (n, a), b in zip(eager.named_parameters(), graphed.parameters()):
        assert torch.equal(a, b), n
