"""GPU (-m gpu): the fine-tuning backward element by element against fp64 (references and bounds in tests/kernel_ref.py; the
faults they catch are shown on the CPU by tests/test_finetune_bounds_cpu.py).

* the head (functions.LinearFunction) and the TRN relation MLP: dX and dW against the true gradients of the fp32 logit
  gradient, so the fp16 cast of that gradient is part of what is held;
* the pool hand-off (FineTunePoolFunction.backward: loss_scale_ then the pool backward), from the head's own gx;
* the derived dgrad filters (engine._dgrad_1x1 / _dgrad_3x3), bit for bit;
* every stage of engine.block_backward, teacher forced: each stage's reference is built from the module's parameters, the
  forward intermediates and the engine's own output of the previous stage, recorded by wrapping the engine's calls.

Every case prints its worst err / bound (pytest -s), pins the kernel that ran and checks that a second call is bitwise equal."""
import os

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import pretorched_x_b200 as P
from pretorched_x_b200 import engine, ops
from pretorched_x_b200 import functions as Fn
from oracle import functional as OF
from tests.conftest import has_h100
from tests.kernel_ref import (FLOOR, bias_grad_bound, colsum_bound, dgamma_ref, dgrad_1x1, dgrad_3x3, grad_bound, head_ref,
                              pool_backward_ref, rows_of, wdot_ref, wgrad_bound, wgrad_ref, where_worst_of, worst_ratio_of,
                              zero_insert_ref)
from tests.test_gpu_kernel_bounds import reset_knobs
from tests.test_gpu_kernel_matrix import DENSEM, IGEMM, KIND, KNOB_ENV, PGEMM, last_kernel, report, seed_of

pytestmark = [
    pytest.mark.gpu,
    pytest.mark.skipif(not has_h100(), reason="needs an H100"),
    pytest.mark.skipif(any(os.environ.get(e) for e in KNOB_ENV),
                       reason="a dispatch override is set in the environment (%s)" % ", ".join(KNOB_ENV)),
]

dev = torch.device("cuda:0")


@pytest.fixture(autouse=True)
def lib():
    from pretorched_x_b200 import _lib
    lib = _lib.load()
    reset_knobs(lib)
    try:
        yield lib
    finally:
        reset_knobs(lib)


def check(name, got, ref, bnd):
    ref, bnd = ref.cpu(), bnd.cpu()
    r = worst_ratio_of(got, ref, bnd)
    report(name, r)
    assert r <= 1.0, "%s: err/bound %.3f at %s" % (name, r, where_worst_of(got, ref, bnd))


def bits(t):
    return t.detach().contiguous().view(torch.int16 if t.element_size() == 2 else torch.int32)


def same_bits(a, b):
    return torch.equal(bits(a), bits(b))


class Recorder:
    """Wraps functions so that every call's arguments, result and b2_debug_last_kernel are kept in call order."""

    def __init__(self, monkeypatch, lib, targets):
        self.calls = {name: [] for _, name in targets}
        for owner, name in targets:
            monkeypatch.setattr(owner, name, self._wrap(name, getattr(owner, name), lib))

    def _wrap(self, name, fn, lib):
        def call(*args, **kwargs):
            out = fn(*args, **kwargs)
            self.calls[name].append((args, kwargs, out, last_kernel(lib)))
            return out
        return call


# ---------------------------------------------------------------------------------------------
# a. head
# ---------------------------------------------------------------------------------------------
HEAD_SHAPES = [(B, C) for B in (3, 32, 256) for C in (7, 339, 400, 1000)]


def run_head(x, w, b, target, temp, mult, relu_input):
    """One forward / backward of Fn.linear under cross-entropy; returns (gx, gw, gb, the fp32 logit gradient)."""
    xd, wd, bd = (t.to(dev).requires_grad_(True) for t in (x, w, b))
    caught = {}
    logits = Fn.linear(xd, wd, bd, relu_input=relu_input)
    logits.register_hook(lambda g: caught.__setitem__("gy", g.detach().clone()))
    (F.cross_entropy(logits * temp, target.to(dev)) * mult).backward()
    torch.cuda.synchronize()
    return xd.grad, wd.grad, bd.grad, caught["gy"]


def check_head(name, gy, w, x16, gx, gw, gb, relu_mask=None):
    dx_ref, bx, dw_ref, bw = head_ref(gy.to(dev), w.to(dev), x16.to(dev), None if relu_mask is None else relu_mask.to(dev))
    check("%s dX" % name, gx, dx_ref, bx)
    check("%s dW" % name, gw, dw_ref, bw)
    if gb is not None:
        db_ref, bb = bias_grad_bound(gy)
        check("%s db" % name, gb, db_ref, bb)


@pytest.mark.parametrize("mult", [1.0, 1e-3])
@pytest.mark.parametrize("temp", [1.0, 8.0], ids=["uniform", "peaked"])
@pytest.mark.parametrize("B,C", HEAD_SHAPES)
def test_head_backward_against_fp64(lib, monkeypatch, B, C, temp, mult):
    """LinearFunction with fp32 input (the fine-tuning head on pooled features); relu_input on the 400-class cases."""
    name = "head B%d C%d t%g x%g" % (B, C, temp, mult)
    g = torch.Generator().manual_seed(seed_of(name))
    relu_input = C == 400
    Fdim = 512
    x = torch.randn(B, Fdim, generator=g)
    x = x if relu_input else x.relu()
    w = torch.randn(C, Fdim, generator=g) / Fdim ** 0.5
    b = torch.randn(C, generator=g) * 0.1
    target = torch.randint(0, C, (B,), generator=g)
    rec = Recorder(monkeypatch, lib, [(ops, "gemm")])
    gx, gw, gb, gy = run_head(x, w, b, target, temp, mult, relu_input)
    kids = [k for _, _, _, k in rec.calls["gemm"]]
    assert len(kids) == 3 and all(k[0] in (DENSEM, IGEMM) for k in kids), kids       # forward, dX, dW: fp32-output GEMMs
    name += " [%s]" % "/".join(KIND[k[0]] for k in kids[1:])
    x16 = (x.relu() if relu_input else x).half()
    check_head(name, gy, w, x16, gx, gw, gb, relu_mask=(x16 > 0) if relu_input else None)
    gx2, gw2, gb2, _ = run_head(x, w, b, target, temp, mult, relu_input)
    assert same_bits(gx, gx2) and same_bits(gw, gw2) and same_bits(gb, gb2), "two identical backward passes differ"


@pytest.mark.parametrize("N,mult", [(5, 1.0), (64, 1e-3)])
def test_relation_mlp_backward_against_fp64(lib, monkeypatch, N, mult):
    """TRN's relation MLP (ReLU, Linear, ReLU, Linear through LinearFunction): both layers held like the head, each from the
    gradient the engine handed it."""
    torch.manual_seed(0)
    r = P.Relation(4, 64, 16, bottleneck_dim=32).to(dev)
    x = OF.seeded_input((N, 4, 64), 3).to(dev).requires_grad_(True)
    layers = []
    orig = Fn.linear

    def linear(xx, w, b=None, relu_input=False):
        y = orig(xx, w, b, relu_input)
        rec = dict(x=xx, w=w, relu=relu_input)
        y.register_hook(lambda g: rec.__setitem__("gy", g.detach().clone()))
        if xx.requires_grad:
            xx.register_hook(lambda g: rec.__setitem__("gx", g.detach().clone()))
        layers.append(rec)
        return y

    monkeypatch.setattr(Fn, "linear", linear)
    (r(x).square().mean() * mult).backward()
    torch.cuda.synchronize()
    assert len(layers) == 2
    for i, (rec, lin) in enumerate(zip(layers, (r.relate[1], r.relate[3]))):
        x16 = rec["x"].detach().float().relu().half().cpu()
        check_head("relation N%d x%g layer %d" % (N, mult, i), rec["gy"].cpu(), lin.weight.detach().cpu(), x16, rec["gx"],
                   lin.weight.grad, lin.bias.grad, relu_mask=x16 > 0)


# ---------------------------------------------------------------------------------------------
# b. pool hand-off
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,S,C,classes,mult", [(2, 49, 512, 400, 1.0), (32, 7, 2048, 339, 1e-3), (3, 98, 512, 1000, 1.0)])
def test_pool_handoff_against_fp64(lib, N, S, C, classes, mult):
    """The gradient at the last fine-tuned block's output: fp16(mask * gx * 2^k / S), gx the head's own input gradient, k the
    loss scale loss_scale_ chose from it (read back from the pair: max |gx| 2^k in [2^7, 2^8))."""
    g = torch.Generator().manual_seed(N * S + C)
    y = torch.randn(N * S, C, generator=g).half()
    w = torch.randn(classes, C, generator=g) / C ** 0.5
    b = torch.randn(classes, generator=g) * 0.1
    target = torch.randint(0, classes, (N,), generator=g)

    def run():
        ls = torch.ones(2, dtype=torch.float32, device=dev)
        y2d = y.to(dev).requires_grad_(True)
        caught = {}
        pooled = Fn.FineTunePoolFunction.apply(y2d, (N, 1, S, 1, C), ls)
        pooled.register_hook(lambda gg: caught.__setitem__("gf", gg.detach().clone()))
        (F.cross_entropy(Fn.linear(pooled, w.to(dev), b.to(dev)) * 8.0, target.to(dev)) * mult).backward()
        torch.cuda.synchronize()
        return y2d.grad, caught["gf"], ls.cpu()

    gyo, gf, ls = run()
    peak = float(gf.abs().max()) * float(ls[0])
    assert 2.0 ** 7 <= peak < 2.0 ** 8 and float(ls[0]) * float(ls[1]) == 1.0, ls
    ref, bnd = pool_backward_ref(gf.cpu(), y, ls[0], S)
    check("pool hand-off N%d S%d C%d x%g (2^%d)" % (N, S, C, mult, int(torch.log2(ls[0]))), gyo, ref, bnd)
    assert torch.all(gyo.cpu()[y <= 0] == 0)
    gyo2, _, _ = run()
    assert same_bits(gyo, gyo2)


# ---------------------------------------------------------------------------------------------
# c. derived dgrad filters
# ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dims", [3, 2])
def test_derived_dgrad_filters_bit_exact(dims):
    """The BN scale, the 1x1 B operand (s W)^T and the 3x3 pack (flipped, transposed, s-folded, padding (1, 1, 1) or, 2-D,
    (0, 1, 1) at kernel (1, 3, 3)) against an independent construction: fp32 product, then one rounding to fp16."""
    torch.manual_seed(dims)
    Conv, BN = (nn.Conv3d, nn.BatchNorm3d) if dims == 3 else (nn.Conv2d, nn.BatchNorm2d)
    Cin, Cout = 40, 20
    bn = OF.randomize_bn_(BN(Cout), 5).eval().to(dev)
    with torch.no_grad():
        bn.weight[3] = 1e-3                                     # a channel with a small BN scale
    s = engine._bn_scale(bn)
    s_ref = bn.weight.detach().double() / torch.sqrt(bn.running_var.double() + bn.eps)
    assert float(((s.double() - s_ref).abs() / s_ref.abs()).max()) <= 2.0 ** -21
    sc = s.cpu()

    c1 = Conv(Cin, Cout, 1, bias=False).to(dev)
    wt = engine._dgrad_1x1(c1, s).cpu()
    want = (c1.weight.detach().cpu().reshape(Cout, Cin) * sc[:, None]).t().half()
    assert wt.shape == want.shape and same_bits(wt, want)

    c3 = Conv(Cin, Cout, 3, padding=1, bias=False).to(dev)
    pitch = 24
    pc = engine._dgrad_3x3(c3, s, pitch)
    w = c3.weight.detach().cpu() * sc.view((-1,) + (1,) * (dims + 1))
    if dims == 2:
        w = w.unsqueeze(2)
    taps = w.shape[2] * w.shape[3] * w.shape[4]
    flip = w.flip(2, 3, 4).transpose(0, 1).half()                 # [Cin][Cout][kt][kh][kw]
    pack = pc.w.view(Cin, taps, pitch).cpu()
    assert (pc.K, pc.Cin, pc.C, pc.k, pc.s) == (Cin, Cout, pitch, (3 if dims == 3 else 1, 3, 3), (1, 1, 1))
    assert pc.p == ((1, 1, 1) if dims == 3 else (0, 1, 1))
    assert same_bits(pack[..., :Cout].contiguous(), flip.permute(0, 2, 3, 4, 1).reshape(Cin, taps, Cout).contiguous())
    assert torch.all(pack[..., Cout:] == 0)


# ---------------------------------------------------------------------------------------------
# d. block backward, stage by stage
# ---------------------------------------------------------------------------------------------
BLOCK_CASES = [
    # arch, layer, index, input size, loss scale, tweak
    ("resnet3d50", "layer4", 0, (2, 14, 14), 64.0, None),       # Bottleneck, type B, stride 2
    ("resnet3d50", "layer4", 1, (1, 7, 7), 64.0, None),         # Bottleneck, identity, T = 1
    ("resnet3d50", "layer1", 0, (2, 14, 14), 64.0, None),       # Bottleneck, type B, stride 1 (two-operand GEMM)
    ("resnet3d50", "layer3", 0, (1, 13, 13), 64.0, None),       # Bottleneck, type B, stride 2, odd size, T = 1
    ("resnet3d18", "layer2", 0, (4, 15, 15), 64.0, None),       # BasicBlock, type A, stride 2, odd size
    ("resnet3d18", "layer4", 1, (2, 7, 7), 64.0, None),         # BasicBlock, identity
    ("resnet3d18B", "layer3", 0, (2, 14, 14), 64.0, None),      # BasicBlock, type B, stride 2
    ("resnet18", "layer1", 1, (15, 15), 64.0, None),            # 2-D BasicBlock, identity
    ("resnet18", "layer2", 0, (15, 13), 64.0, None),            # 2-D BasicBlock, stride-2 projection, odd sizes
    ("resnet50", "layer4", 1, (7, 7), 64.0, None),              # 2-D Bottleneck, identity
    ("resnet50", "layer1", 0, (14, 14), 64.0, None),            # 2-D Bottleneck, stride-1 projection
    ("resnet50", "layer3", 0, (13, 13), 64.0, None),            # 2-D Bottleneck, stride-2 projection, odd size
    ("resnet3d50", "layer3", 0, (1, 13, 13), 2.0 ** 20, "small_scale"),
    ("resnet3d18", "layer2", 0, (4, 15, 15), 2.0 ** -10, "big_mean"),
    ("resnet50", "layer3", 0, (13, 13), 2.0 ** -10, "big_mean"),
    ("resnet18", "layer2", 0, (15, 13), 2.0 ** 20, "small_scale"),
]


def _model(arch):
    if arch == "resnet3d18B":
        return P.resnet3d18(num_classes=10, pretrained=None, shortcut_type='B')
    return getattr(P, arch)(num_classes=10, pretrained=None)


def _tweak(block, tweak):
    """small_scale: one channel of every BN scaled by 1e-3.  big_mean: running means of 40 (>> the spread of the convolution
    outputs), with beta moved so that the forward is unchanged."""
    with torch.no_grad():
        for _, bn in engine._train_units(block):
            if tweak == "small_scale":
                bn.weight[1] = 1e-3
            elif tweak == "big_mean":
                s = bn.weight / torch.sqrt(bn.running_var + bn.eps)
                bn.running_mean += 40.0
                bn.bias += 40.0 * s


def nd(a):
    """Act -> fp64 NCDHW on the device."""
    return a.data[:, :a.C].double().reshape(a.N, a.T, a.H, a.W, a.C).permute(0, 4, 1, 2, 3)


def mat(a):
    return a.data[:, :a.C].double()


def size_of(a):
    return (a.T, a.H, a.W)


def check_grad(name, got, ref, A, R, mask=None):
    """An fp16 loss-scaled gradient Act against its reference: the bound, exact zeros where the ReLU mask is not positive and
    zero padding columns."""
    check(name, got.data[:, :got.C], ref, grad_bound(ref, A, R))
    if mask is not None:
        assert torch.all(got.data[:, :got.C][mask.data[:, :got.C] <= 0] == 0), "%s not zero where the mask is" % name
    assert torch.all(got.data[:, got.C:] == 0), "%s padding columns not zero" % name


def wgrad_splits(lib, x, Cout, k, stride, pad):
    n = lib.b2_conv_wgrad_thw_workspace_elems(x.N, x.T, x.H, x.W, x.C, Cout, k[0], k[1], k[2], stride[0], stride[1], pad[0], pad[1])
    taps = k[0] * k[1] * k[2]
    To, Ho, Wo = ((i + 2 * p - kk) // s + 1 for i, kk, s, p in zip(size_of(x), k, stride, pad))
    return max(1, n // (taps * Cout * x.C)), x.N * To * -(-Ho // 8) * -(-Wo // 8)


def check_params(name, lib, conv, bn, g, x, ls, grads):
    """dW, dgamma, dbeta of one (conv, bn) unit for the gradient g at its BN output and its input x (Acts)."""
    inv = float(ls[1])
    stride, pad = engine._conv_geometry(conv)
    k = engine._kernel_thw(conv)
    s = engine._bn_scale(bn)
    splits, nbox = wgrad_splits(lib, x, g.C, k, stride, pad)
    G, M, dw_ref, Aw = wgrad_ref(nd(x), nd(g), k, stride, pad, s, inv)
    check("%s dW (splits %d)" % (name, splits), grads[0], dw_ref.reshape(grads[0].shape),
          wgrad_bound(Aw, nbox, splits, FLOOR * inv).reshape(grads[0].shape))
    db_ref, bb = colsum_bound(mat(g), inv)
    check("%s dbeta" % name, grads[2], db_ref, bb)
    wd, wb = wdot_ref(G, M, conv.weight.detach(), inv, nbox, splits, floor=FLOOR * inv)
    dg_ref, bg = dgamma_ref(wd, wb, db_ref, bb, bn.running_mean, bn.running_var, bn.eps)
    check("%s dgamma" % name, grads[1], dg_ref, bg)


@pytest.mark.parametrize("case", BLOCK_CASES, ids=["%s_%s_%d_ls%g%s" % (c[:3] + (c[4], "_" + c[5] if c[5] else "")) for c in BLOCK_CASES])
def test_block_backward_stages_against_fp64(lib, monkeypatch, case):
    arch, layer, idx, size, ls_val, tweak = case
    two_d = arch in ("resnet18", "resnet50")
    torch.manual_seed(0)
    model = OF.randomize_bn_(_model(arch), 1).eval()
    block = getattr(model, layer)[idx]
    _tweak(block, tweak)
    engine.check_trainable_block(block)
    block = block.to(dev)
    bottleneck = hasattr(block, "conv3")
    Cin = block.conv1.weight.shape[1]
    N, (T, H, W) = (4, (1,) + size) if two_d else (2, size)
    gen = torch.Generator().manual_seed(seed_of(str(case)))
    x16 = torch.randn((N, Cin, T, H, W), generator=gen).relu().half()
    xa = ops.from_ncdhw(x16.to(dev), pitch=ops._round_up(Cin, 8))
    with torch.no_grad():
        keep = []
        y = (engine._bottleneck_body if bottleneck else engine._basic_body)(block, xa, keep=keep)
        G = torch.randn((y.N, y.C, y.T, y.H, y.W), generator=gen).to(dev) * (ops.to_ncdhw(y) > 0)
        gy = ops.from_ncdhw(G.half(), pitch=y.ld)
        ls = torch.tensor([ls_val, 1.0 / ls_val], dtype=torch.float32, device=dev)
        needs = [True] * len(engine.train_params(block))
        rec = Recorder(monkeypatch, lib, [(engine, "_gemm_dgrad"), (ops, "conv"), (ops, "zero_insert"), (ops, "conv_wgrad")])
        dx, grads = engine.block_backward(block, xa, keep, gy, ls, True, needs)
        torch.cuda.synchronize()
        monkeypatch.undo()
        dx2, grads2 = engine.block_backward(block, xa, keep, gy, ls, True, needs)
        torch.cuda.synchronize()
    assert same_bits(dx.data, dx2.data) and all(same_bits(a, b) for a, b in zip(grads, grads2)), "two identical calls differ"
    name = "%s.%s.%d ls 2^%d%s" % (arch, layer, idx, round(float(torch.log2(ls[0]))), " " + tweak if tweak else "")
    dg, cv, zi = rec.calls["_gemm_dgrad"], rec.calls["conv"], rec.calls["zero_insert"]
    assert len(rec.calls["conv_wgrad"]) == len(engine._train_units(block))

    # every zero insertion, bit for bit
    for args, kw, out, _ in zi:
        g, T_, H_, W_, st = args[:5]
        want = zero_insert_ref(nd(g), (T_, H_, W_), st, channels=kw.get("channels"))
        assert torch.equal(nd(out), want) and torch.all(out.data[:, out.C:] == 0), "zero insertion %s" % (args[1:5],)

    ds = block.downsample
    s1, s2 = engine._bn_scale(block.bn1), engine._bn_scale(block.bn2)
    if bottleneck:
        h1, h2 = keep
        s3 = engine._bn_scale(block.bn3)
        args, kw, g2, kid = dg[0]
        assert kid[0] == PGEMM and kid[1][:2] == (64, 1), kid                    # masked 1x1: persistent GEMM, masked epilogue
        check_grad("%s g2 [pgemm masked]" % name, g2, *dgrad_1x1(mat(gy), block.conv3.weight, s3, mask=mat(h2)), mask=h2)
        args, kw, g1, kid = cv[0]
        assert kid[0] == IGEMM and kid[1][1] == 1, kid                           # masked 3x3: implicit GEMM, masked epilogue
        st = engine._inplane_stride(block.conv2)
        z = nd(g2) if st == 1 else zero_insert_ref(nd(g2), size_of(h1), st)
        check_grad("%s g1 [igemm masked]" % name, g1, *dgrad_3x3(z, block.conv2.weight, s2, mask=nd(h1)), mask=h1)
        units = [(block.conv1, block.bn1, g1, xa), (block.conv2, block.bn2, g2, h1), (block.conv3, block.bn3, gy, h2)]
    else:
        (h1,) = keep
        args, kw, g1, kid = cv[0]
        assert kid[0] == IGEMM and kid[1][1] == 1, kid
        check_grad("%s g1 [igemm masked]" % name, g1, *dgrad_3x3(nd(gy), block.conv2.weight, s2, mask=nd(h1)), mask=h1)
        units = [(block.conv1, block.bn1, g1, xa), (block.conv2, block.bn2, gy, h1)]

    # shortcut gradient and dx
    proj = isinstance(ds, nn.Sequential)
    if proj:
        sd = engine._bn_scale(ds[1])
        units.append((ds[0], ds[1], gy, xa))
    st_ds = engine._inplane_stride(ds[0]) if proj else (ds.stride if ds is not None else 1)
    second = None
    if ds is None:
        res = nd(gy)
    elif not proj:                                                               # type A: zero insertion + channel padding
        res = zero_insert_ref(nd(gy), size_of(xa), ds.stride, channels=xa.C)
    elif st_ds == 1 and bottleneck:                                              # stride-1 projection: second operand pair
        res = None
        second = (mat(gy), ds[0].weight, sd)
    else:                                                                        # pg in fp16, then zero-inserted as the residual
        args, kw, pg, kid = dg[1 if bottleneck else 0]
        assert kid[0] in (PGEMM, DENSEM) and kw.get("mask") is None, kid              # unmasked 1x1 at low resolution
        check_grad("%s pg [%s]" % (name, KIND[kid[0]]), pg, *dgrad_1x1(mat(gy), ds[0].weight, sd))
        res = nd(pg) if st_ds == 1 else zero_insert_ref(nd(pg), size_of(xa), st_ds)
    if bottleneck:
        args, kw, dxo, kid = dg[-1]
        assert dxo is dx and kid[0] == PGEMM and kid[1][:2] == (64, 1), kid
        assert (kw.get("second") is not None) == (second is not None)
        ref = dgrad_1x1(mat(g1), block.conv1.weight, s1, mask=mat(xa), residual=None if res is None else rows_of(res), second=second)
        check_grad("%s dx [pgemm masked%s]" % (name, " gemm2" if second else ""), dx, *ref, mask=xa)
    else:
        args, kw, dxo, kid = cv[1]
        assert dxo is dx and kid[0] == IGEMM and kid[1][1] == 1, kid
        st = engine._inplane_stride(block.conv1)
        z = nd(g1) if st == 1 else zero_insert_ref(nd(g1), size_of(xa), st)
        check_grad("%s dx [igemm masked]" % name, dx, *dgrad_3x3(z, block.conv1.weight, s1, mask=nd(xa), residual=res), mask=xa)

    # parameter gradients of every unit, in train_params order
    order = engine._train_units(block)
    for (conv, bn, g, x) in units:
        u = next(i for i, (c, _) in enumerate(order) if c is conv)
        check_params("%s unit %d" % (name, u), lib, conv, bn, g, x, ls, grads[3 * u:3 * u + 3])
