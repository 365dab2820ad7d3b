"""Forward engine: walks a (reference-layout) module tree and replaces the bodies of its hot blocks by
fused sm_90a kernels.

The nn.Modules in ``models/`` are *parameter containers* that keep the reference's ``state_dict``
layout; nothing in them computes.  This file holds the block bodies:

* ``conv_bn_act``        Conv3d/Conv2d/SpatioTemporalConv + BatchNorm (+residual) (+ReLU) -> one or two
                         implicit-GEMM launches                      (resnet3D.py:91-106, 125-143)
* ``run_basic/run_bottleneck``  residual blocks incl. type-A/B shortcuts (resnet3D.py:65-74, 176-185)
* ``run_nonlocal``       fused theta|phi|g projection, fused attention, W+BN+residual (nonlocalnet.py:143-166)
* ``run_stem`` / ``run_head``   stem conv+BN+ReLU+maxpool, global average + last_linear
                         (torchvision_models.py:448-464)

Packed fp16 filters and folded BN affines are cached on the owning module.  The cache key is
``(data_ptr, _version, shape)`` of every source tensor, so ``load_state_dict`` and in-place edits of the
parameter itself (``p.copy_()``, ``p.mul_()`` under ``no_grad``) rebuild the packed copy.  Edits made through
``p.data`` (the reference's own init style, ``m.weight.data.fill_``) bump a *different* version counter and are
NOT seen: ``model.invalidate()`` / ``engine.invalidate(model)`` drops every packed copy, and it runs by itself on
``train()`` / ``eval()`` and on ``.to()`` / ``.half()`` / ``.cuda()`` (``_apply``).

Every block body is entered through one ``torch.autograd.Function`` (``functions.frozen``, SURVEY.md section 8b-ii): the
body arrives as a callable, the Function's ``forward`` is its ctypes call sequence, and its outputs are marked
non-differentiable (frozen-backbone semantics), except for the stages a ``fine_tune(k)`` call (``ResNet3D``, ``ResNet2D``,
``TRN``) made trainable (``block_backward``), and the dense heads (``last_linear``, the TRN relation MLPs) have a real
backward on the same wgmma GEMM so that a head can be trained on engine features.
"""
import collections
import copy
import os

import torch
import torch.nn as nn

from . import ops
from . import ops_dual
from . import ops_vgg
from . import ops_grouped
from . import ops_xception
from . import ops_pnasnet
from . import functions as Fn
from .ops import Act


# ---------------------------------------------------------------------------------------------
# packed-parameter cache
# ---------------------------------------------------------------------------------------------
def _sig(*tensors):
    return tuple((t.data_ptr(), t._version, tuple(t.shape)) if t is not None else None for t in tensors)


def _bn_tensors(bn):
    if bn is None:
        return ()
    return (bn.weight, bn.bias, bn.running_mean, bn.running_var)


def _reads_trainable(owner, reads):
    """True when a pack built on ``owner`` reads a tensor with ``requires_grad``: a parameter of the owner (itself or its
    children) or one of ``reads`` (e.g. the BatchNorm a convolution's pack folds)."""
    return (any(t is not None and t.requires_grad for t in reads)
            or (isinstance(owner, nn.Module) and any(p.requires_grad for p in owner.parameters())))


# A CUDA-graph replay of an optimizer step (graph.GraphedFineTuneStep) changes the trainable parameters on the device
# without advancing their host-side ``_version``, so the cache key alone cannot see it.  Two rules cover it:
# * while a step is captured (``repack_trainable``), every pack that reads a trainable tensor is rebuilt on each call -- the
#   build becomes part of the graph and reads the live parameters at every replay -- and is not stored (it lives in the
#   graph's memory pool);
# * a pack that reads a trainable tensor is stored with the current parameter epoch and only reused within it;
#   ``parameters_changed()`` (called after every replay) starts a new epoch.
# Packs of frozen tensors ignore both: they are built once and kept.
_REPACK_TRAINABLE = False
_EPOCH = 0


class repack_trainable:
    """``with engine.repack_trainable(): ...`` -- packs that read a trainable tensor bypass the packed-parameter cache."""

    def __enter__(self):
        global _REPACK_TRAINABLE
        self.prev, _REPACK_TRAINABLE = _REPACK_TRAINABLE, True
        return self

    def __exit__(self, *exc):
        global _REPACK_TRAINABLE
        _REPACK_TRAINABLE = self.prev
        return False


def repacking_trainable():
    return _REPACK_TRAINABLE


def parameters_changed():
    """Trainable parameters changed without a host-side version bump: every cached pack that reads a trainable tensor is
    rebuilt at its next use; packs of frozen tensors stay."""
    global _EPOCH
    _EPOCH += 1


def _cached(owner, slot, sig, build, reads=()):
    """Cached ``build()`` on ``owner`` under key ``sig``.  ``reads``: tensors the pack folds that are not parameters of
    ``owner`` (they decide, with the owner's own parameters, whether the pack follows trainable tensors)."""
    if _REPACK_TRAINABLE and _reads_trainable(owner, reads):
        return build()
    cache = owner.__dict__.setdefault("_b2_cache", {})
    hit = cache.get(slot)
    if hit is not None and hit[0] == sig and hit[2] in (None, _EPOCH):
        return hit[1]
    val = build()
    cache[slot] = (sig, val, _EPOCH if _reads_trainable(owner, reads) else None)
    return val


def invalidate(root):
    """Drop every packed filter / folded affine cached under ``root`` (call after editing parameters through ``.data``)."""
    for m in root.modules():
        m.__dict__.pop("_b2_cache", None)
        m.__dict__.pop("_b2_pack", None)
    return root


class CacheOwner:
    """Mixin for engine-backed nn.Modules: packed copies are dropped whenever the module is moved, cast or switched
    between train / eval, and on request (``invalidate()``)."""

    def invalidate(self):
        return invalidate(self)

    def train(self, mode=True):
        invalidate(self)
        return super().train(mode)

    def _apply(self, fn, *args, **kwargs):
        invalidate(self)
        return super()._apply(fn, *args, **kwargs)


def _triple(v):
    if isinstance(v, (tuple, list)):
        v = tuple(int(i) for i in v)
        return (1,) + v if len(v) == 2 else v
    return (int(v),) * 3


def _conv_geometry(conv):
    if isinstance(conv, nn.Conv2d):
        s, p = conv.stride, conv.padding
        return (1, int(s[0]), int(s[1])), (0, int(p[0]), int(p[1]))
    return _triple(conv.stride), _triple(conv.padding)


def grouped_route(conv, stride=None):
    """True when ``packed_conv`` packs ``conv`` for the group-aware kernel (ops.PackedGroupedConv), from its shape alone."""
    cstride, padding = _conv_geometry(conv)
    w = conv.weight
    kernel = (1,) + tuple(w.shape[2:]) if w.dim() == 4 else tuple(w.shape[2:])
    return ops.grouped_pack_applies(w.shape[0], w.shape[1] * conv.groups, conv.groups, kernel, stride or cstride, padding)


def packed_conv(conv, bn, in_pitch, stem=False, stride=None, dense=False):
    """PackedConv for a plain nn.Conv3d / nn.Conv2d followed (optionally) by BatchNorm ``bn``; ops.PackedGroupedConv for a
    grouped convolution inside the group-aware kernel's contract (``grouped_route``) unless ``dense`` asks for the dense
    layout (the CUDA-core cross-check reads no other)."""
    if any(d != 1 for d in conv.dilation):
        raise NotImplementedError("dilated convolutions are outside the engine's scope")
    if conv.groups != 1 and stem:
        raise NotImplementedError("grouped stem convolutions are outside the engine's scope")
    sig = _sig(conv.weight, conv.bias, *_bn_tensors(bn)) + (in_pitch, stem, id(bn), stride)
    cstride, padding = _conv_geometry(conv)
    if stride is None:
        stride = cstride
    if not stem and not dense and grouped_route(conv, stride):
        # conv2 of ResNeXtBottleneck (resnext3D.py:86-93) and its 2-D counterpart: in_pitch is the channel count (C % 64 == 0)
        return _cached(conv, "pc", sig,
                       lambda: ops.PackedGroupedConv(conv.weight.detach(), conv.groups, conv.bias, bn, stride, padding),
                       reads=_bn_tensors(bn))
    # any other grouped convolution: the block-diagonal dense filter, see ops.dense_from_grouped
    return _cached(conv, "pc_dense" if dense else "pc", sig,
                   lambda: ops.PackedConv(ops.dense_from_grouped(conv.weight.detach(), conv.groups), conv.bias, bn, stride, padding,
                                          in_pitch=in_pitch, stem=stem), reads=_bn_tensors(bn))


def _is_stem_shape(conv):
    w = conv.weight
    kw = w.shape[-1]
    stride, padding = _conv_geometry(conv)
    return w.shape[1] <= 4 and kw == 7 and stride[2] == 2 and padding[2] == 3


def _st_conv_body(conv, bn, a, residual, relu, simt, out=None):
    """(2+1)D factorised conv (r2plus1d.py:85-88): spatial conv + its own BN + ReLU, then the temporal conv whose
    epilogue carries the *outer* BN / residual / ReLU."""
    mid = conv_bn_act(conv.spatial_conv, conv.bn, a, relu=True, simt=simt)
    return conv_bn_act(conv.temporal_conv, bn, mid, residual=residual, relu=relu, simt=simt, out=out)


def conv_bn_act(conv, bn, a, residual=None, relu=False, simt=False, pool_w=False, out=None):
    """Run ``conv`` (Conv3d / Conv2d / SpatioTemporalConv-like) -> ``bn`` -> (+residual) -> (ReLU).  ``pool_w``: stem only, see
    ``_stem_body``.  ``out``: preallocated output rows (``ops.conv``)."""
    if hasattr(conv, "spatial_conv") and hasattr(conv, "temporal_conv"):
        return Fn.frozen(lambda x, o: _st_conv_body(conv, bn, x, residual, relu, simt, o), a, out)
    stem = a.ld == 4
    if stem and not _is_stem_shape(conv):
        raise NotImplementedError("NDHWC4 inputs are only supported by 7-wide stride-2 stem convolutions")
    if a.W % 2 != 0 and stem:
        raise ValueError("stem convolution needs an even input width (got %d)" % a.W)
    stride, padding = _conv_geometry(conv)
    if (not simt and tuple(conv.weight.shape[2:]) in ((1, 1, 1), (1, 1)) and padding == (0, 0, 0)
            and stride[0] == stride[1] == stride[2] and stride[0] > 1 and a.T > 1):
        # strided 1x1x1 projection (type-B shortcut, resnet3D.py:176-185): the strided pixel subset is gathered
        # once (1/s^3 of the input) and the projection becomes a plain HBM-bound GEMM on the persistent kernel
        sub = ops.shortcut_a(a, stride[0], a.C)
        pc = packed_conv(conv, bn, sub.ld, stride=(1, 1, 1))
        return ops.conv(sub, pc, residual=residual, relu=relu, out=out)
    pc = packed_conv(conv, bn, a.ld, stem=stem, dense=simt)
    return ops.conv(a, pc, residual=residual, relu=relu, simt=simt, pool_w=pool_w, out=out)


# ---------------------------------------------------------------------------------------------
# residual blocks
# ---------------------------------------------------------------------------------------------
def _shortcut(block, a, simt):
    ds = block.downsample
    if ds is None:
        return a
    if isinstance(ds, nn.Sequential):          # type B: 1x1x1 conv (stride s) + BN
        return conv_bn_act(ds[0], ds[1], a, relu=False, simt=simt)
    if hasattr(ds, "planes") and hasattr(ds, "stride"):   # type A (ShortcutA)
        return ops.shortcut_a(a, ds.stride, ds.planes)
    raise NotImplementedError("unsupported downsample %r" % (ds,))


def run_basic(block, a, simt=False, out=None):
    """conv-BN-ReLU-conv-BN-(+shortcut)-ReLU (resnet3D.py:91-106)."""
    return Fn.frozen(lambda x, o: _basic_body(block, x, simt, o), a, out)


def _basic_body(block, a, simt=False, out=None, keep=None):
    """``keep``: a list that receives the post-ReLU intermediate (the fine-tuning backward reads it)."""
    res = _shortcut(block, a, simt)
    h = conv_bn_act(block.conv1, block.bn1, a, relu=True, simt=simt)
    if keep is not None:
        keep.append(h)
    return conv_bn_act(block.conv2, block.bn2, h, residual=res, relu=True, simt=simt, out=out)


def _plain_1x1(conv):
    return (isinstance(conv, (nn.Conv3d, nn.Conv2d)) and all(k == 1 for k in conv.weight.shape[2:]) and conv.groups == 1
            and all(p == 0 for p in _conv_geometry(conv)[1]))


def _active_nonlocal(block):
    nl = getattr(block, "nonlocalblock", None)
    return nl if nl is not None and getattr(block, "nonlocal_layer", True) else None


def _chains(block, nxt, simt=False):
    """Does ``block``'s closing kernel also compute ``nxt``'s conv1 (ops.gemm_chain), so that the block output is not read
    back from HBM?  Decided from the model alone: two plain (not pre-activation) bottlenecks, no non-local block after
    ``block``, ``nxt.conv1`` a bias-free stride-1 1x1(x1) convolution, a closing width N % 64 == 0 with N <= 256 (layer1)
    and a conv1 of at most 128 output channels; never under ``simt``."""
    import torchvision.models.resnet as tvresnet
    from .models.resnet3d import Bottleneck
    from .models.nonlocalnet import NonLocalBottleneck
    kinds = (Bottleneck, NonLocalBottleneck, tvresnet.Bottleneck)
    if simt or type(block) not in kinds or type(nxt) not in kinds or _active_nonlocal(block) is not None:
        return False
    c3, c1 = block.conv3, nxt.conv1
    if not (_plain_1x1(c3) and _plain_1x1(c1)) or c1.bias is not None:
        return False
    if any(s != 1 for s in _conv_geometry(c3)[0] + _conv_geometry(c1)[0]):
        return False
    N = c3.weight.shape[0]
    return N % 64 == 0 and N <= 256 and c1.weight.shape[1] == N and ops._round_up(c1.weight.shape[0], 8) <= 128


def _chained_close(block, nxt, h, w3, scale, shift, residual=None, second=None, out=None):
    """The closing 1x1x1 GEMM of ``block`` (weights ``w3`` over ``h``) with ``nxt``'s conv1 chained on: (y, nxt's h1).  conv1 uses
    the packed fp16 filter and fp32 affine of its stand-alone launch, so h1 is bit-identical to it."""
    K = w3.shape[0]
    pc1 = packed_conv(nxt.conv1, nxt.bn1, ops._round_up(K, 8))
    w1 = pc1.w.view(pc1.K, pc1.C)
    y, h1 = ops.gemm_chain(h.data, w3, scale, shift, h.M, K, h.ld, w1, pc1.scale, pc1.shift, pc1.K,
                           residual=residual.data if residual is not None else None, relu=True, second=second, out=out)
    return Act(y, h.N, h.T, h.H, h.W, K), Act(h1, h.N, h.T, h.H, h.W, pc1.K)


def _fused_close_with_projection(block, a, h, out=None, nxt=None):
    """conv3 + bn3 + (downsample conv + bn)(x) + ReLU as ONE two-operand GEMM (resnet3D.py:136-143 with the type-B
    shortcut of resnet3D.py:176-185): both BatchNorm scales are folded into the fp16 weight matrices, both products
    accumulate in the same accumulator tile, and the projected shortcut never goes through HBM.  ``nxt``: chain the next
    block's conv1 on (``_chained_close``)."""
    ds_conv, ds_bn = block.downsample[0], block.downsample[1]
    stride = _conv_geometry(ds_conv)[0]
    xs = a if stride == (1, 1, 1) else ops.shortcut_a(a, stride[0], a.C)
    if xs.M != h.M:
        raise RuntimeError("shortcut / main path shape mismatch")
    dev = a.data.device

    def build():
        s3, b3 = ops.fold_affine(block.conv3.weight.shape[0], block.conv3.bias, block.bn3, dev)
        sd, bd = ops.fold_affine(ds_conv.weight.shape[0], ds_conv.bias, ds_bn, dev)
        K = block.conv3.weight.shape[0]
        w3 = torch.zeros((K, h.ld), dtype=torch.float16, device=dev)
        w3[:, :h.C] = (_conv1x1_matrix(block.conv3).float() * s3[:, None]).to(torch.float16)
        wd = torch.zeros((K, xs.ld), dtype=torch.float16, device=dev)
        wd[:, :xs.C] = (_conv1x1_matrix(ds_conv).float() * sd[:, None]).to(torch.float16)
        return w3, wd, torch.ones(K, dtype=torch.float32, device=dev), (b3 + bd).contiguous()

    sig = _sig(block.conv3.weight, block.conv3.bias, *_bn_tensors(block.bn3), ds_conv.weight, ds_conv.bias,
               *_bn_tensors(ds_bn)) + (h.ld, xs.ld)
    w3, wd, ones, shift = _cached(block, "close2", sig, build)
    K = w3.shape[0]
    if nxt is not None:
        return _chained_close(block, nxt, h, w3, ones, shift, second=(xs.data, wd, xs.ld), out=out)
    if out is not None:
        ops._out_rows(out, h.M, ops._round_up(K, 8))
    y = ops.gemm(h.data, w3, ones, shift, h.M, K, h.ld, relu=True, second=(xs.data, wd, xs.ld), out=out)
    return Act(y, h.N, h.T, h.H, h.W, K)


def run_bottleneck(block, a, simt=False, out=None, h1=None, nxt=None):
    """1x1x1-BN-ReLU, 3x3x3(stride)-BN-ReLU, 1x1x1-BN-(+shortcut)-ReLU (resnet3D.py:125-143).  ``h1`` / ``nxt``: see
    ``_bottleneck_body``."""
    return Fn.frozen(lambda x, o: _bottleneck_body(block, x, simt, o, h1=h1, nxt=nxt), a, out)


def _bottleneck_body(block, a, simt=False, out=None, keep=None, h1=None, nxt=None):
    """``keep``: a list that receives the two post-ReLU intermediates (the fine-tuning backward reads them).  ``h1``: this
    block's conv1 output, already computed by the previous block's closing kernel (conv1 is skipped).  ``nxt``: the next
    block (``_chains(block, nxt)`` holds): the closing kernel also computes its conv1 and the body returns (y, nxt's h1)."""
    keep = [] if keep is None else keep
    ds = block.downsample
    if (not simt and isinstance(ds, nn.Sequential) and len(ds) == 2 and _plain_1x1(ds[0]) and _plain_1x1(block.conv3)
            and not ds[1].training and len(set(_conv_geometry(ds[0])[0])) == 1 and (a.T > 1 or _conv_geometry(ds[0])[0][0] == 1)
            and isinstance(ds[0], nn.Conv3d)):
        keep.append(h1 if h1 is not None else conv_bn_act(block.conv1, block.bn1, a, relu=True))
        keep.append(conv_bn_act(block.conv2, block.bn2, keep[-1], relu=True))
        return _fused_close_with_projection(block, a, keep[-1], out, nxt)
    res = _shortcut(block, a, simt)
    keep.append(h1 if h1 is not None else conv_bn_act(block.conv1, block.bn1, a, relu=True, simt=simt))
    keep.append(conv_bn_act(block.conv2, block.bn2, keep[-1], relu=True, simt=simt))
    if nxt is not None:
        h = keep[-1]
        pc3 = packed_conv(block.conv3, block.bn3, h.ld)
        return _chained_close(block, nxt, h, pc3.w.view(pc3.K, pc3.C), pc3.scale, pc3.shift, residual=res, out=out)
    return conv_bn_act(block.conv3, block.bn3, keep[-1], residual=res, relu=True, simt=simt, out=out)


def _bn_relu(bn, a):
    """Stand-alone eval-mode BatchNorm + ReLU over an activation (the pre-activation that opens a pre-act block): one
    element-wise HBM pass with the folded per-channel affine."""
    dev = a.data.device
    sc, sh = _cached(bn, "aff1", _sig(*_bn_tensors(bn)) + (a.ld,),
                     lambda: tuple(t.reshape(1, -1).contiguous() for t in ops.fold_affine(bn.num_features, None, bn, dev)))
    flat = ops.ccbn_act(Act(a.data, a.N, 1, a.T * a.H, a.W, a.C), sc, sh, relu=True)
    return Act(flat.data, a.N, a.T, a.H, a.W, a.C)


def _preact_body(block, a, simt=False, out=None):
    """PreActivationBasicBlock / PreActivationBottleneck (pre_act_resnet3D.py:41-57, 76-96):
    out = conv1(relu(bn1(x))); out = conv2(relu(bn2(out))); [out = conv3(relu(bn3(out)))]; out += shortcut(x); no ReLU.
    bn_{k+1} + ReLU run in conv_k's epilogue; the last convolution's epilogue adds the shortcut of the RAW x."""
    res = _shortcut(block, a, simt)
    h = _bn_relu(block.bn1, a)
    h = conv_bn_act(block.conv1, block.bn2, h, relu=True, simt=simt)
    if hasattr(block, "conv3"):
        h = conv_bn_act(block.conv2, block.bn3, h, relu=True, simt=simt)
        return conv_bn_act(block.conv3, None, h, residual=res, relu=False, simt=simt, out=out)
    return conv_bn_act(block.conv2, None, h, residual=res, relu=False, simt=simt, out=out)


def run_block(block, a, simt=False, out=None, h1=None, nxt=None):
    """One residual block (+ its non-local block).  ``out``: preallocated rows for the block's result (the last kernel writes there).
    ``h1`` / ``nxt`` (bottlenecks paired by ``_chains``): see ``_bottleneck_body``; with ``nxt`` the result is (y, nxt's h1)."""
    nl = _active_nonlocal(block)
    bout = out if nl is None else None
    if h1 is not None or nxt is not None:
        y = run_bottleneck(block, a, simt, bout, h1, nxt)
    elif getattr(block, "preactivation", False):
        y = Fn.frozen(lambda x, o: _preact_body(block, x, simt, o), a, bout)
    else:
        y = run_bottleneck(block, a, simt, bout) if hasattr(block, "conv3") else run_basic(block, a, simt, bout)
    if nl is not None:
        y = run_nonlocal(nl, y, simt=simt, out=out)
    return y


# ---------------------------------------------------------------------------------------------
# non-local block (embedded gaussian, no sub-sampling)
# ---------------------------------------------------------------------------------------------
def _conv1x1_matrix(conv):
    return conv.weight.detach().reshape(conv.weight.shape[0], -1)


def _first(m):
    return m[0] if isinstance(m, nn.Sequential) else m


def _pad_cols(x2d, cols):
    """fp16 [rows][ld] -> [rows][cols] with zero columns appended (glue for operands whose K extent must be a multiple of 64)."""
    if x2d.shape[1] == cols:
        return x2d
    y = x2d.new_zeros((x2d.shape[0], cols))
    y[:, :x2d.shape[1]] = x2d
    return y


def run_nonlocal(nl, a, simt=False, out=None):
    return Fn.frozen(lambda x, o: _nonlocal_body(nl, x, simt, o), a, out)


def _nonlocal_body(nl, a, simt=False, out=None):
    """z = W(y) + x with y = softmax(theta^T phi) g  (embedded gaussian, nonlocalnet.py:143-166),
    y = softmax(x^T phi(x)) g (gaussian, :168-190), y = (theta^T phi / N) g (dot product, :192-211) or
    y = (relu(w . [theta_i ; phi_j]) / N) g (concatenation, :213-243); phi and g are max-pooled when ``sub_sample``
    (:126-131).

    The attention kernel takes d and dv in multiples of 64: the theta / phi / g projections are packed with zero rows up
    to ``dp = round_up(inter_channels, 64)`` (zero logit contributions, zero output columns -- exact), so any width the
    reference accepts runs (nonlocalresnet3d18/34 put a block on C = 64, d = 32).

    Concatenation mode: ``concat_project`` is a bias-free 1x1 Conv2d over the 2d channels of [theta_i ; phi_j] followed
    by ReLU, i.e. f_ij = relu(a_i + b_j) with a_i = w_theta . theta_i and b_j = w_phi . phi_j.  The N x N x 2d tensor the
    reference materialises is never built: a_i + b_j is the rank-2 product of Q_i = [a_i, 1, 0, ...] and K_j = [1, b_j, 0, ...]
    (64-wide), which goes through the same fused kernel with ReLU in place of the softmax (mode 2)."""
    mode = nl.mode
    if mode not in ("embedded_gaussian", "gaussian", "dot_product", "concatenation"):
        raise NotImplementedError("non-local mode %r is outside the engine's scope" % (mode,))
    d, C = nl.inter_channels, nl.in_channels
    dp = ops._round_up(d, 64)
    dev = a.data.device
    w_conv, w_bn = (nl.W[0], nl.W[1]) if isinstance(nl.W, nn.Sequential) else (nl.W, None)
    g_conv = _first(nl.g)
    concat = mode == "concatenation"
    sub = bool(nl.sub_sample)
    if mode == "gaussian":
        projected = [g_conv]
    elif concat:
        projected = [nl.theta, _first(nl.phi), g_conv]
    else:
        projected = [nl.theta, _first(nl.phi), g_conv]           # column order of the GEMM
    cp_w = nl.concat_project[0].weight if concat else None

    def block(conv):                                             # [dp][ld] fp16 weight rows + fp32 bias of one projection
        w = torch.zeros((dp, a.ld), dtype=torch.float32, device=dev)
        w[:d, :C] = _conv1x1_matrix(conv).float()
        b = torch.zeros(dp, dtype=torch.float32, device=dev)
        if conv.bias is not None:
            b[:d] = conv.bias.detach().float()
        return w, b

    def scalar_block(conv, wvec, slot):
        """64 projection columns [.., wvec . conv(x), ..] with the scalar in column ``slot`` and a constant 1 in the other
        of the first two columns: Q_i = [a_i, 1, 0..] (slot 0) resp. K_j = [1, b_j, 0..] (slot 1)."""
        w = torch.zeros((64, a.ld), dtype=torch.float64, device=dev)
        b = torch.zeros(64, dtype=torch.float64, device=dev)
        w[slot, :C] = wvec.double() @ _conv1x1_matrix(conv).double()
        b[slot] = (wvec.double() @ conv.bias.detach().double()) if conv.bias is not None else 0.0
        b[1 - slot] = 1.0
        return w.float(), b.float()

    def build():
        if concat:
            wv = cp_w.detach().reshape(-1)
            q_w, q_b = scalar_block(nl.theta, wv[:d], 0)
            g_w, g_b = block(g_conv)
            if sub:      # phi must be pooled before w_phi is applied (max is not linear): full-resolution phi | g, then a small GEMM
                p_w, p_b = block(_first(nl.phi))
                ws, bs = [q_w, p_w, g_w], [q_b, p_b, g_b]
                kw = torch.zeros((64, dp), dtype=torch.float16, device=dev)
                kw[1, :d] = wv[d:].to(torch.float16)
                kshift = torch.zeros(64, dtype=torch.float32, device=dev)
                kshift[0] = 1.0
                extra = (kw, torch.ones(64, dtype=torch.float32, device=dev), kshift)
            else:
                k_w, k_b = scalar_block(_first(nl.phi), wv[d:], 1)
                ws, bs, extra = [q_w, k_w, g_w], [q_b, k_b, g_b], None
        else:
            pairs = [block(conv) for conv in projected]
            ws, bs, extra = [w for w, _ in pairs], [b for _, b in pairs], None
        w = torch.cat(ws).to(torch.float16).contiguous()
        b = torch.cat(bs).contiguous()
        wo = torch.zeros((C, dp), dtype=torch.float16, device=dev)
        wo[:, :d] = _conv1x1_matrix(w_conv).to(torch.float16)
        so, bo = ops.fold_affine(C, w_conv.bias, w_bn, dev)
        return w, b, torch.ones(w.shape[0], dtype=torch.float32, device=dev), wo, so, bo, extra

    srcs = [t for conv in projected for t in (conv.weight, conv.bias)]
    sig = _sig(*srcs, w_conv.weight, w_conv.bias, cp_w, *_bn_tensors(w_bn)) + (a.ld, mode, sub)
    wp, bp, ones, wo, so, bo, extra = _cached(nl, "proj", sig, build)

    pool = {3: (2, 2, 2), 2: (1, 2, 2), 1: (1, 1, 2)}[nl.dimension]
    B, Nq = a.N, a.positions
    amode = {"dot_product": 1, "concatenation": 2}.get(mode, 0)
    if mode == "gaussian":
        gv = ops.gemm(a.data, wp, ones, bp, a.M, dp, a.ld)                      # g(x): [M][dp]
        Cq = ops._round_up(C, 64)
        xq = _pad_cols(a.data, Cq)                                               # theta = x itself
        if sub:
            xk = ops.maxpool3d(a, pool, pool, (0, 0, 0))                           # phi = max_pool(x)
            gk = ops.maxpool3d(Act(gv, a.N, a.T, a.H, a.W, dp), pool, pool, (0, 0, 0))
            k2d, v2d, Nk = _pad_cols(xk.data, Cq), gk.data, xk.positions
        else:
            k2d, v2d, Nk = xq, gv, Nq
        y = ops.attention(xq, k2d, v2d, Cq, dp, B, Nq, Nk)
    elif concat and sub:
        q = ops.gemm(a.data, wp[:64], ones[:64], bp[:64], a.M, 64, a.ld)        # [a_i, 1, 0..]
        kv = ops.gemm(a.data, wp[64:], ones[64:], bp[64:], a.M, 2 * dp, a.ld)   # phi | g at full resolution
        kvp = ops.maxpool3d(Act(kv, a.N, a.T, a.H, a.W, 2 * dp), pool, pool, (0, 0, 0))
        kw, kones, kshift = extra
        k = ops.gemm(kvp.data, kw, kones, kshift, kvp.M, 64, dp)                 # [1, w_phi . phi_j, 0..]
        y = ops.attention(q, k, kvp.data[:, dp:], 64, dp, B, Nq, kvp.positions, mode=2)
    elif concat:
        qkv = ops.gemm(a.data, wp, ones, bp, a.M, 128 + dp, a.ld)               # [a_i,1,0..] | [1,b_j,0..] | g
        y = ops.attention(qkv, qkv[:, 64:], qkv[:, 128:], 64, dp, B, Nq, Nq, mode=2)
    elif not sub:
        qkv = ops.gemm(a.data, wp, ones, bp, a.M, 3 * dp, a.ld)                  # [M][3dp]: theta | phi | g
        y = ops.attention(qkv, qkv[:, dp:], qkv[:, 2 * dp:], dp, dp, B, Nq, Nq, mode=amode)
    else:
        q = ops.gemm(a.data, wp[:dp], ones[:dp], bp[:dp], a.M, dp, a.ld)         # theta at full resolution
        kv = ops.gemm(a.data, wp[dp:], ones[dp:], bp[dp:], a.M, 2 * dp, a.ld)    # phi | g ...
        kvp = ops.maxpool3d(Act(kv, a.N, a.T, a.H, a.W, 2 * dp), pool, pool, (0, 0, 0))   # ... max-pooled together
        y = ops.attention(q, kvp.data, kvp.data[:, dp:], dp, dp, B, Nq, kvp.positions, mode=amode)
    # W (1x1 conv with bias) + BN + residual x, no ReLU
    if out is not None:
        ops._out_rows(out, a.M, ops._round_up(C, 8))
    z = ops.gemm(y, wo, so, bo, a.M, C, dp, residual=a.data, out=out)
    return Act(z, a.N, a.T, a.H, a.W, C)


# ---------------------------------------------------------------------------------------------
# MobileNetV2 (mobilenet.py:22-126)
# ---------------------------------------------------------------------------------------------
# Every ReLU6 of the network except the last feeds a depthwise convolution: the producers (the stem conv_bn, the expansion
# 1x1 convolutions) store ReLU(x) with their ordinary epilogue and the depthwise kernel reads min(x, 6).  That is exact:
# fp16 rounding is monotone and 6 is representable, so round(min(v, 6)) == min(round(v), 6).  The last ReLU6 (the 1x1
# convolution that feeds the global average) is one in-place clamp pass.
def depthwise_bn_relu6(conv, bn, a, clamp_in=True, out=None):
    """Depthwise 3x3 conv (groups = channels, padding 1, stride 1 or 2) -> eval-mode BN -> ReLU6 on the CUDA-core kernel."""
    C = conv.weight.shape[0]
    stride, padding = _conv_geometry(conv)
    if (conv.groups != C or tuple(conv.weight.shape[1:]) != (1, 3, 3) or padding[1:] != (1, 1) or stride[1] != stride[2]
            or stride[1] not in (1, 2) or any(d != 1 for d in conv.dilation)):
        raise NotImplementedError("the depthwise kernel covers 3x3 convolutions with groups = channels, padding 1, stride 1 or 2")
    if a.C != C:
        raise ValueError("depthwise convolution over %d channels got %r" % (C, a))
    dev = a.data.device

    def build():
        w9 = conv.weight.detach().reshape(C, 9).t().float().contiguous()
        return (w9,) + ops.fold_affine(C, conv.bias, bn, dev)

    w9, scale, shift = _cached(conv, "dw", _sig(conv.weight, conv.bias, *_bn_tensors(bn)), build, reads=_bn_tensors(bn))
    return ops.dwconv3x3(a, w9, scale, shift, stride[1], clamp_in=clamp_in, out=out)


def _conv_bn_relu6_body(seq, a, clamp_out=True):
    """conv_bn / conv_1x1_bn (mobilenet.py:22-35): conv -> BN -> ReLU(6).  ``clamp_out=False`` when the only consumer is a
    depthwise convolution, which applies the upper clamp as it loads."""
    y = conv_bn_act(seq[0], seq[1], a, relu=True)
    return ops.relu6_(y) if clamp_out else y


def _inverted_residual_body(block, a, out=None):
    """[1x1 expand -> BN -> ReLU6] -> depthwise 3x3 -> BN -> ReLU6 -> 1x1 project -> BN (+ x) (mobilenet.py:38-76).  The
    residual joins in the projection GEMM's epilogue."""
    layers = list(block.conv)
    if len(layers) == 8:
        h = conv_bn_act(layers[0], layers[1], a, relu=True)
        dw, dbn, pw, pbn = layers[3], layers[4], layers[6], layers[7]
    elif len(layers) == 5:
        h = a
        dw, dbn, pw, pbn = layers[0], layers[1], layers[3], layers[4]
    else:
        raise NotImplementedError("unsupported inverted residual layout %r" % (block,))
    h = depthwise_bn_relu6(dw, dbn, h, clamp_in=True)
    return conv_bn_act(pw, pbn, h, residual=a if block.use_res_connect else None, relu=False, out=out)


def run_mobilenet_features(features, x):
    """``MobileNetV2.features`` (mobilenet.py:100-113) on the engine: fp32 NCHW (or an Act with channel pitch 8) in, Act out.
    The stem's 3 input channels are stored with pitch 8: its 3x3 stride-2 convolution runs on the generic convolution path."""
    a = x if isinstance(x, Act) else ops.from_ncdhw(x, pitch=8)
    mods = list(features)
    for i, m in enumerate(mods):
        if hasattr(m, "use_res_connect"):
            a = Fn.frozen(lambda x, o: _inverted_residual_body(m, x, o), a)
            continue
        nxt = mods[i + 1] if i + 1 < len(mods) else None
        # the output may skip the upper clamp only when a depthwise convolution is its sole reader
        feeds_dw = hasattr(nxt, "use_res_connect") and not nxt.use_res_connect and nxt.conv[0].groups > 1
        a = Fn.frozen(lambda x, o: _conv_bn_relu6_body(m, x, not feeds_dw), a)
    return a


# ---------------------------------------------------------------------------------------------
# SE-ResNet / SE-ResNeXt (senet.py:85-366)
# ---------------------------------------------------------------------------------------------
def _strided_1x1(conv, bn, a, relu, residual=None, out=None):
    """A 1x1 Conv2d of stride s > 1 (SE-ResNet's conv1, senet.py:166-167, every stage's projection, Xception's skips): the
    strided pixel subset is gathered once (1/s^2 of the input, b2_shortcut_a_ndhwc at T = 1) and the convolution runs as a
    stride-1 GEMM, with ``residual`` added in its epilogue."""
    s = _conv_geometry(conv)[0]
    if s[1] == 1:
        return conv_bn_act(conv, bn, a, residual=residual, relu=relu, out=out)
    if not (_plain_1x1(conv) and s[1] == s[2] and a.T == 1):
        raise NotImplementedError("strided 1x1 convolutions need equal in-plane strides on images")
    sub = ops.shortcut_a(a, s[1], a.C)
    pc = packed_conv(conv, bn, sub.ld, stride=(1, 1, 1))
    return ops.conv(sub, pc, residual=residual, relu=relu, out=out)


def _se_pack(block, C2):
    """Closing-GEMM filter and squeeze-excite parameters of an SE bottleneck: conv3 as fp16 [K][C2], the bn3 affine (s3, t3),
    fc1 composed with conv3 + bn3 -- w1 = W_fc1 diag(s3) W3, b1 = W_fc1 t3 + b_fc1, in fp64 then fp32 -- and fc2 in fp32."""
    se = block.se_module
    conv3, bn3 = block.conv3, block.bn3
    dev = conv3.weight.device

    def build():
        K = conv3.weight.shape[0]
        s3, t3 = ops.fold_affine(K, conv3.bias, bn3, dev)
        w3d = _conv1x1_matrix(conv3).double()                                # [K][C]
        C = w3d.shape[1]
        w3 = torch.zeros((K, C2), dtype=torch.float16, device=dev)
        w3[:, :C] = w3d.to(torch.float16)
        f1 = _conv1x1_matrix(se.fc1).double()                                # [R][K]
        b1 = se.fc1.bias.detach().double() if se.fc1.bias is not None else torch.zeros(f1.shape[0], dtype=torch.float64, device=dev)
        w1 = torch.zeros((f1.shape[0], C2), dtype=torch.float64, device=dev)
        w1[:, :C] = (f1 * s3.double()[None, :]) @ w3d
        b1f = f1 @ t3.double() + b1
        w2 = _conv1x1_matrix(se.fc2).float().contiguous()                   # [K][R]
        b2 = se.fc2.bias.detach().float().contiguous() if se.fc2.bias is not None else torch.zeros(K, dtype=torch.float32, device=dev)
        return w3, s3, t3, w1.float().contiguous(), b1f.float().contiguous(), w2, b2

    sig = _sig(conv3.weight, conv3.bias, *_bn_tensors(bn3), se.fc1.weight, se.fc1.bias, se.fc2.weight, se.fc2.bias) + (C2,)
    return _cached(block, "se", sig, build, reads=_bn_tensors(bn3))


def run_se_bottleneck(block, a, out=None):
    """SEResNetBottleneck / SEResNeXtBottleneck (senet.py:107-131) through the frozen Function."""
    return Fn.frozen(lambda x, o: _se_bottleneck_body(block, x, o), a, out)


def _se_bottleneck_body(block, a, out=None):
    """conv1-bn1-relu, conv2-bn2-relu, then out = relu(e * bn3(conv3(h2)) + shortcut) with e the SE excitation.

    The squeeze runs before conv3 (b2_se_excite: mean of h2, fc1 folded through conv3 + bn3, fc2, sigmoid) and hands the
    closing GEMM per-sample affine rows e * s3, e * t3 (b2_gemm_sample_affine_f16).  A projection shortcut runs as its own
    GEMM whose output is the closing GEMM's residual: SE scales the main path only, so the two-operand GEMM that fuses the
    projection into the closing convolution elsewhere would scale the shortcut too, and a second accumulator set would double
    the persistent kernel's accumulator registers for 4 of the 16 blocks."""
    ds = block.downsample
    if ds is None:
        res = a
    elif isinstance(ds, nn.Sequential) and len(ds) == 2 and _plain_1x1(ds[0]):
        res = _strided_1x1(ds[0], ds[1], a, relu=False)
    else:
        raise NotImplementedError("SE bottlenecks with a projection other than a 1x1 convolution + BatchNorm (senet154) are outside "
                                  "the engine's scope")
    h1 = _strided_1x1(block.conv1, block.bn1, a, relu=True)
    h2 = conv_bn_act(block.conv2, block.bn2, h1, relu=True)
    w3, s3, t3, w1, b1, w2, b2 = _se_pack(block, h2.ld)
    if (h2.N, h2.T, h2.H, h2.W) != (res.N, res.T, res.H, res.W):
        raise RuntimeError("shortcut / main path shape mismatch")
    scale, shift = ops.se_excite(h2, w1, b1, w2, b2, s3, t3)
    K = w3.shape[0]
    y = ops.gemm_sample_affine(h2.data, w3, scale, shift, h2.M, K, h2.ld, h2.positions, residual=res.data, relu=True, out=out)
    return Act(y, h2.N, h2.T, h2.H, h2.W, K)


def _se_stem_body(layer0, a, out=None):
    """layer0 of the SENets (senet.py:272-283): 7x7 stride-2 conv -> bn1 -> ReLU on the stem kernel, then
    MaxPool2d(3, stride=2, ceil_mode=True) on the pooling kernel with the ceil-mode output extent."""
    mp = layer0.pool
    k, s, p = mp.kernel_size, mp.stride, mp.padding
    if not (isinstance(k, int) and isinstance(s, int) and isinstance(p, int)) or mp.dilation not in (1, (1, 1)):
        raise NotImplementedError("the SENet stem pool must be a square, undilated MaxPool2d")
    h = conv_bn_act(layer0.conv1, layer0.bn1, a, relu=True)
    if mp.ceil_mode:
        return ops.maxpool2d_ceil(h, k, s, p, out=out)
    return ops.maxpool3d(h, (1, k, k), (1, s, s), (0, p, p), out=out)


def run_senet_trunk(model, x):
    """layer0 .. layer4 of an SENet: fp32 NCHW images (or an NDHWC4 Act) in, Act out."""
    a = x if isinstance(x, Act) else ops.from_ncdhw(x)
    a = Fn.frozen(lambda x, o: _se_stem_body(model.layer0, x, o), a)
    for name in ("layer1", "layer2", "layer3", "layer4"):
        for blk in getattr(model, name):
            a = run_se_bottleneck(blk, a)
    return a


# ---------------------------------------------------------------------------------------------
# BNInception (bninception.py:27-495)
# ---------------------------------------------------------------------------------------------
def _split_pack(model, names, in_pitch):
    """Packed B and affine of a split GEMM over the 1x1 convolutions ``names`` (each followed by ``name + '_bn'``) that read the
    same input: destination d's fp16 filter rows and folded (conv bias + BN) affine from packed column 64 * box0[d] on, zero
    rows in the padding of its last 64-column box (ops.split_plan).  Cached on the first convolution."""
    return _split_pack_convs([getattr(model, n) for n in names], [getattr(model, n + '_bn') for n in names], in_pitch)


def _split_pack_convs(convs, bns, in_pitch):
    """``_split_pack`` over 1x1 convolutions ``convs``, each followed by BatchNorm ``bns[i]``."""
    dev = convs[0].weight.device

    def build():
        npad, box0 = ops.split_plan([c.weight.shape[0] for c in convs])
        w = torch.zeros((npad, in_pitch), dtype=torch.float16, device=dev)
        scale = torch.zeros(npad, dtype=torch.float32, device=dev)
        shift = torch.zeros(npad, dtype=torch.float32, device=dev)
        for d, (c, bn) in enumerate(zip(convs, bns)):
            K, r0 = c.weight.shape[0], 64 * box0[d]
            w[r0:r0 + K, :c.weight.shape[1]] = _conv1x1_matrix(c).float().to(torch.float16)
            scale[r0:r0 + K], shift[r0:r0 + K] = ops.fold_affine(K, c.bias, bn, dev)
        return w, scale, shift

    tensors = [t for c, bn in zip(convs, bns) for t in (c.weight, c.bias) + _bn_tensors(bn)]
    reads = tuple(t for c, bn in zip(convs[1:], bns[1:]) for t in (c.weight, c.bias)) + tuple(t for bn in bns for t in _bn_tensors(bn))
    return _cached(convs[0], "split", _sig(*tensors) + (in_pitch,), build, reads=reads)


def _pool2d(pool):
    """(kernel, stride, padding) of a square nn.MaxPool2d / nn.AvgPool2d with ceil_mode=True and no dilation."""
    two = lambda v: (v, v) if isinstance(v, int) else tuple(v)
    k, s, p = two(pool.kernel_size), two(pool.stride), two(pool.padding)
    if (k[0] != k[1] or s[0] != s[1] or p[0] != p[1] or not pool.ceil_mode or getattr(pool, 'dilation', 1) not in (1, (1, 1))
            or (isinstance(pool, nn.AvgPool2d) and not pool.count_include_pad)):
        raise NotImplementedError("BNInception pools are square ceil-mode windows (average pools count the padding)")
    return k[0], s[0], p[0]


def run_inception(model, spec, a, out=None):
    """One inception block of BNInception (``spec``: a row of models.bninception.BLOCKS) through the frozen Function."""
    return Fn.frozen(lambda x, o: _inception_body(model, spec, x, o), a, out)


def _inception_body(model, spec, a, out=None):
    """The branches of an inception block (bninception.py:266-288 and the other blocks) each write their columns of the
    concatenated output ``y`` [M][out] in place -- no copies, no padding columns:

    * one split GEMM over the block input computes the 1x1 head straight into its slice and the two 3x3 reduces into their own
      matrices (the three 1x1 convolutions that read the input, as one pass over it);
    * the 3x3 branch and the second 3x3 of the double branch write their slices (slice convolutions, stride 2 in 3c / 4e);
    * the pool branch pools the block input -- AvgPool2d(3, 1, 1) (MaxPool2d at 5b) into a dense matrix that its projection GEMM
      reads and writes into its slice, or, in the stride-2 blocks, MaxPool2d(3, 2, ceil_mode) straight into the pass-through slice.

    Six launches per stride-1 block (the block input is read by the split GEMM and the pool), five per stride-2 block."""
    from .models.bninception import block_out_channels
    n, cin, c1, (c3r, c3), (cdr, cd), (pk, proj) = spec
    p = 'inception_%s_' % n
    if a.C != cin or a.ld != cin:
        raise ValueError("inception_%s takes a dense [M][%d] input, got %r" % (n, cin, a))
    pool = getattr(model, p + 'pool')
    k, s, pd = _pool2d(pool)
    Ho, Wo = ops.ceil_pool_dim(a.H, k, s, pd), ops.ceil_pool_dim(a.W, k, s, pd)
    if s > 1 and (Ho, Wo) != (ops._out_dim(a.H, 3, 2, 1), ops._out_dim(a.W, 3, 2, 1)):
        raise ValueError("inception_%s: the stride-2 pool and convolutions disagree on a %dx%d map" % (n, a.H, a.W))
    C = block_out_channels(spec)
    M = a.N * a.T * Ho * Wo
    dev = a.data.device
    y = ops._out_rows(out, M, C) if out is not None else torch.empty((M, C), dtype=torch.float16, device=dev)
    r3 = torch.empty((a.M, c3r), dtype=torch.float16, device=dev)
    rd = torch.empty((a.M, cdr), dtype=torch.float16, device=dev)
    heads = ([p + '1x1'] if c1 is not None else []) + [p + '3x3_reduce', p + 'double_3x3_reduce']
    w, scale, shift = _split_pack(model, heads, a.ld)
    col = c1 or 0
    ops.gemm_split(a.data, w, scale, shift, a.M, a.ld, ([y[:, :col]] if c1 is not None else []) + [r3, rd], relu=True)
    conv = getattr(model, p + '3x3')
    ops.conv_slice(Act(r3, a.N, a.T, a.H, a.W, c3r), packed_conv(conv, getattr(model, p + '3x3_bn'), c3r), y[:, col:col + c3])
    col += c3
    d1 = conv_bn_act(getattr(model, p + 'double_3x3_1'), getattr(model, p + 'double_3x3_1_bn'), Act(rd, a.N, a.T, a.H, a.W, cdr),
                     relu=True)
    conv = getattr(model, p + 'double_3x3_2')
    ops.conv_slice(d1, packed_conv(conv, getattr(model, p + 'double_3x3_2_bn'), d1.ld), y[:, col:col + cd])
    col += cd
    avg = isinstance(pool, nn.AvgPool2d)
    if proj is None:
        ops.pool_slice(a, k, s, pd, avg, y[:, col:])
    else:
        pooled = ops.pool_slice(a, k, s, pd, avg)
        w, scale, shift = _split_pack(model, [p + 'pool_proj'], pooled.ld)
        ops.gemm_split(pooled.data, w, scale, shift, pooled.M, pooled.ld, [y[:, col:col + proj]], relu=True)
    return Act(y, a.N, a.T, Ho, Wo, C)


def _bninception_stem_body(model, a, out=None):
    """conv1_7x7_s2 -> BN -> ReLU on the stem kernel, pool1 (MaxPool2d(3, 2, ceil_mode)), conv2_3x3_reduce and conv2_3x3 (each
    -> BN -> ReLU), pool2 (bninception.py:255-265)."""
    h = conv_bn_act(model.conv1_7x7_s2, model.conv1_7x7_s2_bn, a, relu=True)
    h = ops.maxpool2d_ceil(h, *_pool2d(model.pool1_3x3_s2))
    h = conv_bn_act(model.conv2_3x3_reduce, model.conv2_3x3_reduce_bn, h, relu=True)
    h = conv_bn_act(model.conv2_3x3, model.conv2_3x3_bn, h, relu=True)
    return ops.maxpool2d_ceil(h, *_pool2d(model.pool2_3x3_s2), out=out)


def run_bninception_trunk(model, x):
    """The BNInception trunk: fp32 NCHW images (or an NDHWC4 Act) in, the 5b block output (an Act) out."""
    from .models.bninception import BLOCKS
    a = x if isinstance(x, Act) else ops.from_ncdhw(x)
    a = Fn.frozen(lambda x, o: _bninception_stem_body(model, x, o), a)
    for spec in BLOCKS:
        a = run_inception(model, spec, a)
    return a


# ---------------------------------------------------------------------------------------------
# Inception-v4 / Inception-ResNet-v2 (inceptionv4.py:34-309, inceptionresnetv2.py:34-331) and Inception-v3 (torchvision's
# Inception3 behind torchvision_models.py:380-437): torchvision's BasicConv2d has the same conv / bn (eps 0.001) fields
# ---------------------------------------------------------------------------------------------
def _is_head(u):
    """A BasicConv2d whose convolution is 1x1, stride 1, padding 0: it runs inside a split GEMM."""
    c = u.conv
    return tuple(c.kernel_size) == (1, 1) and tuple(c.stride) == (1, 1) and tuple(c.padding) == (0, 0)


def _max3s2(a, y=None):
    """nn.MaxPool2d(3, stride=2) (floor mode) on the slice pool; on the odd maps of these networks it is the ceil-mode window."""
    if (a.H - 3) % 2 or (a.W - 3) % 2:
        raise ValueError("MaxPool2d(3, stride=2) runs on odd maps here (299x299 inputs), got %dx%d" % (a.H, a.W))
    return ops.pool_slice(a, 3, 2, 0, False, y)


def _basic_unit(u, a, y=None):
    """BasicConv2d ``u`` (conv -> BN -> ReLU) of ``a``: a 1x1 on the GEMM, any filter with taps on the slab kernel's slice entry,
    written into ``y`` (an fp16 [M][K] column slice) or a fresh dense matrix."""
    if _is_head(u):
        if y is None:
            return conv_bn_act(u.conv, u.bn, a, relu=True)
        w, scale, shift = _split_pack_convs([u.conv], [u.bn], a.ld)
        ops.gemm_split(a.data, w, scale, shift, a.M, a.ld, [y], relu=True)
        return Act(y, a.N, a.T, a.H, a.W, y.shape[1])
    pc = packed_conv(u.conv, u.bn, a.ld)
    if y is None:
        (_, sh, sw), (_, ph, pw) = _conv_geometry(u.conv)
        M = a.N * a.T * ops._out_dim(a.H, pc.k[1], sh, ph) * ops._out_dim(a.W, pc.k[2], sw, pw)
        y = torch.empty((M, ops._round_up(pc.K, 8)), dtype=torch.float16, device=a.data.device)[:, :pc.K]
    return ops.conv_slice(a, pc, y)


def _inception_stem_body(units, a, out=None):
    """The units before the first block (BasicConv2d / MaxPool2d(3, 2)) in sequence, and Inception-ResNet-v2's closing conv2d_7b.
    The 3-channel input has pitch 8: the 3x3 stride-2 valid convolution runs on the slab kernel like MobileNetV2's stem."""
    for i, u in enumerate(units):
        last = i == len(units) - 1
        if isinstance(u, nn.MaxPool2d):
            a = _max3s2(a, None if not last or out is None else out)
        else:
            a = _basic_unit(u, a, out if last and out is not None else None)
    return a


def _branch_width(block, a, br):
    if br[0] == 'max':
        return a.C
    if br[0] == 'fork':
        return sum(block.get_submodule(p).conv.out_channels for p in br[2])
    return block.get_submodule(br[1][-1]).conv.out_channels


def _branch_hw(block, a, br):
    """Output map of a branch: MaxPool2d(3, 2), or its chain's convolutions in sequence (every branch of a block agrees)."""
    if br[0] == 'max':
        return ops._out_dim(a.H, 3, 2, 0), ops._out_dim(a.W, 3, 2, 0)
    H, W = a.H, a.W
    for p in (br[1] if br[0] != 'fork' else br[1] + [br[2][0]]):
        (_, sh, sw), (_, ph, pw) = _conv_geometry(block.get_submodule(p).conv)
        kh, kw = block.get_submodule(p).conv.kernel_size
        H, W = ops._out_dim(H, kh, sh, ph), ops._out_dim(W, kw, sw, pw)
    return H, W


def _branch_heads(get, branches, a, y, cols, temps):
    """The 1x1 units of a row that read the block input ``a`` (``get``: the block's get_submodule) and their split-GEMM
    destinations: a lone 1x1 branch writes its slice of ``y``, the first unit of a longer chain a fresh matrix (kept in ``temps``
    under its path)."""
    heads, dests = [], []
    for br, c0 in zip(branches, cols):
        if br[0] in ('chain', 'fork') and _is_head(get(br[1][0])):
            u = get(br[1][0])
            K = u.conv.out_channels
            if br[0] == 'chain' and len(br[1]) == 1:
                dests.append(y[:, c0:c0 + K])
            else:
                temps[br[1][0]] = torch.empty((a.M, K), dtype=torch.float16, device=a.data.device)
                dests.append(temps[br[1][0]])
            heads.append(u)
    return heads, dests


def _branch_bodies(get, branches, a, y, cols, widths, temps):
    """Everything of a row after its split GEMM: pools, and the units of each chain / fork after its head, each branch ending in
    its slice of ``y``."""
    for br, c0, wd in zip(branches, cols, widths):
        if br[0] == 'max':
            _max3s2(a, y[:, c0:c0 + wd])
        elif br[0] == 'avg':
            pooled = ops.pool_slice(a, 3, 1, 1, True, count_include_pad=br[2])
            _basic_unit(get(br[1][-1]), pooled, y[:, c0:c0 + wd])
        else:
            paths = br[1]
            h = Act(temps[paths[0]], a.N, a.T, a.H, a.W, temps[paths[0]].shape[1]) if paths[0] in temps else a
            rest = [get(p) for p in paths[(1 if paths[0] in temps or _is_head(get(paths[0])) else 0):]]
            ends = [get(p) for p in br[2]] if br[0] == 'fork' else rest[-1:]
            for u in (rest if br[0] == 'fork' else rest[:-1]):
                h = _basic_unit(u, h)
            c = c0
            for u in ends:
                K = u.conv.out_channels
                _basic_unit(u, h, y[:, c:c + K])
                c += K


def _inception_block_body(block, a, out=None, row=None):
    """One block of Inception-v4 / Inception-ResNet-v2 / Inception-v3 from its row of models.inception.BRANCHES (or ``row``: a
    row of another table in that format, as PolyNet's).  The branches write their columns of the concatenated output ``y`` in
    place:

    * the 1x1 units that read the block input (a lone 1x1 branch straight into its slice, the first unit of a longer chain into its
      own matrix) run as one split GEMM -- one pass over the block input;
    * every later unit of a chain runs on the slab kernel's slice entry, the last one into the branch's slice; a fork's two units
      read the same matrix and write adjacent slices;
    * a max branch pools the block input into its slice; an average branch pools it (count_include_pad as its row says: False in
      Inception-v4 / Inception-ResNet-v2, True in Inception-v3) into a matrix that its 1x1 projection reads, writing its slice;
    * a residual block (Block35 / 17 / 8) closes with one GEMM over ``y``: per-column scale ``block.scale``, shift
      ``scale * bias``, the block input as residual, ReLU unless ``noReLU`` (inceptionresnetv2.py:113-117)."""
    from .models.inception import BRANCHES, RESIDUAL
    kind = getattr(type(block), 'kind', None) or type(block).__name__
    branches = BRANCHES[kind] if row is None else row
    get = block.get_submodule
    if a.ld != a.C:
        raise ValueError("%s takes a dense [M][C] input, got %r" % (kind, a))
    Ho, Wo = _branch_hw(block, a, branches[0])
    widths = [_branch_width(block, a, br) for br in branches]
    cols = [sum(widths[:i]) for i in range(len(widths))]
    C = sum(widths)
    M = a.N * a.T * Ho * Wo
    dev = a.data.device
    residual = row is None and kind in RESIDUAL
    if out is not None and not residual:
        y = ops._out_rows(out, M, C)
    else:
        y = torch.empty((M, C), dtype=torch.float16, device=dev)
    temps = {}
    heads, dests = _branch_heads(get, branches, a, y, cols, temps)
    if heads:
        w, scale, shift = _split_pack_convs([u.conv for u in heads], [u.bn for u in heads], a.ld)
        ops.gemm_split(a.data, w, scale, shift, a.M, a.ld, dests, relu=True)
    _branch_bodies(get, branches, a, y, cols, widths, temps)
    if not residual:
        return Act(y, a.N, a.T, Ho, Wo, C)
    conv = block.conv2d
    K = conv.out_channels

    def build():
        s = torch.full((K,), float(block.scale), dtype=torch.float64, device=dev)
        return (_conv1x1_matrix(conv).float().to(torch.float16).contiguous(), s.float().contiguous(),
                (s * conv.bias.detach().double()).float().contiguous())

    w, scale, shift = _cached(conv, "res", _sig(conv.weight, conv.bias) + (float(block.scale),), build)
    z = ops.gemm(y, w, scale, shift, M, K, C, residual=a.data, relu=not getattr(block, 'noReLU', False), out=out)
    return Act(z, a.N, a.T, Ho, Wo, K)


def run_inception_trunk(n_stem, units, x):
    """The trunk of Inception-v4 (``units`` = ``features``), Inception-ResNet-v2 or Inception-v3: fp32 NCHW images (or an Act
    with channel pitch 8) in, the final 8x8 map (an Act; 1536 channels, 2048 for Inception-v3) out.  ``units[:n_stem]`` run as
    one frozen Function call of ``_inception_stem_body``, every block as one of ``_inception_block_body``, a trailing BasicConv2d
    (conv2d_7b) as a stem call of its own."""
    from .models.inception import BasicConv2d
    a = x if isinstance(x, Act) else ops.from_ncdhw(x, pitch=8)
    if (a.H, a.W) != (299, 299):
        # the final pool is the reference's fixed AvgPool2d(8): only an 8x8 final map gives one vector per image
        raise ValueError("the final pool is AvgPool2d(8): it needs an 8x8 final map (299x299 inputs), got a %dx%d input" % (a.H, a.W))
    a = Fn.frozen(lambda x, o: _inception_stem_body(tuple(units[:n_stem]), x, o), a)
    for u in units[n_stem:]:
        if isinstance(u, BasicConv2d):
            a = Fn.frozen(lambda x, o: _inception_stem_body((u,), x, o), a)
        else:
            a = Fn.frozen(lambda x, o: _inception_block_body(u, x, o), a)
    return a


# ---------------------------------------------------------------------------------------------
# PolyNet (polynet.py): the Inception block path above, 2-way modules closed by one two-operand GEMM, poly-3 modules by the dual GEMM
# ---------------------------------------------------------------------------------------------
def _polynet_stem_body(stem, a):
    """conv1 (three BasicConv2d units), then the stem's three concatenations as rows Stem1-3 of models.polynet.BRANCHES
    (polynet.py:91-105)."""
    from .models.polynet import BRANCHES
    a = _inception_stem_body(tuple(stem.conv1), a)
    for k in ('Stem1', 'Stem2', 'Stem3'):
        a = _inception_block_body(stem, a, row=BRANCHES[k])
    return a


def _polynet_2way_body(module, a):
    """out = relu(x + s * A(x) + s * B(x)) (MultiWay, polynet.py:329-344).  Both blocks write their branches into their own
    concatenation matrix; their 1x1 heads, which all read x, run as one split GEMM (two when there are more heads than its four
    destinations: Inception-ResNet-A's three per block).  The close is ONE two-operand GEMM over both matrices, with
    s * (closing BatchNorm scale) folded into each fp16 filter and the shifts summed, x as residual and ReLU: x + s * A(x) is never
    written out."""
    from .models.polynet import BRANCHES
    blocks = list(module.blocks)
    if len(blocks) != 2:
        raise NotImplementedError("the engine runs 2-way modules, got %d blocks" % len(blocks))
    branches = BRANCHES[type(blocks[0]).__name__]
    if a.ld != a.C:
        raise ValueError("%s takes a dense [M][C] input, got %r" % (type(module).__name__, a))
    widths = [_branch_width(blocks[0], a, br) for br in branches]
    cols = [sum(widths[:i]) for i in range(len(widths))]
    C = sum(widths)
    dev = a.data.device
    ys, temps, heads, dests = [], [], [], []
    for b in blocks:
        y = torch.empty((a.M, C), dtype=torch.float16, device=dev)
        t = {}
        h, d = _branch_heads(b.get_submodule, branches, a, y, cols, t)
        ys.append(y)
        temps.append(t)
        heads.append(h)
        dests.append(d)
    groups = [(heads[0] + heads[1], dests[0] + dests[1])] if len(heads[0]) + len(heads[1]) <= 4 else list(zip(heads, dests))
    for hs, ds in groups:
        w, scale, shift = _split_pack_convs([u.conv for u in hs], [u.bn for u in hs], a.ld)
        ops.gemm_split(a.data, w, scale, shift, a.M, a.ld, ds, relu=True)
    for b, y, t in zip(blocks, ys, temps):
        _branch_bodies(b.get_submodule, branches, a, y, cols, widths, t)
    units = [b.conv2d for b in blocks]
    K = units[0].conv.out_channels

    def build():
        s = float(module.scale)
        ws, shift = [], torch.zeros(K, dtype=torch.float64, device=dev)
        for u in units:
            sb, tb = ops.fold_affine(K, None, u.bn, dev)
            ws.append((_conv1x1_matrix(u.conv).double() * (s * sb.double())[:, None]).to(torch.float16).contiguous())
            shift = shift + s * tb.double()
        return ws[0], ws[1], torch.ones(K, dtype=torch.float32, device=dev), shift.float().contiguous()

    sig = _sig(*[t for u in units for t in (u.conv.weight,) + _bn_tensors(u.bn)]) + (float(module.scale),)
    w0, w1, ones, shift = _cached(module, "close2", sig, build)
    z = ops.gemm(ys[0], w0, ones, shift, a.M, K, C, residual=a.data, relu=True, second=(ys[1], w1, C))
    return Act(z, a.N, a.T, a.H, a.W, K)


def _poly_split_pack(module, heads, i, in_pitch):
    """The split GEMM of one poly application's 1x1 heads (PolyConv2d units reading x_i): the fp16 filter rows packed once per
    module, the folded affine of BatchNorms ``bn_blocks[i]`` per application (its cache key holds those BatchNorms)."""
    dev = heads[0].conv.weight.device

    def build(bns):
        npad, box0 = ops.split_plan([u.conv.out_channels for u in heads])
        w = torch.zeros((npad, in_pitch), dtype=torch.float16, device=dev)
        scale = torch.zeros(npad, dtype=torch.float32, device=dev)
        shift = torch.zeros(npad, dtype=torch.float32, device=dev)
        for d, (u, bn) in enumerate(zip(heads, bns)):
            K, r0 = u.conv.out_channels, 64 * box0[d]
            w[r0:r0 + K, :u.conv.in_channels] = _conv1x1_matrix(u.conv).float().to(torch.float16)
            scale[r0:r0 + K], shift[r0:r0 + K] = ops.fold_affine(K, None, bn, dev)
        return w, scale, shift

    bns = [u.bn_blocks[i] for u in heads]
    w = _cached(module, "poly_split_w", _sig(*[u.conv.weight for u in heads]) + (in_pitch,), lambda: build([None] * len(heads))[0])
    sig = _sig(*[t for bn in bns for t in _bn_tensors(bn)]) + (id(bns[0]), in_pitch)
    scale, shift = _cached(module, "poly_split_aff%d" % i, sig, lambda: build(bns)[1:], reads=tuple(t for bn in bns for t in _bn_tensors(bn)))
    return w, scale, shift


def _poly_conv(unit, i, in_pitch):
    """PackedConv of PolyConv2d ``unit`` with BatchNorm ``bn_blocks[i]``: the fp16 filter is packed once (cached on the unit) and
    shared by every application; each application's pack carries only its own folded affine (cached on its BatchNorm)."""
    conv, bn = unit.conv, unit.bn_blocks[i]
    stride, padding = _conv_geometry(conv)
    base = _cached(unit, "poly_w", _sig(conv.weight) + (in_pitch,),
                   lambda: ops.PackedConv(conv.weight.detach(), None, None, stride, padding, in_pitch=in_pitch))

    def build():
        pc = copy.copy(base)
        pc.scale, pc.shift = ops.fold_affine(conv.out_channels, None, bn, conv.weight.device)
        return pc

    return _cached(bn, "poly_pc", _sig(conv.weight, *_bn_tensors(bn)) + (in_pitch,), build, reads=(conv.weight,))


def _polynet_poly_body(module, a):
    """out = x; for i: f = F_i(x_i); out += s * f; x_{i+1} = relu(f); relu(out) (InceptionResNetB/CPoly, polynet.py:229-326).
    Application i: its 1x1 heads over x_i as one split GEMM (the 1x1 into a matrix, ``path1`` into its slice), the 1xn and nx1
    convolutions on the slab kernel (the second into its slice), and the close over the concatenation: with (sb, tb) the folded
    BatchNorm of ``conv2d_blocks[i]``, scale s * sb, shift s * tb and the running sum as residual.  Every application but the last
    closes with the dual GEMM, which also writes x_{i+1} = relu(sb * acc + tb) from the same accumulator; the last one is the
    residual GEMM with ReLU."""
    from .models.polynet import BRANCHES
    (_, chain), (_, (lone,)) = BRANCHES[module.kind]
    h1x1, ha, hb = (getattr(module, n) for n in chain)
    p1 = getattr(module, lone)
    if a.ld != a.C:
        raise ValueError("%s takes a dense [M][C] input, got %r" % (type(module).__name__, a))
    K0, Ka, Kb = h1x1.conv.out_channels, ha.conv.out_channels, hb.conv.out_channels
    C = Kb + p1.conv.out_channels
    K = module.conv2d_blocks[0].conv.out_channels
    dev = a.data.device
    M = a.M
    geo = (a.N, a.T, a.H, a.W)
    x, total = a, a.data
    s = float(module.scale)
    n = module.num_blocks
    for i in range(n):
        y = torch.empty((M, C), dtype=torch.float16, device=dev)
        t0 = torch.empty((M, K0), dtype=torch.float16, device=dev)
        w, scale, shift = _poly_split_pack(module, [h1x1, p1], i, x.ld)
        ops.gemm_split(x.data, w, scale, shift, M, x.ld, [t0, y[:, Kb:]], relu=True)
        ta = torch.empty((M, Ka), dtype=torch.float16, device=dev)
        ops.conv_slice(Act(t0, *geo, K0), _poly_conv(ha, i, K0), ta)
        ops.conv_slice(Act(ta, *geo, Ka), _poly_conv(hb, i, Ka), y[:, :Kb])
        unit = module.conv2d_blocks[i]

        def build(unit=unit):
            sb, tb = ops.fold_affine(K, None, unit.bn, dev)
            return (_conv1x1_matrix(unit.conv).float().to(torch.float16).contiguous(), (s * sb.double()).float().contiguous(),
                    (s * tb.double()).float().contiguous(), sb, tb)

        wc, sc, sh, sb, tb = _cached(unit, "poly_close", _sig(unit.conv.weight, *_bn_tensors(unit.bn)) + (s,), build)
        if i < n - 1:
            total, xn = ops_dual.gemm_dual(y, wc, sc, sh, sb, tb, M, K, C, residual=total)
            x = Act(xn, *geo, K)
        else:
            total = ops.gemm(y, wc, sc, sh, M, K, C, residual=total, relu=True)
    return Act(total, *geo, K)


def _polynet_block_body(module, a):
    """One module of the PolyNet trunk (PolyNet.modules_in_order)."""
    from .models import polynet as PN
    if isinstance(module, PN.Stem):
        return _polynet_stem_body(module, a)
    if isinstance(module, PN.MultiWay):
        return _polynet_2way_body(module, a)
    if isinstance(module, (PN.InceptionResNetBPoly, PN.InceptionResNetCPoly)):
        return _polynet_poly_body(module, a)
    return _inception_block_body(module, a, row=PN.BRANCHES[module.kind])


def run_polynet_trunk(model, x):
    """The PolyNet trunk: fp32 NCHW images (or an Act with channel pitch 8) in, the 9x9x2048 stage_c output (an Act) out; every
    module is one frozen Function call of ``_polynet_block_body``."""
    H, W = (x.H, x.W) if isinstance(x, Act) else tuple(x.shape[-2:])
    if (H, W) != (331, 331):
        # the final pool is the reference's fixed AvgPool2d(9): only a 9x9 final map gives one vector per image
        raise ValueError("the final pool is AvgPool2d(9): it needs a 9x9 final map (331x331 inputs), got a %dx%d input" % (H, W))
    a = x if isinstance(x, Act) else ops.from_ncdhw(x, pitch=8)
    for m in model.modules_in_order():
        a = Fn.frozen(lambda x, o: _polynet_block_body(m, x), a)
    return a


# ---------------------------------------------------------------------------------------------
# DenseNet (torchvision densenet.py behind torchvision_models.py:254-380)
# ---------------------------------------------------------------------------------------------
# Each dense block owns one fp16 [M][C_final] matrix.  Its first C0 columns are written by the stem's pool (first block) or the
# previous transition's GEMM; layer L reads columns [0, C_L) and writes [C_L, C_L + k): every column is written before it is
# read, so the concatenations of torchvision's forward are never materialised and no memset is needed.
def _bn_affine(bn, width=None):
    """Folded eval-mode affine of ``bn`` as fp32 [width] arrays, zero past bn.num_features (cached on ``bn``)."""
    C = bn.num_features
    width = C if width is None else width

    def build():
        s, t = ops.fold_affine(C, None, bn, bn.running_mean.device)
        sp = torch.zeros(width, dtype=torch.float32, device=s.device)
        tp = torch.zeros(width, dtype=torch.float32, device=s.device)
        sp[:C], tp[:C] = s, t
        return sp, tp
    return _cached(bn, "dense_aff%d" % width, _sig(*_bn_tensors(bn)) + (width,), build)


def _dense_layer_pack(layer):
    """conv1 of a dense layer as fp16 [4k][C_L], its norm1 affine padded with zeros to whole 64-column K blocks (the A transform
    of b2_gemm_preact_f16) and its norm2 affine (the epilogue)."""
    conv = layer.conv1
    C_L = conv.in_channels

    def build():
        s1, t1 = ops.fold_affine(C_L, None, layer.norm1, conv.weight.device)
        kpad = ops._round_up(C_L, 64)
        s1p = torch.zeros(kpad, dtype=torch.float32, device=s1.device)
        t1p = torch.zeros(kpad, dtype=torch.float32, device=s1.device)
        s1p[:C_L], t1p[:C_L] = s1, t1
        s2, t2 = ops.fold_affine(conv.out_channels, None, layer.norm2, conv.weight.device)
        return _conv1x1_matrix(conv).to(torch.float16).contiguous(), s1p, t1p, s2, t2
    reads = _bn_tensors(layer.norm1) + _bn_tensors(layer.norm2)
    return _cached(conv, "preact", _sig(conv.weight, *reads), build, reads=reads)


# Growth-rate 3x3 convolutions (4k -> k) that run on an N tile exactly k wide (b2_conv_ndhwc_fprop_slice_narrow) instead of the
# 64-wide one: the (k, map size) pairs where the narrow tile measured faster at both 32 and 256 images (the 7x7 maps of the last
# block; at 14 - 56 the 64-wide tile is as fast or faster at 256 images, DESIGN section 5).  Both give bitwise the same output.
_NARROW_GROWTH = frozenset({(32, 7), (48, 7)})


def _dense_layer(layer, blk):
    """One _DenseLayer (densenet.py: norm1 -> relu1 -> conv1 -> norm2 -> relu2 -> conv2) on the block matrix ``blk`` (an Act
    whose C is the block's final width): conv1 reads columns [0, C_L) through the pre-activated GEMM, with norm2 + ReLU in its
    epilogue; conv2 (3x3, no affine) writes its k columns [C_L, C_L + k) in place."""
    C_L, k = layer.conv1.in_channels, layer.conv2.out_channels
    if tuple(layer.conv1.kernel_size) != (1, 1) or tuple(layer.conv2.kernel_size) != (3, 3) or tuple(layer.conv2.padding) != (1, 1):
        raise NotImplementedError("dense layers are 1x1 -> 3x3 'same' convolutions")
    if C_L % 8 or k % 8:
        raise NotImplementedError("dense layers need input widths and a growth rate that are multiples of 8 (got %d, %d)" % (C_L, k))
    w1, s1, t1, s2, t2 = _dense_layer_pack(layer)
    K1 = w1.shape[0]
    h = ops.gemm_preact(blk.data, w1, s2, t2, s1, t1, blk.M, K1, C_L, relu=True)
    pc = packed_conv(layer.conv2, None, h.shape[1])
    ops.conv_slice(Act(h, blk.N, 1, blk.H, blk.W, K1), pc, blk.data[:, C_L:C_L + k], relu=False, narrow=(k, blk.H) in _NARROW_GROWTH)


def _dense_transition(tr, blk, y):
    """_Transition (densenet.py: norm -> relu -> conv 1x1 -> AvgPool2d(2, 2)) as norm + ReLU + pool in one pass, then the 1x1
    convolution on a quarter of the positions, written into the slice ``y`` (the next block's first C / 2 columns).  The pool and
    the bias-free 1x1 convolution are both linear, so pooling first is exact in real arithmetic."""
    s, t = _bn_affine(tr.norm)
    pooled = ops.bn_relu_avgpool2(blk, s, t)
    w, scale, shift = _split_pack_convs([tr.conv], [None], pooled.ld)
    ops.gemm_split(pooled.data, w, scale, shift, pooled.M, pooled.ld, [y], relu=False)


def _dense_stem(features, a, y):
    """conv0 -> norm0 -> relu0 on the stem kernel, pool0 (MaxPool2d(3, 2, 1)) into the slice ``y`` (the first block's first
    columns).  On the stem kernel's pooled-W path the convolution takes the pool's W direction in its epilogue."""
    conv = features.conv0
    if (a.ld == 4 and _is_stem_shape(conv) and ops._out_dim(a.W, 7, 2, 3) <= 120 and a.W % 2 == 0
            and os.environ.get("B2_STEM_POOLW", "1") != "0"):
        h = conv_bn_act(conv, features.norm0, a, relu=True, pool_w=True)
        return ops.pool_slice(h, (3, 1), (2, 1), (1, 0), False, y, ceil_mode=False)
    h = conv_bn_act(conv, features.norm0, a, relu=True)
    return ops.pool_slice(h, 3, 2, 1, False, y, ceil_mode=False)


def _densenet_trunk_body(features, a):
    """The DenseNet trunk up to the last block's output (norm5 not applied): fp16 NDHWC4 images in, an Act out."""
    mods = features._modules
    blocks = [m for n, m in mods.items() if n.startswith('denseblock')]
    trans = [m for n, m in mods.items() if n.startswith('transition')]
    pool = features.pool0
    if not (isinstance(pool, nn.MaxPool2d) and _pool_args(pool) == ((1, 3, 3), (1, 2, 2), (0, 1, 1)) and not pool.ceil_mode):
        raise NotImplementedError("DenseNet's pool0 is MaxPool2d(3, stride=2, padding=1)")
    dev = a.data.device
    C = features.conv0.out_channels
    H, W = ops._out_dim(a.H, 7, 2, 3), ops._out_dim(a.W, 7, 2, 3)
    H, W = ops._out_dim(H, 3, 2, 1), ops._out_dim(W, 3, 2, 1)
    y = None
    for i, block in enumerate(blocks):
        layers = list(block.children())
        Cf = C + sum(l.conv2.out_channels for l in layers)
        blk = Act(torch.empty((a.N * H * W, Cf), dtype=torch.float16, device=dev), a.N, 1, H, W, Cf)
        if i == 0:
            _dense_stem(features, a, blk.data[:, :C])
        else:
            _dense_transition(trans[i - 1], y, blk.data[:, :C])
        for layer in layers:
            _dense_layer(layer, blk)
        y = blk
        if i < len(trans):
            C, H, W = trans[i].conv.out_channels, H // 2, W // 2
    return y


def run_densenet_trunk(features, x):
    """DenseNet ``features`` up to norm5 through the frozen Function: fp32 NCHW images (or an NDHWC4 Act) in, the last dense block's
    output (an Act, norm5 not applied) out."""
    a = x if isinstance(x, Act) else ops.from_ncdhw(x)
    return Fn.frozen(lambda x, o: _densenet_trunk_body(features, x), a)


def densenet_norm5(features, a):
    """norm5 of the last block's output as an Act (``features()``'s tensor; off the hot path: the head applies it in its pool)."""
    s, t = _bn_affine(features.norm5, a.ld)
    return ops.ccbn_act(a, s.view(1, -1), t.view(1, -1), relu=False)


def run_densenet_head(model, a, bn=None):
    """relu(bn(x)) -> 7x7 mean -> view -> last_linear (torchvision_models.py:262-266) on the last block's output ``a``: the
    affine (norm5, or none when ``a`` already holds features()'s tensor) and the ReLU are applied inside the pool."""
    if (a.T, a.H, a.W) != (1, 7, 7):
        raise NotImplementedError("DenseNet's logits take F.avg_pool2d(kernel_size=7, stride=1) of a 7x7 final map (224x224 inputs), "
                                  "got %dx%d" % (a.H, a.W))
    if bn is None:
        s = torch.ones(a.ld, dtype=torch.float32, device=a.data.device)
        t = torch.zeros(a.ld, dtype=torch.float32, device=a.data.device)
    else:
        s, t = _bn_affine(bn, a.ld)
    return _head_on_pooled(model.last_linear, ops.avgpool_global_affine(a, s, t), a.C)


# ---------------------------------------------------------------------------------------------
# VGG / AlexNet (torchvision vgg.py / alexnet.py behind torchvision_models.py:195-248, 597-725)
# ---------------------------------------------------------------------------------------------
def _check_224(x):
    if x.dim() != 4 or tuple(x.shape[2:]) != (224, 224):
        # the reference skips torchvision's avgpool, so its view(B, -1) only fits fc6 for a 224x224 input
        raise ValueError("VGG / AlexNet take 224x224 images (the classifier reads the 7x7 / 6x6 final map as is), got %s"
                         % (tuple(x.shape),))


def _plain_stack_body(mods, a, i=0):
    """Conv2d [-> BatchNorm2d] -> ReLU units and MaxPool2d layers of a torchvision ``features`` Sequential from layer ``i`` on: each
    convolution on the convolution path with its bias (+ folded BatchNorm) and the ReLU in the epilogue, each pool on the pooling
    kernel (floor mode)."""
    while i < len(mods):
        m = mods[i]
        if isinstance(m, nn.Conv2d):
            bn = mods[i + 1] if i + 1 < len(mods) and isinstance(mods[i + 1], nn.BatchNorm2d) else None
            j = i + 1 + (bn is not None)
            if j >= len(mods) or not isinstance(mods[j], nn.ReLU):
                raise NotImplementedError("VGG / AlexNet convolutions are followed by a ReLU")
            a = conv_bn_act(m, bn, a, relu=True)
            i = j + 1
        elif isinstance(m, nn.MaxPool2d):
            if m.ceil_mode or m.dilation not in (1, (1, 1)):
                raise NotImplementedError("the engine runs floor-mode, undilated max pools here")
            a = ops.maxpool3d(a, *_pool_args(m))
            i += 1
        else:
            raise NotImplementedError("unsupported layer %r in a VGG / AlexNet trunk" % (m,))
    return a


def _vgg_trunk_body(features, a):
    """VGG's ``_features`` on the pitch-8 image ``a``: an Act [N*7*7][512] at 224x224."""
    return _plain_stack_body(list(features), a)


def _alexnet_trunk_body(features, a):
    """AlexNet's ``_features`` on the space-to-depth image ``a`` (ops_vgg.space_to_depth4): conv1 (11x11, stride 4, padding 2) as
    the valid 3x3 convolution with the regrouped filter, then the rest of the stack.  An Act [N*6*6][256] at 224x224."""
    mods = list(features)
    conv = mods[0]
    if (not isinstance(conv, nn.Conv2d) or tuple(conv.kernel_size) != (11, 11) or tuple(conv.stride) != (4, 4)
            or tuple(conv.padding) != (2, 2) or conv.in_channels != 3 or not isinstance(mods[1], nn.ReLU)):
        raise NotImplementedError("AlexNet's conv1 is Conv2d(3, K, 11, stride=4, padding=2) -> ReLU")
    if a.ld != 48:
        raise ValueError("AlexNet's trunk takes the 48-channel space-to-depth image, got %r" % (a,))
    pc = _cached(conv, "s2d", _sig(conv.weight, conv.bias),
                 lambda: ops.PackedConv(ops_vgg.s2d_filter(conv.weight.detach().float()), conv.bias, None, (1, 1, 1), (0, 0, 0),
                                        in_pitch=48))
    return _plain_stack_body(mods, ops.conv(a, pc, relu=True), 2)


def run_vgg_trunk(features, x):
    """VGG ``_features`` through the frozen Function: fp32 NCHW 224x224 images in, the last pool's output (an Act) out."""
    _check_224(x)
    return Fn.frozen(lambda x, o: _vgg_trunk_body(features, x), ops.from_ncdhw(x, pitch=8))


def run_alexnet_trunk(features, x):
    """AlexNet ``_features`` through the frozen Function: fp32 NCHW 224x224 images in, the last pool's output (an Act) out."""
    _check_224(x)
    return Fn.frozen(lambda x, o: _alexnet_trunk_body(features, x), ops_vgg.space_to_depth4(x))


def _fc6_pack(linear, C, H, W):
    """fc6 as fp16 [4096][H*W*C] with its columns in the engine's (h, w, c) order (the reference flattens (c, h, w)), + bias."""
    def build():
        w = linear.weight.detach()
        if w.shape[1] != C * H * W:
            raise ValueError("fc6 takes %d features, the final map has %d x %d x %d" % (w.shape[1], C, H, W))
        wp = w.reshape(w.shape[0], C, H, W).permute(0, 2, 3, 1).reshape(w.shape[0], H * W * C)
        return ops.PackedLinear(wp.contiguous(), linear.bias)
    return _cached(linear, "fc6_hwc", _sig(linear.weight, linear.bias) + (C, H, W), build)


def _packed_linear(linear):
    return _cached(linear, "pl", _sig(linear.weight, linear.bias), lambda: ops.PackedLinear(linear.weight, linear.bias))


def classifier_gemm(x16, pl, relu=False, out_f32=False):
    """One fully connected layer on fp16 rows ``x16``: split-K (ops_vgg.gemm_splitk) with the splits b2_gemm_splitk_plan picks
    when the output tiles leave SMs idle, else the persistent GEMM."""
    M, N, Kd = x16.shape[0], pl.out_features, pl.in_features
    splits = ops_vgg.splitk_plan(M, N, Kd, _sm_count(x16.device))
    if splits > 1:
        return ops_vgg.gemm_splitk(x16, pl.w, pl.scale, pl.shift, M, N, Kd, splits, relu=relu, out_f32=out_f32)
    return ops.gemm(x16, pl.w, pl.scale, pl.shift, M, N, Kd, relu=relu, out_f32=out_f32)


_SM_COUNT = {}


def _sm_count(dev):
    idx = dev.index if dev.index is not None else torch.cuda.current_device()
    if idx not in _SM_COUNT:
        _SM_COUNT[idx] = torch.cuda.get_device_properties(idx).multi_processor_count
    return _SM_COUNT[idx]


def run_vgg_classifier(model, a):
    """view(B, -1) -> linear0 -> relu0 -> linear1 on the trunk output ``a`` ([N*H*W][C] read as [N][H*W*C]): fc6 with bias + ReLU
    into fp16, fc7 with its bias into fp32 -- ``features()``'s tensor [N][4096]."""
    if a.ld != a.C:
        raise ValueError("the classifier reads the final map as [N][H*W*C]: it needs a dense [M][C] map, got %r" % (a,))
    x = a.data.view(a.N, a.H * a.W * a.C)
    h = classifier_gemm(x, _fc6_pack(model.linear0, a.C, a.H, a.W), relu=True)
    return classifier_gemm(h, _packed_linear(model.linear1), out_f32=True)


def run_vgg_logits(model, features):
    """relu1 -> last_linear on fp32 [N][4096] features: the ReLU is applied as the rows are cast to fp16 (or, for a trainable head,
    inside functions.LinearFunction), then the classifier GEMM writes fp32 logits."""
    head = model.last_linear
    if not isinstance(head, nn.Linear):
        # user-swapped head (TRN replaces it by Dropout): hand it relu1's output, as the reference does
        return head(torch.relu(features))
    if torch.is_grad_enabled() and any(p.requires_grad for p in head.parameters()):
        return Fn.linear(features, head.weight, head.bias, relu_input=True)
    return classifier_gemm(ops.cast_rows(features, relu=True), _packed_linear(head), out_f32=True)


# ---------------------------------------------------------------------------------------------
# Xception (xception.py:50-233)
# ---------------------------------------------------------------------------------------------
# Every separable convolution is two launches: the depthwise 3x3 on CUDA cores, then the pointwise 1x1 on the persistent GEMM with
# the BatchNorm that follows it and a ReLU (the next op is another separable convolution) or the block's identity residual in its
# epilogue.  A separable convolution that a ReLU of ``rep`` opens runs its depthwise pass on max(x, 0)
# (ops_xception.dwconv3x3_relu_in): the first one reads the block input, the previous block's signed residual sum, which the skip
# path reads raw; on the later ones (a pointwise output stored after its ReLU) the max is the identity.  One that no ReLU opens (the
# first of a block built with start_with_relu=False, block1) and conv3, which reads block12's signed sum, run their depthwise pass on
# b2_dwconv3x3_ndhwc with a unit affine.
_XUnit = collections.namedtuple("_XUnit", "conv bn")


def _xception_dw(conv):
    """(fp32 [9][C] taps, unit scale, zero shift) of SeparableConv2d.conv1: a depthwise 3x3, stride 1, padding 1, no bias."""
    C = conv.weight.shape[0]
    stride, padding = _conv_geometry(conv)
    if (conv.groups != C or tuple(conv.weight.shape[1:]) != (1, 3, 3) or stride != (1, 1, 1) or padding != (0, 1, 1)
            or conv.bias is not None or any(d != 1 for d in conv.dilation)):
        raise NotImplementedError("Xception's depthwise pass covers 3x3 convolutions with groups = channels, stride 1, padding 1 "
                                  "and no bias")
    dev = conv.weight.device
    return _cached(conv, "dw9", _sig(conv.weight),
                   lambda: (conv.weight.detach().reshape(C, 9).t().float().contiguous(),) + ops.fold_affine(C, None, None, dev))


def _separable(sep, bn, a, relu_in=True, residual=None, relu=False, out=None):
    """SeparableConv2d ``sep`` -> BatchNorm ``bn`` (xception.py:50-60) of max(a, 0) (of ``a`` itself without ``relu_in``): the
    depthwise pass, then the pointwise GEMM with the BatchNorm, ``residual`` and ``relu`` in its epilogue."""
    if a.C != sep.conv1.weight.shape[0]:
        raise ValueError("separable convolution over %d channels got %r" % (sep.conv1.weight.shape[0], a))
    w9, one, zero = _xception_dw(sep.conv1)
    if relu_in:
        h = ops_xception.dwconv3x3_relu_in(a, w9)
    else:
        h = ops.dwconv3x3(a, w9, one, zero, 1, relu6=False)
    return conv_bn_act(sep.pointwise, bn, h, residual=residual, relu=relu, out=out)


def _xception_rep(block):
    """The separable convolutions of ``block.rep`` as (SeparableConv2d, BatchNorm2d, whether a ReLU opens it) triples, and its
    closing pool (or None).  The layout must be the reference's: [ReLU, SeparableConv2d, BatchNorm2d] per repetition, the first ReLU
    absent only in a block built with start_with_relu=False, then MaxPool2d(3, 2, 1) in the blocks with a projection skip."""
    rep = list(block.rep)
    pool = rep.pop() if rep and isinstance(rep[-1], nn.MaxPool2d) else None
    seps, i = [], 0
    while i < len(rep):
        relu = isinstance(rep[i], nn.ReLU)
        if relu:
            i += 1
        elif seps:
            break
        if i + 1 >= len(rep) or not hasattr(rep[i], "pointwise") or not isinstance(rep[i + 1], nn.BatchNorm2d):
            break
        seps.append((rep[i], rep[i + 1], relu))
        i += 2
    ok = bool(seps) and i == len(rep)
    if pool is not None:
        ok = (ok and block.skip is not None and not pool.ceil_mode and pool.dilation in (1, (1, 1))
              and _pool_args(pool) == ((1, 3, 3), (1, 2, 2), (0, 1, 1)))
    else:
        ok = ok and block.skip is None
    if not ok:
        raise NotImplementedError("the engine runs Xception blocks as the reference builds them: [ReLU, SeparableConv2d, BatchNorm2d] "
                                  "repetitions, closed by MaxPool2d(3, 2, 1) with a projection skip or by the identity skip")
    return seps, pool


def _xception_stem_body(model, a):
    """conv1 (3x3, stride 2, valid) -> bn1 -> ReLU -> conv2 (3x3, valid) -> bn2 -> ReLU (xception.py:163-169), each on the slab
    kernel's slice entry as Inception-v3's stem (``_basic_unit``)."""
    a = _basic_unit(_XUnit(model.conv1, model.bn1), a)
    return _basic_unit(_XUnit(model.conv2, model.bn2), a)


def _xception_block_body(block, a, out=None):
    """Block (xception.py:63-112): the separable convolutions of ``rep``, the first on max(x, 0) only when a ReLU opens it, each
    but the last with the ReLU that opens the next in its GEMM epilogue; the last adds the block input (blocks 4-11) in its epilogue, or, in a strided block, is pooled
    (MaxPool2d(3, 2, 1)) and the skip's 1x1 stride-2 convolution + skipbn adds the pooled tensor as its residual
    (``x += skip``): the strided pixels are gathered and the projection runs as a GEMM (``_strided_1x1``)."""
    seps, pool = _xception_rep(block)
    h = a
    for i, (sep, bn, relu_in) in enumerate(seps):
        if i < len(seps) - 1:
            h = _separable(sep, bn, h, relu_in=relu_in, relu=True)
        elif pool is None:
            h = _separable(sep, bn, h, relu_in=relu_in, residual=a, out=out)
        else:
            h = _separable(sep, bn, h, relu_in=relu_in)
    if pool is None:
        return h
    pooled = ops.maxpool3d(h, *_pool_args(pool))
    return _strided_1x1(block.skip, block.skipbn, a, relu=False, residual=pooled, out=out)


def _xception_exit_body(model, a):
    """conv3 -> bn3 -> ReLU -> conv4 -> bn4 (xception.py:183-192): bn4's output, before the head's ReLU."""
    h = _separable(model.conv3, model.bn3, a, relu_in=False, relu=True)
    return _separable(model.conv4, model.bn4, h)


def run_xception_trunk(model, x):
    """Xception's ``features`` on the engine: fp32 NCHW images (or an Act with channel pitch 8) in, bn4's output (an Act) out.  The
    stem, each block and the exit flow are one frozen Function call each."""
    a = x if isinstance(x, Act) else ops.from_ncdhw(x, pitch=8)
    if a.T != 1 or a.H < 7 or a.W < 7:
        # conv1 and conv2 are valid 3x3 convolutions: below 7x7 the reference's conv2 has no output either
        raise ValueError("Xception takes images of at least 7x7, got %r" % (a,))
    a = Fn.frozen(lambda x, o: _xception_stem_body(model, x), a)
    for i in range(1, 13):
        blk = getattr(model, "block%d" % i)
        a = Fn.frozen(lambda x, o: _xception_block_body(blk, x, o), a)
    return Fn.frozen(lambda x, o: _xception_exit_body(model, x), a)


def run_xception_head(model, a):
    """ReLU -> adaptive mean -> view -> last_linear (xception.py:195-202) on bn4's output ``a``: the ReLU and the mean are one pass
    (b2_avgpool_global_affine_ndhwc with a unit affine), so any final map size works."""
    dev = a.data.device
    s, t = _cached(model, "head_unit", (a.ld, dev), lambda: ops.fold_affine(a.ld, None, None, dev))
    return _head_on_pooled(model.last_linear, ops.avgpool_global_affine(a, s, t), a.C)


# ---------------------------------------------------------------------------------------------
# PNASNet-5-Large (pnasnet.py:33-369)
# ---------------------------------------------------------------------------------------------
# Channel layouts.  A tensor of ``seg * n`` logical channels is stored as n segments of ``seg`` channels at a pitch of ``pitch``
# columns each (pad columns zero): a cell output is five combinations side by side, and the 54- and 108-wide combinations of the
# stem cells sit at pitches 56 and 112 so that every segment starts on a 16-byte column.  Filters that read such a tensor get zero
# rows at the pad columns when they are packed (``_scatter``).  Every other tensor is one dense segment.
# A combination is the sum of two operands: its separable branch's closing pointwise GEMM adds the other operand as its residual
# into a dense [M][pitch] matrix, which is then copied into the combination's columns of the cell output by the slice pool kernel as
# a 1x1 window (no GEMM entry writes a column slice and adds a residual; b2_gemm_f16 stores whole rows of pitch ldd).
def _dense_layout(C):
    return (C, ops._round_up(C, 8), 1)


def _scatter(w, layout, width):
    """fp32 [rows][seg * n] -> [rows][width]: logical column c at (c // seg) * pitch + c % seg, zeros elsewhere."""
    seg, pitch, n = layout
    if w.shape[1] != seg * n or pitch * n != width:
        raise ValueError("a filter over %d channels does not read the layout %s of width %d" % (w.shape[1], layout, width))
    out = w.new_zeros((w.shape[0], width))
    for j in range(n):
        out[:, j * pitch:j * pitch + seg] = w[:, j * seg:(j + 1) * seg]
    return out


def _pn_pointwise(conv, bn, layout, width):
    """(fp16 [K][width] filter with zero pad rows, scale, shift) of a 1x1 Conv2d + BatchNorm reading ``layout``."""
    K = conv.weight.shape[0]

    def build():
        w = _scatter(conv.weight.detach().reshape(K, -1).float(), layout, width)
        return (w.half().contiguous(),) + ops.fold_affine(K, None, bn, w.device)
    return _cached(conv, "pn1x1", (_sig(conv.weight) + _sig(*_bn_tensors(bn)), layout, width), build, reads=_bn_tensors(bn))


def _pn_unit_affine(width, dev, owner):
    """The pre-activation GEMM's input affine for a bare ReLU: ones over ``width`` columns, zero past them up to round_up(width, 64)."""
    def build():
        n = ops._round_up(width, 64)
        one = torch.zeros(n, dtype=torch.float32, device=dev)
        one[:width] = 1.0
        return one, torch.zeros(n, dtype=torch.float32, device=dev)
    return _cached(owner, "pn_unit", (width, dev), build)


def _pn_gemm(a, conv, bn, layout, relu=False, residual=None, preact=False):
    """1x1 Conv2d + BatchNorm of ``a`` (stored in ``layout``) on the persistent GEMM: ``preact`` applies ReLU to the A operand
    (ReluConvBn), ``relu`` to the output; ``residual`` (an Act of the output's shape) joins in the epilogue."""
    w, scale, shift = _pn_pointwise(conv, bn, layout, a.ld)
    K = w.shape[0]
    if preact:
        one, zero = _pn_unit_affine(a.ld, a.data.device, conv)
        y = ops.gemm_preact(a.data, w, scale, shift, one, zero, a.M, K, a.ld, relu=relu)
    else:
        y = ops.gemm(a.data, w, scale, shift, a.M, K, a.ld, residual=residual.data if residual is not None else None, relu=relu)
    return Act(y, a.N, 1, a.H, a.W, y.shape[1])


def _pn_depthwise(a, conv, layout, zero_pad=False):
    """SeparableConv2d.depthwise_conv2d of max(a, 0) (ops_pnasnet.dwconv_kxk_relu_in), the taps scattered to ``layout``.  A branch
    built with zero_pad (ZeroPad2d((1, 0, 1, 0)) before the stride-2 convolution, [1:, 1:] after) runs at padding k // 2 - 1 with the
    cropped extent H // 2."""
    k, s = conv.kernel_size[0], conv.stride[0]
    C = conv.weight.shape[0]
    if conv.groups != C or conv.kernel_size != (k, k) or conv.stride != (s, s) or conv.padding != (k // 2, k // 2) or conv.bias is not None:
        raise NotImplementedError("PNASNet's depthwise pass covers square k x k depthwise convolutions with padding k // 2")
    wk = _cached(conv, "pn_dw", (_sig(conv.weight), layout, a.C),
                 lambda: _scatter(conv.weight.detach().reshape(C, k * k).t().float(), layout, a.C).contiguous())
    if zero_pad:
        pad, Ho, Wo = k // 2 - 1, a.H // 2, a.W // 2
    else:
        pad = k // 2
        Ho, Wo = (a.H + 2 * pad - k) // s + 1, (a.W + 2 * pad - k) // s + 1
    return ops_pnasnet.dwconv_kxk_relu_in(a, wk, k, s, pad, Ho, Wo)


def _pn_branch(br, a, layout, residual=None):
    """BranchSeparables ``br`` (pnasnet.py:67-97) of ``a``: depthwise (ReLU on load) -> pointwise + bn_sep_1 + ReLU -> depthwise ->
    pointwise + bn_sep_2 (+ ``residual``).  Returns a dense Act of the output width."""
    sep1, sep2 = br.separable_1, br.separable_2
    h = _pn_depthwise(a, sep1.depthwise_conv2d, layout, zero_pad=br.zero_pad is not None)
    h = _pn_gemm(h, sep1.pointwise_conv2d, br.bn_sep_1, layout, relu=True)
    mid = _dense_layout(sep1.pointwise_conv2d.weight.shape[0])
    h = _pn_depthwise(h, sep2.depthwise_conv2d, mid)
    return _pn_gemm(h, sep2.pointwise_conv2d, br.bn_sep_2, mid, residual=residual)


def _pn_relu_conv_bn(u, a, layout):
    """ReluConvBn (pnasnet.py:100-114): the pre-activation GEMM with a unit affine; at stride 2 the strided pixels are gathered
    first (b2_shortcut_a_ndhwc)."""
    s = u.conv.stride[0]
    if u.conv.kernel_size != (1, 1) or u.conv.stride != (s, s) or s not in (1, 2):
        raise NotImplementedError("ReluConvBn runs 1x1 convolutions at stride 1 or 2")
    if s == 2:
        a = ops.shortcut_a(a, 2, a.ld)
    return _pn_gemm(a, u.conv, u.bn, layout, preact=True)


def _pn_factorized_reduction(u, a, layout):
    """FactorizedReduction (pnasnet.py:117-146): ReLU and the gathers x[2i, 2j] / x[2i + 1, 2j + 1] (ops_pnasnet.gather_offset), then
    one two-operand GEMM whose filters hold path_1's rows in the first half and path_2's in the second (zeros elsewhere), with
    final_path_bn: the concatenation of the two half-width convolutions at any half width (54 and 108 do not start on a 16-byte
    column)."""
    c1, c2 = u.path_1.conv, u.path_2.conv
    h, K = c1.weight.shape[0], 2 * c1.weight.shape[0]

    def build():
        w1 = _scatter(c1.weight.detach().reshape(h, -1).float(), layout, a.ld)
        w2 = _scatter(c2.weight.detach().reshape(h, -1).float(), layout, a.ld)
        b1, b2 = w1.new_zeros((K, a.ld)), w1.new_zeros((K, a.ld))
        b1[:h], b2[h:] = w1, w2
        return (b1.half().contiguous(), b2.half().contiguous()) + ops.fold_affine(K, None, u.final_path_bn, w1.device)
    b1, b2, scale, shift = _cached(u, "pn_fr", (_sig(c1.weight, c2.weight) + _sig(*_bn_tensors(u.final_path_bn)), layout, a.ld),
                                   build, reads=_bn_tensors(u.final_path_bn))
    g1 = ops_pnasnet.gather_offset(a, 2, 0, relu=True)
    g2 = ops_pnasnet.gather_offset(a, 2, 1, relu=True)
    y = ops.gemm(g1.data, b1, scale, shift, g1.M, K, a.ld, second=(g2.data, b2, a.ld))
    return Act(y, g1.N, 1, g1.H, g1.W, y.shape[1])


def _pn_pool(m, a):
    """MaxPool (pnasnet.py:33-46) on the slice pool: the zero-pad form is the ceil-extent 3x3 pool without padding."""
    k, s, p = m.pool.kernel_size, m.pool.stride, m.pool.padding
    if m.zero_pad is not None:
        return ops.pool_slice(a, k, s, 0, False)
    return ops.pool_slice(a, k, s, p, False)


def _pn_cell_body(cell, left, left_layout, right, right_layout):
    """One cell (pnasnet.py:149-288): (output Act, its layout).  ``left`` / ``right``: the cell's two inputs (CellStem0: conv_0's
    output and None)."""
    from .models.pnasnet import CellStem0
    stem0 = isinstance(cell, CellStem0)
    if stem0:
        x_left, l_lay = left, left_layout
        x_right = _pn_relu_conv_bn(cell.conv_1x1, left, left_layout)
    else:
        if cell.match_prev_layer_dimensions:
            x_left = _pn_factorized_reduction(cell.conv_prev_1x1, left, left_layout)
        else:
            x_left = _pn_relu_conv_bn(cell.conv_prev_1x1, left, left_layout)
        l_lay = _dense_layout(cell.comb_iter_0_left.bn_sep_2.num_features)
        x_right = _pn_relu_conv_bn(cell.conv_1x1, right, right_layout)
    r_lay = _dense_layout(cell.conv_1x1.bn.num_features)
    Cb = cell.comb_iter_1_left.bn_sep_2.num_features
    Cp = ops._round_up(Cb, 8)
    lay = (Cb, Cp, 1)
    c0 = _pn_pool(cell.comb_iter_0_right.max_pool if stem0 else cell.comb_iter_0_right, x_left)
    if stem0:
        c0 = _pn_gemm(c0, cell.comb_iter_0_right.conv, cell.comb_iter_0_right.bn, l_lay)
    c0 = _pn_branch(cell.comb_iter_0_left, x_left, l_lay, residual=c0)
    out = torch.empty((c0.M, 5 * Cp), dtype=torch.float16, device=c0.data.device)

    def put(j, c):
        ops.pool_slice(Act(c.data, c.N, 1, c.H, c.W, c.ld), 1, 1, 0, False, y=out[:, j * Cp:(j + 1) * Cp])

    put(0, c0)
    put(1, _pn_branch(cell.comb_iter_1_left, x_right, r_lay, residual=_pn_pool(cell.comb_iter_1_right, x_right)))
    c2 = _pn_branch(cell.comb_iter_2_right, x_right, r_lay)
    put(2, _pn_branch(cell.comb_iter_2_left, x_right, r_lay, residual=c2))
    slot2 = Act(out[:, 2 * Cp:3 * Cp], c0.N, 1, c0.H, c0.W, Cp)
    put(3, _pn_branch(cell.comb_iter_3_left, slot2, lay, residual=_pn_pool(cell.comb_iter_3_right, x_right)))
    r4 = x_right if cell.comb_iter_4_right is None else _pn_relu_conv_bn(cell.comb_iter_4_right, x_right, r_lay)
    put(4, _pn_branch(cell.comb_iter_4_left, x_left, l_lay, residual=r4))
    return Act(out, c0.N, 1, c0.H, c0.W, 5 * Cp), (Cb, Cp, 5)


def pnasnet_stages(model, a):
    """conv_0, cell_stem_0, cell_stem_1, cell_0 .. cell_11 of ``a`` (an NHWC Act with channel pitch 8): a list of (name, Act,
    layout).  conv_0 (3x3, stride 2, valid) + BN runs on the slab kernel's slice entry without a ReLU."""
    from .models.pnasnet import CELLS
    pc = packed_conv(model.conv_0.conv, model.conv_0.bn, a.ld)
    Ho, Wo = (a.H - 3) // 2 + 1, (a.W - 3) // 2 + 1
    y = torch.empty((a.N * Ho * Wo, pc.K), dtype=torch.float16, device=a.data.device)
    x0 = ops.conv_slice(a, pc, y, relu=False)
    stages = [("conv_0", x0, _dense_layout(96))]
    s0 = _pn_cell_body(model.cell_stem_0, x0, stages[0][2], None, None)
    stages.append(("cell_stem_0",) + s0)
    for name, *_ in CELLS:
        (_, pa, pl), (_, ca, cl) = stages[-2], stages[-1]
        stages.append((name,) + _pn_cell_body(getattr(model, name), pa, pl, ca, cl))
    return stages


def run_pnasnet_trunk(model, x):
    """PNASNet-5-Large's ``features`` on the engine: fp32 NCHW 331x331 images (or an Act with channel pitch 8) in, cell_11's output
    (an Act) out, in one frozen Function call."""
    a = x if isinstance(x, Act) else ops.from_ncdhw(x, pitch=8)
    if a.T != 1 or (a.H, a.W) != (331, 331):
        # the reference's head is a fixed AvgPool2d(11): only 331x331 inputs reach it with an 11x11 map
        raise ValueError("PNASNet-5-Large takes 331x331 images, got %r" % (a,))
    return Fn.frozen(lambda x, o: pnasnet_stages(model, x)[-1][1], a)


def run_pnasnet_head(model, a):
    """ReLU -> AvgPool2d(11) -> view -> dropout (identity in eval) -> last_linear (pnasnet.py:358-364) on cell_11's output: the ReLU
    and the mean in one pass (b2_avgpool_global_affine_ndhwc with a unit affine)."""
    if (a.H, a.W) != (11, 11):
        raise ValueError("PNASNet-5-Large's head pools an 11x11 map, got %r" % (a,))
    dev = a.data.device
    s, t = _cached(model, "head_unit", (a.ld, dev), lambda: ops.fold_affine(a.ld, None, None, dev))
    return _head_on_pooled(model.last_linear, ops.avgpool_global_affine(a, s, t), a.C)


# ---------------------------------------------------------------------------------------------
# stem / trunk / head
# ---------------------------------------------------------------------------------------------
def _pool_args(mp):
    if isinstance(mp, nn.MaxPool2d):
        k, s, p = mp.kernel_size, mp.stride, mp.padding
        two = lambda v: (v, v) if isinstance(v, int) else tuple(v)
        k, s, p = two(k), two(s), two(p)
        return (1, k[0], k[1]), (1, s[0], s[1]), (0, p[0], p[1])
    return _triple(mp.kernel_size), _triple(mp.stride), _triple(mp.padding)


def run_stem(model, x, simt=False, out=None):
    """conv1 -> bn1 -> relu -> maxpool (torchvision_models.py:449-452)."""
    a = x if isinstance(x, Act) else ops.from_ncdhw(x)
    return Fn.frozen(lambda x, o: _stem_body(model, x, simt, o), a, out)


def _stem_body(model, a, simt=False, out=None):
    """conv1 -> bn1 -> ReLU -> maxpool.  When the stem runs on the Toeplitz kernel and the pool is the usual 3-wide / stride-2 /
    pad-1 window along W, that direction of the pool is taken in the convolution's epilogue (max-pooling is separable, so this is
    exact): the stem writes half of its output and the remaining (kt, kh, 1) pool reads half as much."""
    k, s, p = _pool_args(model.maxpool)
    conv = model.conv1
    plain = isinstance(conv, (nn.Conv3d, nn.Conv2d))
    if (plain and not simt and a.ld == 4 and _is_stem_shape(conv) and (k[2], s[2], p[2]) == (3, 2, 1)
            and ops._out_dim(a.W, 7, 2, 3) <= 120 and os.environ.get("B2_STEM_POOLW", "1") != "0"):
        a = conv_bn_act(conv, model.bn1, a, relu=True, pool_w=True)
        return ops.maxpool3d(a, (k[0], k[1], 1), (s[0], s[1], 1), (p[0], p[1], 0), out=out)
    a = conv_bn_act(conv, model.bn1, a, relu=True, simt=simt)
    return ops.maxpool3d(a, k, s, p, out=out)


# ---------------------------------------------------------------------------------------------
# trunk schedule: breadth-first (default) or, on request, depth-first in clip chunks
# ---------------------------------------------------------------------------------------------
# Clips are independent in every layer (eval-mode BN, per-clip attention), so the trunk may be walked in any clip order.  The
# breadth-first walk (one launch per layer over the whole batch) is the default.  ``set_dfs("units:clips,...")`` walks consecutive
# segments of trunk units DEPTH-first instead -- a chunk of a few clips goes through stem, pool and a run of residual blocks before
# the next chunk starts, so that a chunk's intermediates are write-then-read inside the 50 MB L2 (the allocator hands the next
# chunk the same addresses) and only a segment's first input and last output cross HBM; the last kernel of a chunk writes straight
# into its row range of the whole-batch tensor (``out=``).  Every extra launch of these persistent kernels costs pipeline fill,
# drain and tile quantisation, so breadth-first is the default; tools/dfs_sweep.py times the alternatives.  The schedule stays as
# an opt-in (same kernels per output element: results equal the breadth-first walk up to kernel-dispatch boundaries).
_DFS_SPEC = os.environ.get("B2_DFS", "off")


def set_dfs(spec):
    """Trunk schedule: ``"off"`` (breadth-first, the default) or an explicit
    ``"units:clips,units:clips"`` list -- consecutive segments of trunk units (unit 0 = stem + pool, then the residual blocks in
    order), each walked depth-first in chunks of ``clips``; units not covered run breadth-first."""
    global _DFS_SPEC
    _DFS_SPEC = str(spec)


def _trunk_units(model):
    units = [("stem", model)]
    for name in ("layer1", "layer2", "layer3", "layer4"):
        units += [("block", blk) for blk in getattr(model, name)]
    return units


def dfs_plan(model=None, N=None, geom=None):
    """[(units, clips per chunk)] for ``run_trunk`` (empty = breadth-first)."""
    spec = _DFS_SPEC.strip().lower()
    if spec in ("0", "off", "none", "", "auto"):       # "auto" = the default rule: never chunk
        return []
    return [tuple(int(v) for v in part.split(":")) for part in spec.split(",")]


def _slice_clips(x, n0, n1):
    if isinstance(x, Act):
        r = x.positions
        return Act(x.data[n0 * r:n1 * r], n1 - n0, x.T, x.H, x.W, x.C)
    return x[n0:n1]


def _chained_pairs(units, simt):
    """Indices j of the units whose closing kernel computes unit j + 1's conv1 (``_chains``)."""
    return {j for j in range(len(units) - 1)
            if units[j][0] == units[j + 1][0] == "block" and _chains(units[j][1], units[j + 1][1], simt)}


def _run_units(units, a, simt, out=None):
    chained = _chained_pairs(units, simt)
    h1 = None
    for j, (kind, m) in enumerate(units):
        o = out if j == len(units) - 1 else None
        if kind == "stem":
            a = run_stem(m, a, simt=simt, out=o)
        elif j in chained:
            a, h1 = run_block(m, a, simt=simt, out=o, h1=h1, nxt=units[j + 1][1])
        elif h1 is not None:
            a, h1 = run_block(m, a, simt=simt, out=o, h1=h1), None
        else:
            a = run_block(m, a, simt=simt, out=o)
    return a


def _run_segment(units, x, N, clips, simt):
    """Depth-first walk of ``units`` in chunks of ``clips``; the last kernel of each chunk writes straight into its row range of the
    segment's whole-batch output (allocated once the first chunk has shown the output geometry)."""
    buf = None
    for n0 in range(0, N, clips):
        n1 = min(N, n0 + clips)
        o = buf.data[n0 * buf.positions:n1 * buf.positions] if buf is not None else None
        y = _run_units(units, _slice_clips(x, n0, n1), simt, out=o)
        if buf is None:
            buf = Act(torch.empty((N * y.positions, y.ld), dtype=torch.float16, device=y.data.device), N, y.T, y.H, y.W, y.C)
            o = buf.data[:y.M]
        if y.data.data_ptr() != o.data_ptr():      # first chunk, or a unit whose last kernel takes no ``out``
            o.copy_(y.data)
    return buf


def run_trunk(model, x, simt=False):
    units = _trunk_units(model)
    N = x.N if isinstance(x, Act) else x.shape[0]
    plan = [] if simt else dfs_plan()
    a, ui = x, 0
    for n_units, clips in plan:
        seg = units[ui:ui + n_units]
        if not seg:
            break
        ui += len(seg)
        a = _run_segment(seg, a, N, clips, simt) if 0 < clips < N else _run_units(seg, a, simt)
    return _run_units(units[ui:], a, simt) if ui < len(units) else a


# ---------------------------------------------------------------------------------------------
# fine-tuning: backward through plain BasicBlock / Bottleneck blocks with eval-mode ("frozen") BatchNorm
# ---------------------------------------------------------------------------------------------
# Notation for one conv -> BN -> (+res) -> ReLU: s = gamma / sqrt(var + eps), g = gradient at the BN output (already through
# the ReLU mask), G = sum_m g (x) x_tap the UNSCALED weight gradient (b2_conv_wgrad).  Then dW = s G, dbeta = sum_m g,
# dgamma = (<W, G> - mean dbeta) / sqrt(var + eps) (sum g conv(x) = <W, G>: no pre-BN tensor is kept), and the input gradient
# is the convolution of g with the transposed, flipped, s-folded filter on the forward kernels.  Gradients cross kernels as
# fp16 times a power-of-two loss scale chosen on the device where the gradient enters the trunk (ops.loss_scale_); every fp32
# result divides it out.
class TrainAct(Act):
    """Act produced by the fine-tuned part of the trunk: ``data`` carries the autograd graph and ``loss_scale`` is the
    device pair [scale, 1/scale] its backward fills in."""
    __slots__ = ("loss_scale",)


def _check_trainable_2d(block, grouped=False):
    """torchvision BasicBlock / Bottleneck (the 2-D ResNets) and ResNeXt-101's bottleneck: Conv2d 1x1 / 3x3 with padding k // 2,
    stride 1 or 2, no bias or dilation, no groups except (``grouped``, ResNeXt-101) a 3x3 inside the group-aware kernels'
    contract (C == K, 4 / 8 / 16 / 32 channels per group), BatchNorm2d, identity or (Conv2d 1x1, BatchNorm2d) shortcut."""
    convs = [(block.conv1, block.bn1), (block.conv2, block.bn2)] + ([(block.conv3, block.bn3)] if hasattr(block, "conv3") else [])
    ds = block.downsample
    ok = True
    if isinstance(ds, nn.Sequential):
        ok = len(ds) == 2 and type(ds[0]) is nn.Conv2d and tuple(ds[0].weight.shape[2:]) == (1, 1)
        convs.append((ds[0], ds[1]) if ok else (None, None))
    elif ds is not None:
        ok = False
    for conv, bn in convs if ok else ():
        k = tuple(conv.weight.shape[2:])
        ok = ok and type(conv) is nn.Conv2d and conv.bias is None and all(d == 1 for d in conv.dilation)
        ok = ok and (conv.groups == 1 or (grouped and k == (3, 3) and grouped_route(conv)))   # the group-aware kernels' contract
        ok = ok and k in ((1, 1), (3, 3)) and tuple(conv.padding) == (k[0] // 2,) * 2
        ok = ok and len(set(conv.stride)) == 1 and conv.stride[0] in (1, 2)
        ok = ok and isinstance(bn, nn.BatchNorm2d) and bn.affine and bn.running_var is not None
    if not ok:
        raise NotImplementedError("fine-tuning backward covers torchvision's BasicBlock / Bottleneck with 1x1 / 3x3 Conv2d filters "
                                  "and an identity or 1x1 projection shortcut; got a %s that is not of that form" % type(block).__name__)


def check_trainable_block(block):
    """Raise NotImplementedError unless ``block`` is a plain 3-D ResNet BasicBlock / Bottleneck or a torchvision (2-D)
    BasicBlock / Bottleneck the backward covers."""
    import torchvision.models.resnet as tvresnet
    from .models.resnet3d import BasicBlock, Bottleneck, ShortcutA
    from .models.resnext import ResNeXt101Bottleneck
    if type(block) in (tvresnet.BasicBlock, tvresnet.Bottleneck, ResNeXt101Bottleneck):
        return _check_trainable_2d(block, grouped=type(block) is ResNeXt101Bottleneck)
    name = type(block).__name__
    ok = type(block) in (BasicBlock, Bottleneck) and getattr(block, "nonlocalblock", None) is None
    convs = [(block.conv1, block.bn1), (block.conv2, block.bn2)] + ([(block.conv3, block.bn3)] if ok and hasattr(block, "conv3") else [])
    ds = getattr(block, "downsample", None)
    if isinstance(ds, nn.Sequential):
        ok = ok and len(ds) == 2 and _plain_1x1(ds[0])
        convs.append((ds[0], ds[1]) if ok else (None, None))
    elif ds is not None and not isinstance(ds, ShortcutA):
        ok = False
    for conv, bn in convs if ok else ():
        k = tuple(conv.weight.shape[2:])
        ok = ok and type(conv) is nn.Conv3d and conv.groups == 1 and conv.bias is None and all(d == 1 for d in conv.dilation)
        ok = ok and k in ((1, 1, 1), (3, 3, 3)) and tuple(conv.padding) == (k[0] // 2,) * 3
        ok = ok and len(set(conv.stride)) == 1 and conv.stride[0] in (1, 2)
        ok = ok and isinstance(bn, nn.BatchNorm3d) and bn.affine and bn.running_var is not None
    if not ok:
        raise NotImplementedError("fine-tuning backward covers the plain BasicBlock / Bottleneck of the 3-D ResNets (shortcut A, B or "
                                  "identity); got a %s" % name)


def _train_units(block):
    """(conv, bn) pairs of a block in parameter order: conv1, conv2[, conv3][, downsample projection]."""
    units = [(block.conv1, block.bn1), (block.conv2, block.bn2)]
    if hasattr(block, "conv3"):
        units.append((block.conv3, block.bn3))
    if isinstance(block.downsample, nn.Sequential):
        units.append((block.downsample[0], block.downsample[1]))
    return units


def train_params(block):
    return [t for conv, bn in _train_units(block) for t in (conv.weight, bn.weight, bn.bias)]


def _bn_scale(bn):
    return (bn.weight.detach().float() * torch.rsqrt(bn.running_var.float() + bn.eps)).contiguous()


def _dgrad_1x1(conv, s):
    """B operand [Cin][Cout] (fp16) of the input gradient g . (s W) of a 1x1x1 convolution."""
    w = conv.weight.detach().reshape(conv.weight.shape[0], -1).float() * s[:, None]
    return w.t().contiguous().to(torch.float16)


def _kernel_thw(conv):
    """(kt, kh, kw) of a Conv3d / Conv2d filter (a 2-D filter is (1, kh, kw))."""
    k = tuple(conv.weight.shape[2:])
    return (1,) + k if len(k) == 2 else k


def _dgrad_3x3(conv, s, g_pitch):
    """The input gradient of a 3x3x3 (or 2-D 3x3) convolution as a stride-1 convolution with the transposed, flipped,
    s-folded filter and padding (1, 1, 1) (or (0, 1, 1))."""
    w = conv.weight.detach().float()
    w = w * s.view((-1,) + (1,) * (w.dim() - 1))
    if w.dim() == 4:                                   # Conv2d: a (1, 3, 3) filter at T = 1
        w = w.unsqueeze(2)
    pad = tuple(k // 2 for k in w.shape[2:])
    return ops.PackedConv(w.flip(2, 3, 4).transpose(0, 1).contiguous(), None, None, (1, 1, 1), pad, in_pitch=g_pitch)


def _inplane_stride(conv):
    """The stride b2_zero_insert_ndhwc applies.  It takes one stride for all three axes: the 3-D blocks have cubic strides,
    and a 2-D convolution runs at T = 1, where inserting zeros along T is the identity."""
    return _conv_geometry(conv)[0][1]


def _gemm_dgrad(g, wt, residual=None, second=None, mask=None):
    """g . wt^T (+ residual), zeroed where ``mask`` (an Act of the result's shape) is not positive."""
    C = wt.shape[0]
    one = torch.ones(C, dtype=torch.float32, device=g.data.device)
    zero = torch.zeros(C, dtype=torch.float32, device=g.data.device)
    y = ops.gemm(g.data, wt, one, zero, g.M, C, g.C, residual=residual.data if residual is not None else None, second=second,
                 mask=mask.data if mask is not None else None)
    return Act(y, g.N, g.T, g.H, g.W, C)


def _dgrad_grouped(conv, s):
    """The input gradient of a grouped 2-D 3x3 convolution (C == K) as a stride-1 grouped convolution with the same groups: its
    filter transposed within each group, flipped and s-folded, on the group-aware kernel."""
    K, cg = conv.weight.shape[:2]
    G = conv.groups
    w = (conv.weight.detach().float() * s.view(-1, 1, 1, 1)).view(G, cg, cg, 3, 3).transpose(1, 2).flip(3, 4).reshape(K, cg, 3, 3)
    return ops.PackedGroupedConv(w.contiguous(), G, None, None, (1, 1, 1), (0, 1, 1))


def _conv_dgrad_masked(conv, s, g, x):
    """Gradient at the input ``x`` of a 3x3x3 (or 2-D 3x3, grouped or not) convolution for the gradient ``g`` at its (BN-scaled)
    output, times the ReLU mask [x > 0]."""
    stride = _inplane_stride(conv)
    z = g if stride == 1 else ops.zero_insert(g, x.T, x.H, x.W, stride)
    if conv.groups > 1:
        return ops_grouped.conv_grouped_dgrad(z, _dgrad_grouped(conv, s), mask=x)
    return ops.conv(z, _dgrad_3x3(conv, s, z.ld), mask=x)


def _conv_dgrad(conv, s, g, x):
    """Gradient at the input ``x`` of a 3x3x3 convolution for the gradient ``g`` at its (BN-scaled) output, before any residual."""
    stride = _inplane_stride(conv)
    z = g if stride == 1 else ops.zero_insert(g, x.T, x.H, x.W, stride)
    return z, _dgrad_3x3(conv, s, z.ld)


def _param_grads(conv, bn, g, x, ls, needs):
    """(dW, dgamma, dbeta) of conv -> eval-mode bn for the gradient ``g`` at the BN output; None where not needed."""
    need_w, need_g, need_b = needs
    dw = wdot = dbeta = dgamma = None
    inv = ls[1:]
    if need_w or need_g:
        stride, pad = _conv_geometry(conv)
        if conv.groups > 1:
            dw, wdot = ops_grouped.conv_wgrad_grouped(g, x, conv.groups, stride[1], weight=conv.weight if need_g else None, scale=_bn_scale(bn),
                                              inv_loss_scale=inv)
        else:
            dw, wdot = ops.conv_wgrad(g, x, _kernel_thw(conv), stride, pad, weight=conv.weight if need_g else None,
                                      scale=_bn_scale(bn), inv_loss_scale=inv)
        dw = dw.view(conv.weight.shape)
    if need_b or need_g:
        dbeta = ops.colsum(g, inv)
    if need_g:
        dgamma = (wdot - bn.running_mean.float() * dbeta) * torch.rsqrt(bn.running_var.float() + bn.eps)
    return [dw if need_w else None, dgamma, dbeta if need_b else None]


def _shortcut_grad(block, g, x):
    """Gradient the shortcut sends to the block input (``g`` itself for the identity)."""
    ds = block.downsample
    if ds is None:
        return g
    if isinstance(ds, nn.Sequential):
        stride = _inplane_stride(ds[0])
        pg = _gemm_dgrad(g, _dgrad_1x1(ds[0], _bn_scale(ds[1])))
        return pg if stride == 1 else ops.zero_insert(pg, x.T, x.H, x.W, stride, ld=x.ld)
    return ops.zero_insert(g, x.T, x.H, x.W, ds.stride, channels=x.C, ld=x.ld)       # type A: subsample + zero channels


def block_backward(block, x, hs, gy, ls, need_x, needs):
    """Backward of one fine-tuned block.  ``gy``: loss-scaled fp16 gradient at the block output, already multiplied by the
    block's closing ReLU mask; ``hs``: the post-ReLU intermediates of the forward; ``needs``: needs_input_grad of the
    parameters in ``train_params`` order.  Returns (gradient at the block input times [x > 0], or None; parameter grads)."""
    units = _train_units(block)
    grads = [None] * (3 * len(units))
    if hasattr(block, "conv3"):
        h1, h2 = hs
        grads[6:9] = _param_grads(block.conv3, block.bn3, gy, h2, ls, needs[6:9])
        g2 = _gemm_dgrad(gy, _dgrad_1x1(block.conv3, _bn_scale(block.bn3)), mask=h2)
        grads[3:6] = _param_grads(block.conv2, block.bn2, g2, h1, ls, needs[3:6])
        g1 = _conv_dgrad_masked(block.conv2, _bn_scale(block.bn2), g2, h1)
    else:
        (h1,) = hs
        grads[3:6] = _param_grads(block.conv2, block.bn2, gy, h1, ls, needs[3:6])
        g1 = ops.conv(gy, _dgrad_3x3(block.conv2, _bn_scale(block.bn2), gy.ld), mask=h1)
    grads[0:3] = _param_grads(block.conv1, block.bn1, g1, x, ls, needs[0:3])
    if isinstance(block.downsample, nn.Sequential):
        ds = block.downsample
        grads[-3:] = _param_grads(ds[0], ds[1], gy, x, ls, needs[-3:])
    if not need_x:
        return None, grads
    s1 = _bn_scale(block.bn1)
    ds = block.downsample
    if hasattr(block, "conv3"):
        w1 = _dgrad_1x1(block.conv1, s1)
        if isinstance(ds, nn.Sequential) and _inplane_stride(ds[0]) == 1:     # both 1x1 products in one two-operand GEMM
            dx = _gemm_dgrad(g1, w1, second=(gy.data, _dgrad_1x1(ds[0], _bn_scale(ds[1])), gy.C), mask=x)
        else:
            dx = _gemm_dgrad(g1, w1, residual=_shortcut_grad(block, gy, x), mask=x)
    else:
        z, pc = _conv_dgrad(block.conv1, s1, g1, x)
        dx = ops.conv(z, pc, residual=_shortcut_grad(block, gy, x), mask=x)
    return dx, grads


def run_trunk_finetune(model, x, k):
    """Stem and layer1..layer{k-1} frozen (the forward path), layer{k}..layer4 through the differentiable block Functions.
    The depth-first schedule is not used."""
    units = _trunk_units(model)
    n_frozen = 1 + sum(len(getattr(model, "layer%d" % i)) for i in range(1, k))
    a = _run_units(units[:n_frozen], x, simt=False)
    ls = torch.ones(2, dtype=torch.float32, device=a.data.device)
    for _, blk in units[n_frozen:]:
        a = Fn.BlockTrainFunction.run(blk, a, ls)
    out = TrainAct(a.data, a.N, a.T, a.H, a.W, a.C)
    out.loss_scale = ls
    return out


def run_head(model, a, head):
    """avgpool -> view(B,-1) -> last_linear (torchvision_models.py:460-464).  Returns fp32 [N][classes]."""
    if isinstance(a, TrainAct):
        # fine-tuning: fp32 pooled features, so that the head's input gradient reaches the pool backward unrounded
        pooled = Fn.FineTunePoolFunction.apply(a.data, (a.N, a.T, a.H, a.W, a.C), a.loss_scale)
        return Fn.linear(pooled, head.weight, head.bias) if isinstance(head, nn.Linear) else head(pooled)
    return _head_on_pooled(head, ops.avgpool_global(a), a.C)


def _head_on_pooled(head, pooled, C):
    """``head`` on the fp16 pooled features [N][ld] (``C`` of them used) -> fp32 [N][classes]."""
    if isinstance(head, nn.Linear) and torch.is_grad_enabled() and any(p.requires_grad for p in head.parameters()):
        # trainable head on frozen engine features: differentiable GEMM (functions.LinearFunction), same kernel
        return Fn.linear(pooled[:, :head.in_features], head.weight, head.bias)
    if isinstance(head, nn.Linear):
        pl = _cached(head, "pl", _sig(head.weight, head.bias), lambda: ops.PackedLinear(head.weight, head.bias))
        return ops.linear(pooled, pl, out_f32=True)
    # user-swapped head (Identity, Dropout, custom module): hand it the pooled features like the reference does
    return head(pooled[:, :C].float())
