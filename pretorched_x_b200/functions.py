"""torch.autograd.Function wrappers around the C-ABI call sequences (SURVEY.md section 8b-ii; BASELINE.json north_star:
"exposed to Python through a thin C-ABI/ctypes shim wrapped as torch.autograd.Function").

Two kinds:

* **Frozen block bodies** -- ``StemFunction``, ``BottleneckFunction`` (resnet3D.py:125-143), ``BasicBlockFunction``
  (:91-106), ``SpatioTemporalConvFunction`` (r2plus1d.py:85-88), ``NonLocalFunction`` (nonlocalnet.py:143-243),
  ``GBlockFunction`` (BigGAN-deep GBlock).  ``forward`` is the ctypes launch sequence of ``engine.py`` /
  ``biggan_engine.py`` on fp16 NDHWC matrices; every output is marked non-differentiable, so the modules can sit inside
  an autograd graph as a frozen feature extractor (the way the reference's zoo models are used with a replaced
  ``last_linear``, README.md:520-547).  These frozen bodies have no backward: asking for one raises.
* **Fine-tuned residual blocks** -- ``BlockTrainFunction`` / ``FineTunePoolFunction``, used instead of the frozen bodies for
  ``layer{k}..layer4`` after ``ResNet3D.fine_tune(k)`` (engine.block_backward).
* **Dense heads with a real backward** -- ``LinearFunction`` (``last_linear`` / ``fc``: resnet3D.py:162,
  torchvision_models.py:463-464) and, built from it, the TRN relation MLP (trn.py:39-49).  ``forward`` and both
  gradient products run on the same wgmma GEMM (``b2_gemm_f16``: fp16 operands, fp32 accumulation and output), so a
  head can be trained on engine features without leaving the library.

Tensors cross a Function boundary as the raw ``[N*T*H*W][ld]`` fp16 matrix of an ``ops.Act`` plus its geometry tuple.
``out`` (optional, last argument of the block bodies): a preallocated ``[rows][ld]`` fp16 row range the body's LAST kernel writes
its result into -- how the depth-first trunk schedule (``engine.run_trunk``) assembles a full-batch tensor chunk by chunk.
"""
import torch

from . import ops
from .ops import Act


def _geom(a):
    return (a.N, a.T, a.H, a.W, a.C)


class _FrozenFunction(torch.autograd.Function):
    """Base: outputs are constants to autograd."""

    @staticmethod
    def backward(ctx, *grads):      # pragma: no cover - unreachable: every output is marked non-differentiable
        raise RuntimeError("pretorched_x_b200 is a forward-pass engine: the convolutional trunk has no backward "
                           "(frozen-backbone semantics); only LinearFunction / the relation MLP are differentiable")

    @classmethod
    def run(cls, module, a, *extra):
        """Act in -> Act out through ``cls.apply``."""
        data, geom = cls.apply(a.data, _geom(a), module, *extra)
        return Act(data, *geom)

    @classmethod
    def _finish(cls, ctx, out):
        ctx.mark_non_differentiable(out.data)
        return out.data, _geom(out)


class StemFunction(_FrozenFunction):
    """conv1 -> bn1 -> relu -> maxpool (torchvision_models.py:449-452).  ``x`` is the NDHWC4 / NDHWC input matrix."""

    @staticmethod
    def forward(ctx, x2d, geom, model, simt=False, out=None):
        from . import engine
        return StemFunction._finish(ctx, engine._stem_body(model, Act(x2d, *geom), simt, out))


class BottleneckFunction(_FrozenFunction):
    """``h1``: the block's conv1 output, computed by the previous block's closing kernel.  ``nxt``: the next block, whose conv1
    the closing kernel computes too (engine._chains); then the result is (block output, next block's h1), as in GBlockFunction."""

    @staticmethod
    def forward(ctx, x2d, geom, block, simt=False, out=None, h1=None, nxt=None):
        from . import engine
        out = engine._bottleneck_body(block, Act(x2d, *geom), simt, out, h1=h1, nxt=nxt)
        if isinstance(out, tuple):
            ctx.mark_non_differentiable(out[0].data, out[1].data)
            return out[0].data, _geom(out[0]), out[1].data, _geom(out[1])
        ctx.mark_non_differentiable(out.data)
        return out.data, _geom(out), None, None

    @classmethod
    def run(cls, block, a, simt=False, out=None, h1=None, nxt=None):
        y2d, geom, h2d, hgeom = cls.apply(a.data, _geom(a), block, simt, out, h1, nxt)
        return (Act(y2d, *geom), Act(h2d, *hgeom)) if nxt is not None else Act(y2d, *geom)


class BasicBlockFunction(_FrozenFunction):
    @staticmethod
    def forward(ctx, x2d, geom, block, simt=False, out=None):
        from . import engine
        return BasicBlockFunction._finish(ctx, engine._basic_body(block, Act(x2d, *geom), simt, out))


class PreActBlockFunction(_FrozenFunction):
    """Pre-activation residual blocks (pre_act_resnet3D.py:27-96)."""

    @staticmethod
    def forward(ctx, x2d, geom, block, simt=False, out=None):
        from . import engine
        return PreActBlockFunction._finish(ctx, engine._preact_body(block, Act(x2d, *geom), simt, out))


class SpatioTemporalConvFunction(_FrozenFunction):
    """(1,k,k) conv -> BN -> ReLU -> (k,1,1) conv [-> outer BN -> +residual -> ReLU] (r2plus1d.py:85-88)."""

    @staticmethod
    def forward(ctx, x2d, geom, conv, bn=None, residual=None, relu=False, simt=False, out=None):
        from . import engine
        return SpatioTemporalConvFunction._finish(ctx, engine._st_conv_body(conv, bn, Act(x2d, *geom), residual, relu, simt, out))


class NonLocalFunction(_FrozenFunction):
    @staticmethod
    def forward(ctx, x2d, geom, nl, simt=False, out=None):
        from . import engine
        return NonLocalFunction._finish(ctx, engine._nonlocal_body(nl, Act(x2d, *geom), simt, out))


class ConvBNReLU6Function(_FrozenFunction):
    """MobileNetV2 conv_bn / conv_1x1_bn: conv -> BN -> ReLU6 (mobilenet.py:22-35)."""

    @staticmethod
    def forward(ctx, x2d, geom, seq, clamp_out=True):
        from . import engine
        return ConvBNReLU6Function._finish(ctx, engine._conv_bn_relu6_body(seq, Act(x2d, *geom), clamp_out))


class InvertedResidualFunction(_FrozenFunction):
    """MobileNetV2 inverted residual: expand -> depthwise -> project (+ x) (mobilenet.py:38-76)."""

    @staticmethod
    def forward(ctx, x2d, geom, block, out=None):
        from . import engine
        return InvertedResidualFunction._finish(ctx, engine._inverted_residual_body(block, Act(x2d, *geom), out))


class SEStemFunction(_FrozenFunction):
    """layer0 of the SENets: conv1 -> bn1 -> relu1 -> ceil-mode pool (senet.py:272-283)."""

    @staticmethod
    def forward(ctx, x2d, geom, layer0, out=None):
        from . import engine
        return SEStemFunction._finish(ctx, engine._se_stem_body(layer0, Act(x2d, *geom), out))


class SEBottleneckFunction(_FrozenFunction):
    """SEResNetBottleneck / SEResNeXtBottleneck (senet.py:107-131): convolutions, squeeze-excite and the closing GEMM."""

    @staticmethod
    def forward(ctx, x2d, geom, block, out=None):
        from . import engine
        return SEBottleneckFunction._finish(ctx, engine._se_bottleneck_body(block, Act(x2d, *geom), out))


class BNInceptionStemFunction(_FrozenFunction):
    """The BNInception stem: conv1_7x7_s2 .. pool2_3x3_s2 (bninception.py:255-265)."""

    @staticmethod
    def forward(ctx, x2d, geom, model, out=None):
        from . import engine
        return BNInceptionStemFunction._finish(ctx, engine._bninception_stem_body(model, Act(x2d, *geom), out))


class InceptionFunction(_FrozenFunction):
    """One BNInception block (``spec``: a row of models.bninception.BLOCKS): its branches written in place into the
    concatenated output (bninception.py:266-483)."""

    @staticmethod
    def forward(ctx, x2d, geom, model, spec, out=None):
        from . import engine
        return InceptionFunction._finish(ctx, engine._inception_body(model, spec, Act(x2d, *geom), out))


class InceptionStemFunction(_FrozenFunction):
    """Units of Inception-v4 / Inception-ResNet-v2 / Inception-v3 outside the blocks, in sequence (``units``: a tuple of
    BasicConv2d / MaxPool2d): the stems (inceptionv4.py:274-276, inceptionresnetv2.py:305-311, torchvision_models.py:397-403)
    and conv2d_7b (inceptionresnetv2.py:319)."""

    @staticmethod
    def forward(ctx, x2d, geom, units, out=None):
        from . import engine
        return InceptionStemFunction._finish(ctx, engine._inception_stem_body(units, Act(x2d, *geom), out))


class InceptionBlockFunction(_FrozenFunction):
    """One block of Inception-v4 / Inception-ResNet-v2 / Inception-v3 (models.inception.BRANCHES): its branches written in place
    into the concatenated output, and the residual close of Block35 / 17 / 8."""

    @staticmethod
    def forward(ctx, x2d, geom, block, out=None):
        from . import engine
        return InceptionBlockFunction._finish(ctx, engine._inception_block_body(block, Act(x2d, *geom), out))


class PolyNetBlockFunction(_FrozenFunction):
    """One module of the PolyNet trunk (polynet.py:71-371): the stem, a reduction, a 2-way module or a poly-3 module, every
    branch written in place into its concatenation matrix."""

    @staticmethod
    def forward(ctx, x2d, geom, module):
        from . import engine
        return PolyNetBlockFunction._finish(ctx, engine._polynet_block_body(module, Act(x2d, *geom)))


class DenseNetTrunkFunction(_FrozenFunction):
    """The DenseNet trunk up to norm5 (torchvision densenet.py ``features`` without its last BatchNorm): every dense block as one
    matrix that its layers and the preceding transition (or the stem's pool) write in place."""

    @staticmethod
    def forward(ctx, x2d, geom, features):
        from . import engine
        return DenseNetTrunkFunction._finish(ctx, engine._densenet_trunk_body(features, Act(x2d, *geom)))


class VGGTrunkFunction(_FrozenFunction):
    """VGG's ``_features`` (torchvision vgg.py): convolutions with bias (+ folded BatchNorm) and ReLU, 2x2 max pools."""

    @staticmethod
    def forward(ctx, x2d, geom, features):
        from . import engine
        return VGGTrunkFunction._finish(ctx, engine._vgg_trunk_body(features, Act(x2d, *geom)))


class AlexNetTrunkFunction(_FrozenFunction):
    """AlexNet's ``_features`` (torchvision alexnet.py) on the space-to-depth image: conv1 as a valid 3x3 convolution, then
    convolutions with bias and ReLU and 3x3 stride-2 max pools."""

    @staticmethod
    def forward(ctx, x2d, geom, features):
        from . import engine
        return AlexNetTrunkFunction._finish(ctx, engine._alexnet_trunk_body(features, Act(x2d, *geom)))


class GBlockFunction(_FrozenFunction):
    """BigGAN-deep GBlock: ccbn-ReLU-1x1 -> ccbn-ReLU-[up]-3x3 -> ccbn-ReLU-3x3 -> ccbn-ReLU-1x1 (+ skip)."""

    @staticmethod
    def forward(ctx, x2d, geom, blk, aff, pk, kwargs):
        from . import biggan_engine
        out = biggan_engine._gblock_body(blk, Act(x2d, *geom), aff, pk, **kwargs)
        if isinstance(out, tuple):          # (block output, pre-activated input of the next block)
            ctx.mark_non_differentiable(out[0].data, out[1].data)
            return out[0].data, _geom(out[0]), out[1].data, _geom(out[1])
        ctx.mark_non_differentiable(out.data)
        return out.data, _geom(out), None, None


# ---------------------------------------------------------------------------------------------------------------
# fine-tuned residual blocks (models.resnet3d.ResNet3D.fine_tune)
# ---------------------------------------------------------------------------------------------------------------
class BlockTrainFunction(torch.autograd.Function):
    """BasicBlock / Bottleneck with a backward (engine.block_backward).  Inputs: the block input matrix and the block's
    conv weights and BatchNorm gamma / beta (engine.train_params), so autograd routes their gradients.  The forward runs
    the same kernels as the frozen path and keeps the block input, its post-ReLU intermediates and its output.  Gradients
    in and out are loss-scaled fp16 matrices already multiplied by the ReLU mask of the tensor they belong to; ``ls`` is
    the device pair [scale, 1/scale] shared by every fine-tuned block of one forward."""

    @staticmethod
    def forward(ctx, x2d, geom, block, ls, *params):
        from . import engine
        keep = []
        body = engine._bottleneck_body if hasattr(block, "conv3") else engine._basic_body
        y = body(block, Act(x2d, *geom), keep=keep)
        ctx.save_for_backward(x2d, y.data)
        ctx.hs = [h.data for h in keep]
        ctx.geoms = (geom, _geom(y), [_geom(h) for h in keep])
        ctx.block, ctx.ls = block, ls
        return y.data, _geom(y)

    @staticmethod
    def backward(ctx, gy, _geom_grad):
        from . import engine
        x2d, y2d = ctx.saved_tensors
        gx, gyo, ghs = ctx.geoms
        hs = [Act(h, *g) for h, g in zip(ctx.hs, ghs)]
        dx, grads = engine.block_backward(ctx.block, Act(x2d, *gx), hs, Act(gy.contiguous(), *gyo), ctx.ls, ctx.needs_input_grad[0],
                                          ctx.needs_input_grad[4:])
        return (dx.data if dx is not None else None, None, None, None) + tuple(grads)

    @classmethod
    def run(cls, block, a, ls):
        from . import engine
        data, geom = cls.apply(a.data, _geom(a), block, ls, *engine.train_params(block))
        return Act(data, *geom)


class FineTunePoolFunction(torch.autograd.Function):
    """Global average pool of the last fine-tuned block: fp32 [N][C] features out.  The backward picks the loss scale from
    the incoming fp32 gradient (ops.loss_scale_) and writes the scaled, ReLU-masked fp16 gradient of the block output."""

    @staticmethod
    def forward(ctx, y2d, geom, ls):
        a = Act(y2d, *geom)
        ctx.save_for_backward(y2d)
        ctx.geom, ctx.ls = geom, ls
        return ops.avgpool_global(a)[:, :a.C].float()

    @staticmethod
    def backward(ctx, gf):
        (y2d,) = ctx.saved_tensors
        ops.loss_scale_(gf, ctx.ls)
        return ops.avgpool_global_backward(gf, ctx.ls, Act(y2d, *ctx.geom)).data, None, None


# ---------------------------------------------------------------------------------------------------------------
# dense head with a backward on the same GEMM kernel
# ---------------------------------------------------------------------------------------------------------------
def _f16_padded(t2d):
    """fp32 / fp16 [rows][cols] -> contiguous fp16 [rows][round_up(cols, 8)] with zero padding columns."""
    rows, cols = t2d.shape
    out = torch.zeros((rows, ops._round_up(cols, 8)), dtype=torch.float16, device=t2d.device)
    out[:, :cols] = t2d
    return out


def _unit_affine(n, dev):
    return torch.ones(n, dtype=torch.float32, device=dev), torch.zeros(n, dtype=torch.float32, device=dev)


def _pow2(k):
    """int32 exponents in [-126, 126] -> fp32 2^k, exactly (built from the exponent bits)."""
    return ((k + 127) << 23).view(torch.float32)


def _row_exponents(g):
    """Per-row power-of-two scale of an fp32 [rows][cols] gradient, on the device: k with max |g[r]| * 2^k in [2^7, 2^8) (the
    target of ops.loss_scale_), 0 for an all-zero or non-finite row.  Returns (2^k, 2^-k), fp32 [rows][1]."""
    amax = g.abs().amax(1)
    _, e = torch.frexp(amax)                                         # amax = f * 2^e, f in [0.5, 1)
    ok = (amax > 0) & torch.isfinite(amax)
    k = torch.where(ok, 8 - e, torch.zeros_like(e)).clamp(-126, 126)
    return _pow2(k)[:, None], _pow2(-k)[:, None]


class LinearFunction(torch.autograd.Function):
    """y = x W^T + b on wgmma (fp16 operands, fp32 accumulate / output), with
    dL/dx = g W, dL/dW = g^T x, dL/db = sum_rows g computed by the same kernel (D = A . B^T with K-major operands:
    the gradient products take the transposed fp16 copies as their operands).

    The fp32 gradient g is rounded to fp16 for the products.  Cross-entropy gradients are (p - onehot) / B, mostly far below
    fp16's normal range, so each row of the A operand (a sample row of g for dL/dx, a class row of g^T for dL/dW) is first
    multiplied by its own power of two 2^k, which puts the row's peak in [2^7, 2^8); the fp32 product row is multiplied by
    2^-k afterwards, which is exact."""

    @staticmethod
    def forward(ctx, x, weight, bias, relu_input=False):
        if x.dim() != 2:
            raise ValueError("LinearFunction takes a [rows][features] matrix")
        x16 = ops.cast_rows(x, relu=relu_input) if x.dtype != torch.float16 else x
        pl = ops.PackedLinear(weight, bias)
        y = ops.linear(x16, pl, out_f32=True)
        ctx.save_for_backward(x16, weight)
        ctx.has_bias = bias is not None
        ctx.relu_input = relu_input
        ctx.in_features = weight.shape[1]
        return y

    @staticmethod
    def backward(ctx, gy):
        x16, weight = ctx.saved_tensors
        dev = gy.device
        rows, out_f = gy.shape
        in_f = ctx.in_features
        gx = gw = gb = None
        gy = gy.float()
        if ctx.needs_input_grad[0]:
            up, down = _row_exponents(gy)
            g16 = _f16_padded(gy * up)                                   # [rows][out_p]: A operand, K = out
            wt = _f16_padded(weight.detach().t())                        # [in][out_p]: B operand
            one, zero = _unit_affine(in_f, dev)
            gx = ops.gemm(g16, wt, one, zero, rows, in_f, out_f, out_f32=True) * down
            if ctx.relu_input:
                gx = gx * (x16[:, :in_f] > 0)
        if ctx.needs_input_grad[1]:
            g_t = gy.t()
            up, down = _row_exponents(g_t)
            gt = _f16_padded(g_t * up)                                   # [out][rows_p]: A operand, K = rows
            xt = _f16_padded(x16[:, :in_f].t())                          # [in][rows_p]
            one, zero = _unit_affine(in_f, dev)
            gw = ops.gemm(gt, xt, one, zero, out_f, in_f, rows, out_f32=True) * down
        if ctx.has_bias and ctx.needs_input_grad[2]:
            gb = gy.sum(0)
        return gx, gw, gb, None


def linear(x, weight, bias=None, relu_input=False):
    return LinearFunction.apply(x, weight, bias, relu_input)
