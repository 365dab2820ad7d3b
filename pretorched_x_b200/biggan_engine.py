"""BigGAN-deep generator forward on the H100 kernels (BASELINE.json configs[4]).

There is no reference code for this path (SURVEY.md section 8a row a14): the block bodies below implement the published
GBlock / SAGAN-attention / class-conditional-BN arithmetic restated in ``oracle/biggan.py`` (test infrastructure), on the
same hand-written kernels as the video path -- the persistent 1x1 GEMM, the slab 3x3 convolution, the fused attention --
plus the HBM-bound helpers in ``csrc/b2_gan.cu``.

How the pieces map:

* **All 48+ class-conditional BatchNorms of a forward come out of ONE GEMM.**  ``ccbn(x, y) = (x - mu) * rstd * (1 + Wg y)
  + Wb y`` is an affine map per (sample, channel): ``scale = rstd + (rstd * Wg) y`` and ``shift = (Wb - m * rstd * Wg) y
  - m * rstd`` are both linear in the conditioning vector y, so the (spectrally normalised) gain / bias matrices of every
  ccbn are stacked, with ``rstd`` and the mean folded in, into one fp16 matrix ``[2 * sum(C)][3 * 256]`` and a single
  wgmma GEMM with fp32 output produces every scale and shift of the network: ``aff[B][2 * sum(C)]`` (operands split
  into fp16 hi + lo parts, K = 3 x 256, so the gains carry ~22 bits).
* ccbn -> ReLU that FOLLOWS a convolution is that convolution's epilogue (per-sample affine, ``b2_conv_args.aff_ld``):
  conv2 carries bn3, conv3 carries bn4, conv1 carries bn2 (from 16x16 images on: a 128-row tile must stay inside one
  image); the conv bias is folded into the shift (``m = mean - bias``).  bn1 (its input also feeds the skip path) is one ``b2_ccbn_act_ndhwc`` pass.
* The nearest-2x upsampling in front of conv2 is never materialised: a 3x3 convolution of an upsampled image is four
  2x2 convolutions of the low-res image (one per output phase, filters summed when packed), which the slab kernel runs
  as 4 x 4 taps with a strided output write -- 2.25x fewer MACs and a quarter of the input bytes.
* bn1 + ReLU of block i+1 CAN be a second output of block i's conv4 (or of the attention's output GEMM): a second epilogue
  pass over the accumulator tile writes relu(ccbn1_next(h + skip)) next to h + skip (``next_affine``,
  ``dual_output=True``).  These layers are write-bound and the second 2-byte-per-element stream costs the 1x1 kernel about as
  much as the stand-alone ``b2_ccbn_act_ndhwc`` read+write pass it replaces, so it is off by default.
* conv4's epilogue adds the skip path: channel drop = the residual pitch, and for the upsampling block the epilogue reads
  the LOW-res x and upsamples on the fly (``residual_up``), so ``upsample(x)`` is never written either.
* Tail: the output BatchNorm + ReLU is folded into the last block's conv4 (``residual_pre``: the skip joins before the
  affine), and the 3x3 convolution to RGB runs as one 1x1 GEMM to 9 taps x 4 partial-product columns followed by a gather
  that also adds the bias, applies tanh and writes NCHW (``b2_rgb_head_gather_tanh``).
* Spectral norm: weights are divided by sigma (one power iteration from the stored ``u0``) when they are packed.
* Self-attention: theta and phi|g projections (zero-padded to the 64-column granularity of the attention kernel),
  2x2 max-pool of phi|g, the fused softmax(theta^T phi) g kernel, and the output 1x1 GEMM with gamma as its scale and x
  as its residual.
"""
import os

import torch
import torch.nn.functional as F

from . import functions as Fn
from . import ops
from .ops import Act, _round_up


def _sn_sigma(weight, u, eps):
    wm = weight.detach().double().reshape(weight.shape[0], -1)
    u = u.detach().double()
    v = F.normalize(u @ wm, eps=eps)
    u2 = F.normalize(v @ wm.t(), eps=eps)
    return ((v @ wm.t()) @ u2.t()).squeeze()


def _sn_weight(mod, eps):
    """fp64 weight / sigma of a spectrally normalised layer (eval mode: no update of u0)."""
    return mod.weight.detach().double() / _sn_sigma(mod.weight, mod.u0, eps)


FUSE_BN1 = os.environ.get("B2_GAN_FUSE_BN1", "1") != "0"      # A/B switch (tools, tests)


class _NS:
    pass


def _pack_conv(conv, eps, in_pitch, upsample=False):
    w = _sn_weight(conv, eps).float()
    pad = conv.padding
    return ops.PackedConv(w, conv.bias, None, (1, 1, 1), (0, int(pad[0]), int(pad[1])), in_pitch=in_pitch, upsample=upsample)


def _pack(model, dev):
    """Everything derived from the parameters: packed filters, the stacked ccbn GEMM, attention matrices."""
    eps_sn = model.SN_eps
    cond = model.dim_z + model.shared_dim
    pk = _NS()
    pk.cond_pitch = _round_up(cond, 8)
    rows_w, rows_scale, rows_shift = [], [], []       # of the stacked ccbn GEMM
    col = [0]

    def add_ccbn(bn, prev_bias):
        """Append this ccbn's scale and shift columns; returns (scale offset, shift offset, C)."""
        C = bn.output_size
        rstd = torch.rsqrt(bn.stored_var.detach().double() + bn.eps)
        m = bn.stored_mean.detach().double()
        if prev_bias is not None:
            m = m - prev_bias.detach().double()                     # ccbn(acc + bias) == affine of acc with mean - bias
        wg = _sn_weight(bn.gain, eps_sn)                           # [C][cond]
        wb = _sn_weight(bn.bias, eps_sn)
        rows_w.append(wg * rstd[:, None]);                   rows_scale.append(torch.ones_like(rstd)); rows_shift.append(rstd)
        rows_w.append(wb - (m * rstd)[:, None] * wg);        rows_scale.append(torch.ones_like(rstd)); rows_shift.append(-m * rstd)
        o = col[0]
        col[0] += 2 * C
        return (o, o + C, C)

    # first linear: rows re-ordered so that the GEMM output [B][16 * C0] is already channels-last [B * 16][C0]
    C0 = model.arch['in_channels'][0]
    bw2 = model.bottom_width ** 2
    wl = _sn_weight(model.linear, eps_sn).reshape(C0, bw2, cond).permute(1, 0, 2).reshape(bw2 * C0, cond)
    pk.lin_w = torch.zeros((bw2 * C0, pk.cond_pitch), dtype=torch.float16, device=dev)
    pk.lin_w[:, :cond] = wl.to(torch.float16)
    pk.lin_b = model.linear.bias.detach().reshape(C0, bw2).t().reshape(-1).float().contiguous()
    pk.lin_ones = torch.ones_like(pk.lin_b)

    pk.blocks, pk.att = {}, {}
    res = model.bottom_width
    for stage in model.blocks:
        for blk in stage:
            if hasattr(blk, 'conv4'):
                bp = _NS()
                hw_in = res * res
                h8, in8 = _round_up(blk.hidden_channels, 8), _round_up(blk.in_channels, 8)
                if blk.hidden_channels % 8 or blk.in_channels % 8 or blk.out_channels % 8:
                    raise NotImplementedError("GBlock channel counts must be multiples of 8 (got %d / %d / %d)" %
                                              (blk.in_channels, blk.hidden_channels, blk.out_channels))
                # bn2 rides in conv1's epilogue when a 128-row tile stays in one image (the upsampling of the second block
                # happens inside conv2, so nothing sits between conv1 and bn2 any more)
                bp.fuse2 = hw_in % 128 == 0
                bp.bn = [add_ccbn(blk.bn1, None),
                         add_ccbn(blk.bn2, blk.conv1.bias if bp.fuse2 else None),
                         add_ccbn(blk.bn3, blk.conv2.bias),
                         add_ccbn(blk.bn4, blk.conv3.bias)]
                bp.conv = [_pack_conv(blk.conv1, eps_sn, in8), _pack_conv(blk.conv2, eps_sn, h8, upsample=blk.upsample),
                           _pack_conv(blk.conv3, eps_sn, h8), _pack_conv(blk.conv4, eps_sn, h8)]
                pk.blocks[id(blk)] = bp
                if blk.upsample:
                    res *= 2
            else:
                C = blk.ch
                d, dv = C // 8, C // 2
                ap = _NS()
                ap.d, ap.dv = _round_up(d, 64), _round_up(dv, 64)        # attention kernel granularity; padding is zero weights
                ld = _round_up(C, 8)
                ap.wq = torch.zeros((ap.d, ld), dtype=torch.float16, device=dev)
                ap.wq[:d, :C] = _sn_weight(blk.theta, eps_sn).reshape(d, C).to(torch.float16)
                ap.wkv = torch.zeros((ap.d + ap.dv, ld), dtype=torch.float16, device=dev)
                ap.wkv[:d, :C] = _sn_weight(blk.phi, eps_sn).reshape(d, C).to(torch.float16)
                ap.wkv[ap.d:ap.d + dv, :C] = _sn_weight(blk.g, eps_sn).reshape(dv, C).to(torch.float16)
                ap.wo = torch.zeros((C, ap.dv), dtype=torch.float16, device=dev)
                ap.wo[:, :dv] = _sn_weight(blk.o, eps_sn).reshape(C, dv).to(torch.float16)
                ap.ones = torch.ones(max(ap.d + ap.dv, C), dtype=torch.float32, device=dev)
                ap.zeros = torch.zeros_like(ap.ones)
                ap.gamma = (torch.ones(C, dtype=torch.float32, device=dev) * blk.gamma.detach().float()).contiguous()
                pk.att[id(blk)] = ap

    # output layer: plain BN (shared by all samples) + ReLU pass, then 3x3 conv to RGB
    obn, oconv = model.output_layer[0], model.output_layer[2]
    rstd = torch.rsqrt(obn.stored_var.detach().double() + obn.eps)
    sc = obn.gain.detach().double() * rstd
    pk.out_scale = sc.float().reshape(1, -1).contiguous()
    pk.out_shift = (obn.bias.detach().double() - obn.stored_mean.detach().double() * sc).float().reshape(1, -1).contiguous()
    pk.out_conv = _pack_conv(oconv, eps_sn, _round_up(obn.output_size, 8))
    # Split RGB head: the 3x3 conv to 3 channels as ONE 1x1 GEMM to 9 taps x (3 + 1 pad) partial-product columns followed
    # by a gather-sum (+ bias, tanh, NCHW).  As a 3x3 slab convolution the layer streams x through the tensor core nine
    # times using 3 of 16 MMA columns (2.1 ms at B = 256); as a GEMM it is one HBM-bound pass.
    pk.head_w = None
    if oconv.weight.shape[0] <= 4 and tuple(oconv.weight.shape[2:]) == (3, 3):
        wo = _sn_weight(oconv, eps_sn)                                         # [K][C][3][3]
        Kh, Ch = wo.shape[0], wo.shape[1]
        hw_ = torch.zeros((40, _round_up(Ch, 8)), dtype=torch.float16, device=dev)
        for tap in range(9):
            hw_[tap * 4:tap * 4 + Kh, :Ch] = wo[:, :, tap // 3, tap % 3].to(torch.float16)
        pk.head_w, pk.head_k = hw_, Kh
        pk.head_ones = torch.ones(40, dtype=torch.float32, device=dev)
        pk.head_zeros = torch.zeros(40, dtype=torch.float32, device=dev)
        pk.head_bias = (oconv.bias.detach().float() if oconv.bias is not None else torch.zeros(Kh, device=dev)).contiguous()
    # Output BN + ReLU folded into the LAST GBlock's closing convolution: relu(s * (acc + b4 + skip) + t) =
    # relu(s * (acc + skip) + (s * b4 + t)), i.e. conv4 with per-channel scale s, shift s * b4 + t and the residual joining
    # before the affine (residual_pre).  Removes one full read + write of the largest activation.
    last = [blk for stage in model.blocks for blk in stage][-1]
    pk.last_block = last if hasattr(last, 'conv4') else None
    if pk.last_block is not None:
        c4 = pk.last_block.conv4
        pk.out_conv4 = _pack_conv(c4, eps_sn, _round_up(pk.last_block.hidden_channels, 8))
        pk.out_conv4.scale = pk.out_scale.reshape(-1).contiguous()
        pk.out_conv4.shift = (pk.out_scale.reshape(-1).double() * c4.bias.detach().double()
                              + pk.out_shift.reshape(-1).double()).float().contiguous()

    # stacked ccbn matrix as [W_hi | W_hi | W_lo] against the conditioning vector stored as [y_hi | y_lo | y_hi]: the fp16
    # GEMM then carries ~22 mantissa bits (a plain fp16 W and y put a 5e-4 relative error on every gain, which 48 stacked
    # ccbn layers turn into ~1e-2 of the image range)
    pk.ncols = col[0]
    D = pk.cond_pitch
    wall = torch.cat(rows_w, 0)
    w_hi = wall.to(torch.float16)
    w_lo = (wall - w_hi.double()).to(torch.float16)
    pk.cond_w = torch.zeros((pk.ncols, 3 * D), dtype=torch.float16, device=dev)
    pk.cond_w[:, :cond] = w_hi
    pk.cond_w[:, D:D + cond] = w_hi
    pk.cond_w[:, 2 * D:2 * D + cond] = w_lo
    pk.cond_scale = torch.cat(rows_scale).float().contiguous()
    pk.cond_shift = torch.cat(rows_shift).float().contiguous()
    return pk


def _packed(model, dev):
    tensors = list(model.parameters()) + list(model.buffers())
    sig = tuple((t.data_ptr(), t._version) for t in tensors) + (str(dev),)
    hit = model.__dict__.get('_b2_pack')
    if hit is not None and hit[0] == sig:
        return hit[1]
    with torch.no_grad():
        pk = _pack(model, dev)
    model.__dict__['_b2_pack'] = (sig, pk)
    return pk


def _aff(aff, slot):
    o_scale, o_shift, C = slot
    return aff[:, o_scale:o_scale + C], aff[:, o_shift:o_shift + C]


def _next_affine(nxt, a_out_hw, aff, pk):
    """(scale, shift) of the ccbn that opens the GBlock ``nxt`` when the producer of its input may write it as a second
    output (a 128-row tile must stay inside one image), else None."""
    if nxt is None or not hasattr(nxt, 'conv4') or a_out_hw % 128 != 0:
        return None
    return _aff(aff, pk.blocks[id(nxt)].bn[0])


def run_gblock(blk, a, aff, pk, fuse_output_bn=False, pre=None, nxt=None, out=None):
    """One GBlock through the frozen torch.autograd.Function (``functions.frozen``: forward = the launch sequence of
    ``_gblock_body``, outputs non-differentiable).  Returns (block output, relu(bn1_next(output)) or None).  ``out``:
    preallocated rows for the block output (written by conv4's epilogue)."""
    y = Fn.frozen(lambda x, o: _gblock_body(blk, x, aff, pk, fuse_output_bn=fuse_output_bn, pre=pre, nxt=nxt, out=o), a, out)
    return y if isinstance(y, tuple) else (y, None)


def _gblock_body(blk, a, aff, pk, fuse_output_bn=False, pre=None, nxt=None, out=None):
    """One GBlock: h = conv4(relu(bn4(conv3(relu(bn3(conv2(up(relu(bn2(conv1(relu(bn1(x))))))))))))) + up(x[:, :out]).
    ``pre``: relu(bn1(x)) when the previous kernel already produced it; ``nxt``: the module that consumes the result --
    if it is a GBlock its opening ccbn + ReLU is written as a second output of conv4 (returned as the second value).
    ``fuse_output_bn`` (last block only): returns relu(bn_out(h)) instead, see ``_pack``."""
    bp = pk.blocks[id(blk)]
    up = 2 if blk.upsample else 1
    in_aff = None
    if pre is None:
        s1, t1 = _aff(aff, bp.bn[0])
        if bp.fuse2 and (a.H * a.W) % 128 == 0 and a.ld % 64 == 0 and FUSE_BN1:
            in_aff, pre = (s1, t1), a            # bn1 + ReLU applied to conv1's A operand inside the GEMM: no stand-alone pass
        else:
            pre = ops.ccbn_act(a, s1, t1)                                    # relu(bn1(x))
    t = pre
    if bp.fuse2:
        t = ops.conv(t, bp.conv[0], relu=True, sample_affine=_aff(aff, bp.bn[1]), in_affine=in_aff)     # relu(bn2(conv1(relu(bn1(x)))))
    else:
        t = ops.conv(t, bp.conv[0])                                          # conv1 + bias
        s2, t2 = _aff(aff, bp.bn[1])
        t = ops.ccbn_act(t, s2, t2)                                          # relu(bn2(.)) (4x4 / 8x8 images only)
    # conv2; in the upsampling block it reads the LOW-res tensor: conv3x3(up2(.)) == four folded 2x2 phase filters
    t = ops.conv(t, bp.conv[1], relu=True, sample_affine=_aff(aff, bp.bn[2]))          # relu(bn3(conv2(up(.))))
    t = ops.conv(t, bp.conv[2], relu=True, sample_affine=_aff(aff, bp.bn[3]))          # relu(bn4(conv3(.)))
    # conv4 + skip: the skip path x[:, :out] (channel drop = residual pitch) is read at LOW resolution by the epilogue and
    # upsampled on the fly, so up(x) is never written; the last block also carries the output BN + ReLU (see _pack)
    if fuse_output_bn:
        return ops.conv(t, pk.out_conv4, residual=a, relu=True, residual_up=up == 2, residual_pre=True, out=out)
    nxt_aff = _next_affine(nxt, t.H * t.W, aff, pk)
    return ops.conv(t, bp.conv[3], residual=a, residual_up=up == 2, next_affine=nxt_aff, out=out)    # Act, or (Act, Act) with nxt_aff


def run_attention(att, a, aff, pk, nxt=None, out=None):
    """SAGAN self-attention with 2x2 max-pooled keys / values: gamma * o(softmax(theta^T phi) g) + x.  Returns (result,
    relu(bn1_next(result)) or None) like ``run_gblock``."""
    ap = pk.att[id(att)]
    C, M = att.ch, a.M
    nkv = ap.d + ap.dv
    q = ops.gemm(a.data, ap.wq, ap.ones[:ap.d], ap.zeros[:ap.d], M, ap.d, a.ld)
    kv = ops.gemm(a.data, ap.wkv, ap.ones[:nkv], ap.zeros[:nkv], M, nkv, a.ld)
    kvp = ops.maxpool3d(Act(kv, a.N, 1, a.H, a.W, nkv), (1, 2, 2), (1, 2, 2), (0, 0, 0))
    o = ops.attention(q, kvp.data, kvp.data[:, ap.d:], ap.d, ap.dv, a.N, a.H * a.W, kvp.positions)
    nxt_aff = _next_affine(nxt, a.H * a.W, aff, pk)
    if nxt_aff is not None:
        z, z2 = ops.gemm(o, ap.wo, ap.gamma, ap.zeros[:C], M, C, ap.dv, residual=a.data,
                         next_affine=(nxt_aff[0], nxt_aff[1], a.H * a.W))
        return Act(z, a.N, 1, a.H, a.W, C), Act(z2, a.N, 1, a.H, a.W, C)
    if out is not None:
        ops._out_rows(out, M, _round_up(C, 8))
    z = ops.gemm(o, ap.wo, ap.gamma, ap.zeros[:C], M, C, ap.dv, residual=a.data, out=out)
    return Act(z, a.N, 1, a.H, a.W, C), None


_DFS_SPEC = os.environ.get("B2_GAN_DFS", "off")


def set_dfs(spec):
    """Schedule of the generator's high-resolution tail: ``"off"`` (whole batch per launch: the default,
    see ``engine.set_dfs``) or ``"res:images,res:images"`` -- modules whose OUTPUT resolution is at least ``res`` (up to the next
    listed resolution) run depth-first on chunks of ``images``."""
    global _DFS_SPEC
    _DFS_SPEC = str(spec)


def dfs_plan(model, B, mods):
    """[(first module, end module, images per chunk)] covering a suffix of ``mods`` (empty = whole batch everywhere)."""
    spec = _DFS_SPEC.strip().lower()
    if spec in ("0", "off", "none", "", "auto"):      # "auto" = the default rule: never chunk
        return []
    levels = sorted(tuple(int(v) for v in part.split(":")) for part in spec.split(","))
    res, out_res = model.bottom_width, []
    for _, blk in mods:
        if hasattr(blk, 'conv4') and blk.upsample:
            res *= 2
        out_res.append(res)
    plan = []
    for li, (r0, chunk) in enumerate(levels):
        r1 = levels[li + 1][0] if li + 1 < len(levels) else 1 << 30
        js = [j for j, r in enumerate(out_res) if r0 <= r < r1]
        if not js or chunk >= B:
            if plan:              # a whole-batch level after a chunked one: keep the suffix contiguous by chunking it by B
                if js:
                    plan.append((js[0], js[-1] + 1, B))
            continue
        plan.append((js[0], js[-1] + 1, chunk))
    return plan


def generator_forward(model, z, y, out_dtype=torch.float32, stages=None, fuse_output_bn=True, split_head=True,
                      dual_output=False):
    """z fp32 [B, dim_z] (CUDA), y int64 [B] class indices or fp32 [B, shared_dim] embeddings -> images [B, 3, R, R].
    ``stages``: optional dict receiving the Act after the first linear, every stage, the output BN+ReLU ('out_act') and
    the RGB conv ('pre_tanh').  With ``fuse_output_bn`` (default) the last stage's raw output never exists (its closing
    convolution writes relu(bn_out(.)) directly), so 'stage{last}' is only recorded when it is off; with ``split_head``
    (default) the RGB convolution runs as a 1x1 GEMM + gather and 'pre_tanh' is only recorded when it is off."""
    if model.training:
        raise RuntimeError("the H100 engine is inference-only: call model.eval() (standing statistics, no SN update)")
    if not z.is_cuda:
        raise RuntimeError("the generator runs on a CUDA (sm_90a) device only: this engine has no CPU path")
    dev = z.device
    pk = _packed(model, dev)
    B = z.shape[0]
    cond = model.dim_z + model.shared_dim
    y16 = ops.embed_concat(z, y.to(dev), model.shared.weight, split=True)                # [B][3D] = [hi | lo | hi]
    aff = ops.gemm(y16, pk.cond_w, pk.cond_scale, pk.cond_shift, B, pk.ncols, 3 * pk.cond_pitch, out_f32=True)   # every ccbn at once
    C0, bw = model.arch['in_channels'][0], model.bottom_width
    h = ops.gemm(y16, pk.lin_w, pk.lin_ones, pk.lin_b, B, bw * bw * C0, cond)
    a = Act(h.view(B * bw * bw, C0), B, 1, bw, bw, C0)
    if stages is not None:
        stages['linear'] = a
    mods = [(i, blk) for i, stage in enumerate(model.blocks) for blk in stage]

    def run_mods(a, aff, j0, j1, out=None):
        """Modules j0 .. j1-1 on the activation ``a`` (whole batch or a chunk of images, ``aff`` sliced alike)."""
        fused_tail, pre = False, None           # pre: relu(bn1(a)) of the upcoming GBlock when its producer already wrote it
        for j in range(j0, j1):
            i, blk = mods[j]
            nxt = mods[j + 1][1] if (j + 1 < len(mods) and dual_output) else None
            o = out if j == j1 - 1 else None
            if hasattr(blk, 'conv4'):
                fused_tail = fuse_output_bn and blk is pk.last_block
                a, pre = run_gblock(blk, a, aff, pk, fuse_output_bn=fused_tail, pre=pre, nxt=nxt, out=o)
            else:
                a, pre = run_attention(blk, a, aff, pk, nxt=nxt, out=o)
            if stages is not None and not fused_tail and (j + 1 == len(mods) or mods[j + 1][0] != i):
                stages['stage%d' % i] = a
        return a, fused_tail

    def run_tail(a, fused_tail, out=None):
        t = a if fused_tail else ops.ccbn_act(a, pk.out_scale, pk.out_shift)
        if stages is not None:
            stages['out_act'] = t
        if split_head and pk.head_w is not None:
            part = ops.gemm(t.data, pk.head_w, pk.head_ones, pk.head_zeros, t.M, 40, t.ld)      # per-tap partial products
            return ops.rgb_head(part, pk.head_bias, t.N, t.H, t.W, pk.head_k, out_dtype, out=out)   # gather + bias + tanh + NCHW
        t = ops.conv(t, pk.out_conv)
        if stages is not None:
            stages['pre_tanh'] = t
        return ops.tanh_to_nchw(t, out_dtype, out=out)

    # Optional depth-first tail (set_dfs; off by default, see engine.set_dfs): the modules of the listed
    # resolutions run on chunks of images, every intermediate a write-then-read inside L2; chunk outputs land in their slice of the
    # next segment's input (or of the image tensor).  Not with ``stages`` (whole-batch stage tensors wanted) or ``dual_output``.
    plan = [] if (stages is not None or dual_output) else dfs_plan(model, B, mods)
    j_first = plan[0][0] if plan else len(mods)
    a, fused_tail = run_mods(a, aff, 0, j_first)
    images = None
    for j0, j1, chunk in plan:
        last = j1 == len(mods)
        if chunk >= B:                              # a whole-batch level behind a chunked one
            a, fused_tail = run_mods(a, aff, j0, j1)
            continue
        buf = None
        r = a.positions
        for n0 in range(0, B, chunk):
            n1 = min(B, n0 + chunk)
            ca, caff = Act(a.data[n0 * r:n1 * r], n1 - n0, 1, a.H, a.W, a.C), aff[n0:n1]
            if last:                                # ... through the RGB head: the chunk's images go straight into the batch tensor
                y, ft = run_mods(ca, caff, j0, j1)
                if images is None:
                    K = pk.head_k if (split_head and pk.head_w is not None) else pk.out_conv.K
                    images = torch.empty((B, K, y.H, y.W), dtype=out_dtype, device=dev)
                run_tail(y, ft, out=images[n0:n1])
                continue
            o = buf.data[n0 * buf.positions:n1 * buf.positions] if buf is not None else None
            y, _ = run_mods(ca, caff, j0, j1, out=o)
            if buf is None:                         # the first chunk shows the segment's output geometry
                buf = Act(torch.empty((B * y.positions, y.ld), dtype=torch.float16, device=dev), B, 1, y.H, y.W, y.C)
                o = buf.data[:y.M]
            if y.data.data_ptr() != o.data_ptr():
                o.copy_(y.data)
        if not last:
            a = buf
    if images is not None:
        return images
    return run_tail(a, fused_tail)
