/* b2_pretorched.h -- C ABI of the H100-native forward engine for pretorched-x's video-ConvNet hot path.
 *
 * The reference (alexandonian/pretorched-x @ 36a5754) has no FFI layer of its own: every FLOP of
 * its hot path is a torch.nn call inside a Python `forward` body.  Each entry point below therefore
 * cites the reference *operator call site(s)* it replaces (file:line under /root/reference).  The
 * Python host side (pretorched_x_b200/) binds these with ctypes; INTEGRATION.md shows the stub a
 * reference maintainer would add.
 *
 * Conventions
 *   - All data pointers are DEVICE pointers owned by the caller.  The library never allocates, frees
 *     or retains them; work is enqueued on `stream` (a cudaStream_t passed as void*) and the call
 *     returns immediately.  Safe under CUDA-graph capture (no syncs, no allocations).
 *   - Activations are fp16 NDHWC ("channels last"), i.e. a dense matrix [N*T*H*W][ld] with channel
 *     pitch `ld` (elements) a multiple of 8.  Channels in [C, ld) must be zero.
 *   - Returns 0 on success, a negative B2_ERR_* code otherwise; b2_last_error() returns a
 *     thread-local message.  No C++ exception crosses the ABI.
 *   - There is NO CPU fallback: on a machine without an sm_90 GPU every compute call fails with
 *     B2_ERR_CUDA / B2_ERR_UNSUPPORTED.
 */
#ifndef B2_PRETORCHED_H_
#define B2_PRETORCHED_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B2_OK 0
#define B2_ERR_INVALID (-1)     /* bad argument (shape, alignment, null pointer) */
#define B2_ERR_CUDA (-2)        /* a CUDA runtime / driver call failed */
#define B2_ERR_UNSUPPORTED (-3) /* valid request the engine does not implement */

#define B2_CONV_AUTO 0  /* generic implicit GEMM: x has channel pitch C (multiple of 8)            */
#define B2_CONV_STEM7 1 /* kw == 7, strides (1,2,2), pw == 3, Cin <= 4 stored as NDHWC4 (stem convs)  */

int b2_version(void);
const char* b2_last_error(void);
/* number of kernels this library has launched from the calling process so far (bench bookkeeping) */
uint64_t b2_launch_count(void);

/* ---------------------------------------------------------------------------------------------
 * Convolution as implicit GEMM on wgmma tensor cores, with the eval-mode BatchNorm affine
 * (scale/shift), the residual add and the ReLU fused into the epilogue:
 *     y[m, k] = act( scale[k] * sum_{tap,c} x[m @ tap, c] * w[k, tap, c] + shift[k] + residual[m, k] )
 * Replaces nn.Conv3d -> nn.BatchNorm3d -> (+=residual) -> nn.ReLU chains at
 *   resnet3D.py:91-106 (BasicBlock.forward), resnet3D.py:125-143 (Bottleneck.forward),
 *   resnet3D.py:176-185 (type-B shortcut), r2plus1d.py:85-88 (SpatioTemporalConv.forward),
 *   nonlocalnet.py:143-166 (theta/phi/g/W 1x1x1 convs), torchvision_models.py:448-452 (stem).
 * ------------------------------------------------------------------------------------------- */
typedef struct b2_conv_args {
  const void* x;        /* fp16 [N,T,H,W,C]; C is the channel pitch                               */
  const void* w;        /* fp16 packed [K][taps][C] (b2_pack_conv_weight), taps = kt*kh*kw        */
  const float* scale;   /* fp32 [K]                                                                */
  const float* shift;   /* fp32 [K]                                                                */
  const void* residual; /* nullable; fp16 [M][ldr], M = N*To*Ho*Wo.  Only columns [0, K) are read: whatever columns
                           [K, ldr) hold (a wider skip tensor's dropped channels) never reaches y, and ldr < ldy is fine */
  void* y;              /* fp16 [M][ldy]  (fp32 when out_f32)                                      */
  int32_t N, T, H, W, C;
  int32_t K;            /* logical output channels; columns [K, ldy) of an fp16 y are written as zero, those of an fp32 y
                           (out_f32) are left untouched                                            */
  int32_t ldy, ldr;
  int32_t kt, kh, kw;
  int32_t st, sh, sw;
  int32_t pt, ph, pw;
  int32_t relu;
  int32_t out_f32;      /* y is fp32 (direct-store epilogue)                                       */
  int32_t accumulate;   /* out_f32 only: y += result                                               */
  int32_t mode;         /* B2_CONV_AUTO | B2_CONV_STEM7                                            */
  int32_t aff_ld;       /* 0: scale/shift are [K].  > 0: per-SAMPLE affine, scale/shift are fp32 [N][aff_ld], 16-byte aligned,
                           aff_ld % 4 == 0
                           (class-conditional BatchNorm of the layer that FOLLOWS this convolution, BigGAN GBlock);
                           multi-tap convolutions with in-plane padding between 0 and "same" (temporal "same") and
                           1x1x1 convolutions with To*Ho*Wo % 128 == 0 only                                        */
  int32_t upsample;     /* 1: y = conv3x3(nearest_upsample_2x(x)) without materialising the upsampled image (GBlock conv2):
                           x is the LOW-resolution input [N,1,H,W,C], y has (2H) x (2W) pixels per image, and w is the
                           phase-folded filter bank [K][16][C] written by b2_pack_upconv3x3_weight.  kt=1, kh=kw=3,
                           strides 1, padding (0,1,1) only                                                        */
  int32_t residual_up;  /* 1: `residual` is the LOW-resolution tensor [N][H/2][W/2][ldr] of the skip path and is nearest-2x
                           upsampled on the fly (GBlock: h + upsample(x[:, :out]); the channel drop is the pitch ldr).
                           1x1 stride-1 2-D convolutions only                                                     */
  int32_t residual_pre; /* 1: y = act(scale * (acc + residual) + shift) -- the residual joins BEFORE the affine (BatchNorm of
                           the block output folded into its closing convolution).  1x1 convolutions only           */
  void* y2;             /* nullable second output, fp16 [M][ldy]: y2 = relu(y * scale2[n] + shift2[n]) with y the fp32 value of
                           the first output -- the class-conditional BatchNorm + ReLU that OPENS the next GBlock, produced
                           while the tile is still on chip.  1x1 stride-1 convolutions with To*Ho*Wo % 128 == 0 only */
  const float* scale2;  /* fp32 [N][aff2_ld] */
  const float* shift2;
  int32_t aff2_ld;
  int32_t pool_w;       /* B2_CONV_STEM7 only, needs relu: the MaxPool (k = 3, stride 2, padding 1 ALONG W) that follows the stem
                           (resnet3D.py:156, torchvision_models.py:452) is applied in the epilogue.  y then has
                           Wp = (Wo - 1) / 2 + 1 columns per output row ([N*To*Ho*Wp][ldy]); the H / T directions of the pool
                           are a second b2_maxpool3d_ndhwc call with kernel (kt, kh, 1) -- max-pooling is separable -- over a
                           tensor half the size.  Output rows of at most 120 columns                                   */
  const float* in_scale; /* nullable.  Per-SAMPLE affine + ReLU applied to the INPUT of a 1x1 stride-1 convolution on its way to the
                            tensor core: the convolution sees relu(x * in_scale[n][c] + in_shift[n][c]) -- the class-conditional
                            BatchNorm + ReLU that opens a GBlock, without a stand-alone pass over x (x itself stays untouched in
                            memory: the block's skip path reads it raw).  fp32 [N][in_aff_ld], 16-byte aligned, in_aff_ld % 4 == 0,
                            To*Ho*Wo % 128 == 0                                                                           */
  const float* in_shift;
  int32_t in_aff_ld;
  const void* mask;     /* nullable fp16 [M][ldm] (ldm % 8 == 0, ldm >= ldy): y = (scale * acc + shift + residual) where mask > 0,
                           else 0, in fp32 before the single rounding -- the ReLU derivative of the fine-tuning backward.  fp16
                           output without relu / per-sample affine / generator extras; taken by the persistent GEMM and the
                           implicit-GEMM kernel only (the dispatcher skips every other path for a masked call)              */
  int32_t ldm;
} b2_conv_args;

int b2_conv_ndhwc_fprop(const b2_conv_args* a, void* stream);
/* Same contract on plain CUDA cores (one thread per output element, fp32 accumulate).  A debugging
 * cross-check for the tensor-core path; never used by the model forward. */
int b2_conv_ndhwc_fprop_simt(const b2_conv_args* a, void* stream);

/* fp32 [K][Cin][kt][kh][kw] (nn.Conv3d.weight layout, resnet3D.py:60,115-119) -> fp16 packed
 * [K][taps][C] with zero padding of channels [Cin, C).  mode B2_CONV_STEM7: a pre-laid-out shared-memory image
 * [ntile][kt][kh taps, even dh descending then odd dh descending][BN x 32] (see csrc/b2_stemconv.cuh). */
size_t b2_pack_conv_weight_elems(int K, int Cin, int kt, int kh, int kw, int C, int mode);
int b2_pack_conv_weight(const float* w_oidhw, void* w_packed, int K, int Cin, int kt, int kh, int kw, int C,
                        int mode, void* stream);

/* fp32 [K][Cin][3][3] (nn.Conv2d.weight) -> fp16 [K][16][C]: the four 2x2 filters that a 3x3 convolution of a nearest-2x
 * upsampled image collapses to, one per output phase ph = 2*py + px, tap index ph*4 + 2*a + b.  Output pixel (2h+py, 2w+px)
 * reads low-res rows h-1+py+a, columns w-1+px+b (a, b in {0,1}); the folded weight is the sum of the 3x3 taps that land on
 * that low-res pixel (rows: py=0 -> {0},{1,2}; py=1 -> {0,1},{2}).  2.25x fewer MACs, input read at 1/4 of the size. */
int b2_pack_upconv3x3_weight(const float* w_oihw, void* w_packed, int K, int Cin, int C, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Dense layer / 1x1x1 convolution as a plain GEMM:  D[M][N] = act(scale * (A[M][Kd] . B[N][Kd]^T) + shift
 * + residual).  scale/shift index the N dimension, or the M dimension when per_row != 0 (swap-AB use:
 * D^T = B . A^T with the affine following the rows).  Replaces nn.Linear at
 * resnet3D.py:162 / torchvision_models.py:460-464 (head), trn.py:39-49 (Relation MLP).
 * ------------------------------------------------------------------------------------------- */
typedef struct b2_gemm_args {
  const void* a; /* fp16 [M][lda] */
  const void* b; /* fp16 [N][ldb] */
  const float* scale;
  const float* shift;
  const void* residual; /* nullable fp16 [M][ldr]; only columns [0, N) are read */
  void* d;              /* fp16 [M][ldd] or fp32 when out_f32 */
  int32_t M, N, Kd;
  int32_t lda, ldb, ldd, ldr;
  int32_t per_row;
  int32_t relu;
  int32_t out_f32;
  int32_t accumulate;
  int32_t aff_ld;   /* 0: scale/shift are [N] (or [M] when per_row).  > 0: per-sample affine, fp32 [M / aff_rows][aff_ld]:
                       row m uses scale[(m / aff_rows) * aff_ld + n]; fp16 output only, aff_rows % 128 == 0 */
  int32_t aff_rows;
  void* d2;             /* nullable second output fp16 [M][ldd]: d2 = relu(d * scale2[m / aff2_rows] + shift2[...]) (see y2 above) */
  const float* scale2;
  const float* shift2;
  int32_t aff2_ld, aff2_rows;
  const void* mask;     /* nullable fp16 [M][ldm] ReLU-derivative mask of the output, see b2_conv_args.mask */
  int32_t ldm;
} b2_gemm_args;
int b2_gemm_f16(const b2_gemm_args* a, void* stream);
/* D = act(scale * (A.B^T + A2.B2^T) + shift + residual): both products accumulate in the same accumulator tile.  Used to
 * fuse the type-B shortcut projection (resnet3D.py:176-185) into the block-closing 1x1x1 convolution
 * (resnet3D.py:136-143) with the two BatchNorm scales folded into B and B2: the shortcut never touches HBM.
 * fp16 output, per-column affine only. */
int b2_gemm2_f16(const b2_gemm_args* a, const void* a2, int lda2, const void* b2, int ldb2, int k2, void* stream);
/* A bottleneck's closing 1x1x1 convolution chained into the next block's conv1 in one kernel:
 *     d  = act(scale * (A.B^T [+ A2.B2^T]) + shift + residual)        (as b2_gemm_f16 / b2_gemm2_f16; k2 = 0: no second pair)
 *     d1 = relu(scale1[n] * (d . W1^T) + shift1[n])                   W1 fp16 [n1][ldw1 >= N], d1 fp16 [M][ldd1]
 * d1 is computed from the fp16 d tile while it is still on chip, so d is written once and not read back.  Both results are
 * bit-identical to the two stand-alone calls.  Contract: fp16 output, per-column affine, no per-sample affine, mask or second
 * output, N % 64 == 0, N <= 256, ldd == N, ldd1 <= 128 (columns [n1, ldd1) of d1 are written as zero); anything else returns
 * B2_ERR_UNSUPPORTED and the caller runs the two calls. */
int b2_gemm_chain_f16(const b2_gemm_args* a, const void* a2, int lda2, const void* b2, int ldb2, int k2, const void* w1, int ldw1, int n1,
                      const float* scale1, const float* shift1, void* d1, int ldd1, void* stream);
/* b2_gemm_f16 with a per-sample affine at ANY number of rows per sample (b2_gemm_f16 needs aff_rows % 128 == 0, so that a
 * 128-row tile never straddles two samples):
 *     D[m][n] = act(scale[m / aff_rows][n] * (A.B^T)[m][n] + shift[m / aff_rows][n] + residual[m][n])
 * Each output row resolves its own sample.  The closing 1x1 convolution of an SE bottleneck (senet.py:111-131) with the
 * squeeze-excite factor folded into the bn3 affine (b2_se_excite): at 224^2 its rows per sample are 3136 / 784 / 196 / 49.
 * Contract: aff_ld > 0, aff_ld % 4 == 0, aff_ld >= N, scale / shift 16-byte aligned, aff_rows > 0, M % aff_rows == 0,
 * N % 8 == 0; fp16 output (columns [N, ldd) written as zero; residual columns >= N never read); per_row, out_f32, accumulate,
 * d2 and mask must be zero / NULL (B2_ERR_INVALID).  Always the persistent GEMM (b2_debug_last_gemm_path() == 2). */
int b2_gemm_sample_affine_f16(const b2_gemm_args* a, void* stream);
/* Two fp16 outputs from one fp32 accumulator acc = A.B^T:
 *     d  = act(scale[n] * acc + shift[n] + residual[m][n])          (as b2_gemm_f16; a: its args, act = ReLU when a->relu)
 *     d2 = relu(scale2[n] * acc + shift2[n])                         fp16 [M][ldd2], scale2 / shift2 fp32 [N]
 * The closing 1x1 convolution of one application of a PolyNet poly-3 module (polynet.py:229-326): with (sb, tb) the folded
 * BatchNorm of that application's conv2d and s the module's scale, scale = s * sb, shift = s * tb, residual = the running sum,
 * so d is the new running sum and d2 = relu(sb * acc + tb) the next application's input.  d2 is not relu(d * scale2 + shift2)
 * (the generator's second output, b2_gemm_args.d2): it is taken from the accumulator, before the residual joins.
 * Contract: fp16 d with a per-column affine (columns [N, ldd) written as zero, residual columns >= N never read); d2 has d's
 * pitch (ldd2 == ldd; its columns [N, ldd) are written as zero too), is 16-byte aligned and shares no byte with d, A, B or the
 * residual (B2_ERR_INVALID).  out_f32, per_row, accumulate, aff_ld / aff_rows (per-sample affines), mask, and the args' own d2 / scale2 /
 * shift2 / aff2 fields must be zero (B2_ERR_UNSUPPORTED).  Always the persistent GEMM (b2_debug_last_gemm_path() == 2;
 * b2_debug_last_kernel: KID 6, info = {N tile, 4, 0}).  d is bitwise what b2_gemm_f16 writes for the same arguments. */
int b2_gemm_dual_f16(const b2_gemm_args* a, const float* scale2, const float* shift2, void* d2, int ldd2, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Non-local block core (nonlocalnet.py:143-211):
 *     mode 0:  O[b] = softmax_rows(Q[b] . K[b]^T) . V[b]   (`_embedded_gaussian` :143-166, `_gaussian` :168-190;
 *                                                          unscaled logits, softmax over keys)
 *     mode 1:  O[b] = (Q[b] . K[b]^T / Nk) . V[b]          (`_dot_product` :192-211)
 *     mode 2:  O[b] = (relu(Q[b] . K[b]^T) / Nk) . V[b]    (`_concatenation` :213-243: concat_project's 1x1 conv over
 *                                                          [theta_i ; phi_j] is a_i + b_j, which the caller encodes as the
 *                                                          rank-2 product Q_i = [a_i, 1, 0..], K_j = [1, b_j, 0..])
 * Q: fp16 [B*Nq][ldq] (d columns used); K, V: fp16 [B*Nk][ld] (d resp. dv columns; Nk < Nq when phi and g were
 * max-pooled, `sub_sample=True` :126-131); O: fp16 [B*Nq][ldo].  One fused kernel, the Nq x Nk matrix is never
 * materialised.
 * ------------------------------------------------------------------------------------------- */
int b2_nonlocal_attention(const void* q, int ldq, const void* k, int ldk, const void* v, int ldv, void* o,
                          int ldo, int B, int Nq, int Nk, int d, int dv, int mode, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Pooling / layout / elementwise helpers (all HBM-bound, 128-bit accesses)
 * ------------------------------------------------------------------------------------------- */
/* nn.MaxPool3d (resnet3D.py:156): padding taps are skipped (== -inf padding). */
int b2_maxpool3d_ndhwc(const void* x, void* y, int N, int T, int H, int W, int C, int kt, int kh, int kw,
                       int st, int sh, int sw, int pt, int ph, int pw, void* stream);
/* The same pooling with the output extent (To, Ho, Wo) given by the caller, for windows that b2_maxpool3d_ndhwc's floor rule
 * does not produce: nn.MaxPool2d(3, stride=2, ceil_mode=True) of the SENet stem (senet.py:279-282) maps 112 -> 56 with the last
 * window clipped at the edge.  Taps outside the input are skipped; every window must overlap the input (B2_ERR_INVALID). */
int b2_maxpool3d_ndhwc_out(const void* x, void* y, int N, int T, int H, int W, int C, int kt, int kh, int kw, int st, int sh, int sw,
                           int pt, int ph, int pw, int To, int Ho, int Wo, void* stream);
/* nn.AdaptiveAvgPool3d(1) (resnet3D.py:161): x fp16 [N][S][C] -> y fp16 [N][C], fp32 accumulation. */
int b2_avgpool_global_ndhwc(const void* x, void* y, int N, int S, int C, void* stream);
/* fp32 NCDHW (the reference's input layout) -> fp16 NDHWC with channel pitch Cp (zero padded). */
int b2_ncdhw_f32_to_ndhwc_f16(const float* x, void* y, int N, int C, int T, int H, int W, int Cp, void* stream);
/* Same for callers that already hold fp16 clips (halves the host->device traffic of the input). */
int b2_ncdhw_f16_to_ndhwc_f16(const void* x, void* y, int N, int C, int T, int H, int W, int Cp, void* stream);
/* fp16 NDHWC (pitch Cp) -> fp32 NCDHW, for `features()` callers that want the reference layout. */
int b2_ndhwc_f16_to_ncdhw_f32(const void* x, float* y, int N, int C, int T, int H, int W, int Cp, void* stream);
/* y[r][c] = (relu ? max(x,0) : x) as fp16, rows x cols with pitches ldx / ldy; columns [cols, ldy) zeroed.
 * Used for the leading nn.ReLU of the TRN relation MLP (trn.py:40-41). */
int b2_cast_f32_to_f16(const float* x, int ldx, void* y, int ldy, int rows, int cols, int relu, void* stream);
/* Parameter-free type-A shortcut (resnet3D.py:65-74, nonlocalnet.py:322-332): spatial/temporal
 * subsampling by `stride` and zero-padding of channels [C, Cout). */
int b2_shortcut_a_ndhwc(const void* x, void* y, int N, int T, int H, int W, int C, int stride, int Cout,
                        void* stream);
/* y[r] = [a[r][0:Ca] | b[r][0:Cb] | 0]: torch.cat(dim=1) of two channels-last activations (SlowFast lateral
 * connections, slowfast.py:143-150, and its two-pathway head, slowfast.py:392).  Ca, Cb multiples of 8. */
int b2_concat_channels(const void* a, int lda, int Ca, const void* b, int ldb, int Cb, void* y, int ldy, long long rows,
                       void* stream);
/* y[n][j*F + f] = x[n][idx[j]][f]: frame-tuple gather of MultiScaleRelation (trn.py:108), fp16. */
int b2_gather_frames(const void* x, void* y, const int32_t* idx_dev, int N, int T, int F, int n_idx,
                     void* stream);
/* All tuples of one scale at once: y[n * n_tuples + t][j*F + f] = x[n][idx[t][j]][f], idx_dev int32 [n_tuples][n_idx] on the
 * device (one table for the whole forward, filled by a single host->device copy: trn.py:100-110 without a copy per tuple). */
int b2_gather_frame_tuples(const void* x, void* y, const int32_t* idx_dev, int N, int T, int F, int n_idx, int n_tuples,
                           void* stream);

/* ---------------------------------------------------------------------------------------------
 * MobileNetV2 (mobilenet.py:38-126)
 * ------------------------------------------------------------------------------------------- */
/* Depthwise 3x3 convolution (nn.Conv2d(C, C, 3, stride, 1, groups=C), mobilenet.py:50,64) -> BatchNorm -> ReLU6:
 *     y[n, ho, wo, c] = act( scale[c] * sum_{kh,kw} in(x[n, ho*s + kh - 1, wo*s + kw - 1, c]) * w[kh*3 + kw][c] + shift[c] )
 * with zero padding 1, in(v) = clamp_in ? min(v, 6) : v (the ReLU6 of the producer, which stored ReLU(v)) and
 * act = relu6 ? clamp to [0, 6] : identity.  fp32 accumulation in the fixed tap order (kh, kw), the affine in fp32, one fp16
 * rounding.  x: fp16 [N*H*W][ld] (N counts images: a clip's frames fold into it); y: fp16 [N*Ho*Wo][ld] with
 * Ho = (H - 1) / stride + 1 (same for W), channels [C, ld) written as zero; w: fp32 [9][C] (tap-major); scale, shift: fp32 [C].
 * C % 8 == 0, ld % 8 == 0, ld >= C, stride 1 or 2, every pointer 16-byte aligned. */
int b2_dwconv3x3_ndhwc(const void* x, const float* w, const float* scale, const float* shift, void* y, int N, int H, int W, int C,
                       int ld, int stride, int clamp_in, int relu6, void* stream);
/* x = min(max(x, 0), 6) in place over an fp16 [rows][ld] matrix: the ReLU6 of the last 1x1 convolution (mobilenet.py:30-35),
 * whose epilogue stored ReLU(x), ahead of the global average. */
int b2_relu6_inplace_ndhwc(void* x, long long rows, int ld, void* stream);

/* ---------------------------------------------------------------------------------------------
 * ResNeXt-3D (resnext3D.py:76-121)
 * ------------------------------------------------------------------------------------------- */
/* Grouped convolution (nn.Conv3d(C, C, 3, stride, 1, groups=32), conv2 of ResNeXtBottleneck, resnext3D.py:86-93) -> BatchNorm
 * -> (+residual) -> ReLU on wgmma at the grouped cost:
 *     y[m, k] = act( scale[k] * sum_{tap, c in group(k)} x[m @ tap, c] * w[k, c - first(group(k)), tap] + shift[k] + residual[m, k] )
 * Reads b2_conv_args as b2_conv_ndhwc_fprop does, with `w` the packed grouped filter below.  Contract: C == K (C is also the
 * channel pitch of x), C % 64 == 0, C / groups in {4, 8, 16, 32}, a 3x3x3 or 1x3x3 filter with padding (kt / 2, 1, 1), sh == sw
 * in {1, 2}, st in {1, 2}; anything else returns B2_ERR_UNSUPPORTED.  mode, out_f32, accumulate, aff_ld, upsample, residual_up,
 * residual_pre, y2 / scale2 / shift2 / aff2_ld, pool_w, in_scale / in_shift / in_aff_ld and mask / ldm must be zero / NULL
 * (B2_ERR_INVALID).  Columns [K, ldy) of y are left untouched.  fp32 accumulation in a fixed order, no atomics.
 * Executed multiply-accumulates over the algorithmic count: 4x for 4 channels per group, 2x for 8, 1x for 16 and 32 (the
 * block-diagonal dense filter through b2_conv_ndhwc_fprop: `groups` x).
 *
 * Packed filter: fp32 [K][Cin_per_group][kt][kh][kw] (nn.Conv3d.weight of the grouped layer) -> fp16 [K / 64][taps][G][64] with
 * G = 16 (G = 32 for 32 channels per group), K * G * taps elements: row r, 16-element segment j of a (64-channel slice, tap)
 * tile is output channel 16 j + r (G = 32: 32 (j / 2) + r) of the slice against its input channels [16 j, 16 j + 16), zero where
 * the two channels belong to different groups.  b2_pack_grouped_conv_weight_elems is host arithmetic and returns 0 for a filter
 * outside the contract. */
size_t b2_pack_grouped_conv_weight_elems(int K, int Cin_per_group, int groups, int kt, int kh, int kw);
int b2_pack_grouped_conv_weight(const float* w, void* w_packed, int K, int Cin_per_group, int groups, int kt, int kh, int kw,
                                void* stream);
int b2_conv_grouped_ndhwc_fprop(const b2_conv_args* a, int groups, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Fine-tuning backward of the residual blocks (the backward of resnet3D.py:91-143 with eval-mode BatchNorm).  Gradients
 * travel between kernels as fp16 NDHWC matrices multiplied by a device-resident power-of-two loss scale; the fp32 results
 * (weight, gamma and beta gradients) divide it out.  `inv_loss_scale` / `scale_pair` are DEVICE pointers.
 * ------------------------------------------------------------------------------------------- */
/* Weight gradient of a k x k x k convolution (k = 1, padding 0, or k = 3, padding 1; stride 1 or 2) on wgmma:
 *     G[co][ci][tap] = sum over output positions p of g[p][co] * x[stride * p + tap - pad][ci]
 *     dw[co][ci][tap] = scale[co] * G * inv_loss_scale      (fp32, nn.Conv3d.weight layout [Cout][Cin][k][k][k])
 *     wdot[co]        = sum_{ci,tap} w[co][ci][tap] * G * inv_loss_scale      (nullable; needs w, fp32 same layout)
 * g: fp16 [N*To*Ho*Wo][ldg] (gradient at the convolution output), x: fp16 [N*T*H*W][ldx] (its input).  scale and
 * inv_loss_scale nullable (= 1).  ws: fp32 workspace of b2_conv_wgrad_workspace_elems(...) elements; the result does not
 * depend on how the position sum is split (fixed-order reduction, no atomics). */
size_t b2_conv_wgrad_workspace_elems(int N, int T, int H, int W, int Cin, int Cout, int k, int stride, int pad);
int b2_conv_wgrad(const void* g, int ldg, const void* x, int ldx, const float* w, const float* scale, const float* inv_loss_scale,
                  float* dw, float* wdot, float* ws, size_t ws_elems, int N, int T, int H, int W, int Cin, int Cout, int k,
                  int stride, int pad, void* stream);
/* The same for a kt x kh x kw filter with separate temporal and in-plane geometry (kt, kh = kw in {1, 3}; padding pt = kt / 2,
 * p = kh / 2; strides st, s in {1, 2}):
 *     G[co][ci][dt][dh][dw] = sum over output positions (n, t, h, w) of g[n, t, h, w][co] * x[n, st*t+dt-pt, s*h+dh-p, s*w+dw-p][ci]
 * dw is fp32 [Cout][Cin][kt][kh][kw]; a 2-D filter is the (1, kh, kw) case with T = 1, whose dw is nn.Conv2d.weight's layout.
 * b2_conv_wgrad(..., k, stride, pad) computes bitwise the same as this entry with (k, k, k, stride, stride, pad, pad). */
size_t b2_conv_wgrad_thw_workspace_elems(int N, int T, int H, int W, int Cin, int Cout, int kt, int kh, int kw, int st, int s,
                                         int pt, int p);
int b2_conv_wgrad_thw(const void* g, int ldg, const void* x, int ldx, const float* w, const float* scale, const float* inv_loss_scale,
                      float* dw, float* wdot, float* ws, size_t ws_elems, int N, int T, int H, int W, int Cin, int Cout, int kt,
                      int kh, int kw, int st, int s, int pt, int p, void* stream);
/* Adjoint of b2_shortcut_a_ndhwc: y[n, s*to, s*ho, s*wo, 0:C] = g[n, to, ho, wo, 0:C] for the low-resolution extent
 * To = (T-1)/s + 1 (etc.), every other pixel and channels [C, ldy) zero; y is [N*T*H*W][ldy].  The backward of the type-A
 * shortcut, the placement of the type-B projection gradient, and the zero-insertion that turns the input gradient of a
 * stride-2 3x3x3 convolution into a stride-1 convolution with the flipped filter. */
int b2_zero_insert_ndhwc(const void* g, int ldg, int C, void* y, int ldy, int N, int T, int H, int W, int stride, void* stream);
/* out[c] = inv_loss_scale * sum_r g[r][c] (fp32, fixed-order two-pass reduction; ws: b2_colsum_workspace_elems(C) floats). */
size_t b2_colsum_workspace_elems(int C);
int b2_colsum_f16(const void* g, int ldg, long long rows, int C, const float* inv_loss_scale, float* out, float* ws, void* stream);
/* scale_pair = [2^k, 2^-k] with max |g| * 2^k in [2^7, 2^8), |k| <= 126 (k = 0 when g is all zero or has a non-finite entry). */
int b2_loss_scale_f32(const float* g, int rows, int cols, int ldg, float* scale_pair, void* stream);
/* Backward of b2_avgpool_global_ndhwc followed by the block's closing ReLU: y[n*S + p][c] = fp16(gf[n][c] * scale_pair[0] / S)
 * where out[n*S + p][c] > 0, else 0 (channels [C, ld) zero).  gf fp32 [N][ldf]; out, y fp16 [N*S][ld]. */
int b2_avgpool_global_backward(const float* gf, int ldf, const float* scale_pair, const void* out, void* y, int N, int S, int C,
                               int ld, void* stream);

/* ---------------------------------------------------------------------------------------------
 * Image preprocessing on the device -- TransformImage (pretorched/transforms/utils.py:34-81; used by
 * examples/imagenet_logits.py:38-43): transforms.Resize (Pillow 8-bit BILINEAR: horizontal pass then vertical pass,
 * 22-bit fixed-point coefficients, each pass rounds to uint8) -> Center/RandomCrop -> flips -> ToTensor -> ToSpaceBGR ->
 * ToRange255 -> Normalize, bit-exact with the Pillow + torchvision pipeline the reference composes.
 *   img       uint8 [H][W][3] RGB on the device
 *   hbounds/hk  int32 [Wr][2] (first source column, count) and [Wr][hksize] coefficients of the horizontal pass (null when Wr == W)
 *   vbounds/vk  the same for the vertical pass to Hr rows (null when Hr == H);  tmp: uint8 [H][Wr][3] scratch (horizontal result)
 *   top/left/crop_h/crop_w  crop window inside the resized [Hr][Wr] image
 *   flags     bit 0 horizontal flip, bit 1 vertical flip, bit 2 BGR, bit 3 range 255
 *   mean/stdv HOST pointers to 3 floats each
 *   out_f32   nullable fp32 [3][crop_h][crop_w] (what the reference returns); out_h4: nullable fp16 [crop_h*crop_w][4]
 *             (NDHWC4: the stem convolution's input layout, channel 3 zero)
 * ------------------------------------------------------------------------------------------- */
/* Decoded video frames, uint8 [N*T*H*W][3] (channels last, RGB) -> the stem's fp16 NDHWC4 input with ToTensor (/255), ToSpaceBGR,
 * ToRange255 and Normalize applied per pixel (the per-frame tail of TransformImage, transforms/utils.py:72-75, for clips that are
 * already at network resolution): a clip crosses PCIe as 3 bytes per pixel instead of 12.  flags: bit 2 BGR, bit 3 range 255;
 * mean / stdv: HOST pointers to 3 floats. */
int b2_u8_frames_to_ndhwc4_f16(const uint8_t* frames, void* y, long long pixels, int flags, const float* mean, const float* stdv,
                               void* stream);
int b2_transform_image_u8(const uint8_t* img, int H, int W, const int32_t* hbounds, const int32_t* hk, int hksize, int Wr,
                          const int32_t* vbounds, const int32_t* vk, int vksize, int Hr, uint8_t* tmp, int top, int left,
                          int crop_h, int crop_w, int flags, const float* mean, const float* stdv, float* out_f32,
                          void* out_h4, void* stream);

/* ---------------------------------------------------------------------------------------------
 * BigGAN-deep generator helpers (BASELINE.json configs[4]).  The architecture is NOT in the reference tree
 * (SURVEY.md section 8a row a14): these replace the F.batch_norm * (1 + gain(y)) + bias(y) -> ReLU ->
 * F.interpolate(scale_factor=2) chain of the published GBlock, its embedding lookup + torch.cat, and the final
 * torch.tanh; see oracle/biggan.py for the restatement they are checked against.
 * ------------------------------------------------------------------------------------------- */
/* v[b] = [ (embedded ? embedded[b] : table[labels[b]]) (ds) | z[b] (dz) | 0 ], D = round_up(ds + dz, 8) entries.
 * split == 0: y[b] = fp16(v), pitch ldy >= D.  split != 0: y[b] = [ hi | lo | hi ] (hi = fp16(v), lo = fp16(v - hi)),
 * pitch ldy >= 3 * D -- the A operand of an fp16 GEMM against [ W_hi | W_hi | W_lo ] that reproduces v . W to ~fp32
 * accuracy.  z, table, embedded fp32; labels int64 (clamped to [0, n_classes)). */
int b2_embed_concat(const float* z, const long long* labels, const float* table, const float* embedded, void* y, int B,
                    int dz, int ds, int n_classes, int ldy, int split, void* stream);
/* y[n, up*h+i, up*w+j, c] = act(x[n,h,w,c] * scale[n*lda + c] + shift[n*lda + c]) for c < C, i,j < up (up = 1 or 2,
 * nearest-neighbour upsampling); channels [C, ldy) written as zero.  scale/shift fp32 [N][lda] (lda = 0: one row shared
 * by all samples, i.e. a plain BatchNorm), or both NULL for a pure copy / channel slice / upsample. */
int b2_ccbn_act_ndhwc(const void* x, int ldx, void* y, int ldy, const float* scale, const float* shift, int lda, int N,
                      int H, int W, int C, int up, int relu, void* stream);
/* RGB head of the generator (3x3 convolution to K <= 4 channels, + bias, tanh, NCHW write) split in two: a 1x1 GEMM
 * (b2_gemm_f16) writes partial[q][(dh*3+dw)*4 + k] = sum_c x[q][c] * w[k][c][dh][dw] for every pixel q (36 columns, pitch
 * ldp >= 36), and this call gathers y[n][k][h][w] = tanh(bias[k] + sum_taps partial[(n,h+dh-1,w+dw-1)][tap*4 + k]) with
 * zero padding.  One pass of the tensor core over x instead of nine shifted passes that use 3 of 16 MMA columns. */
int b2_rgb_head_gather_tanh(const void* partial, int ldp, const float* bias, void* y, int N, int H, int W, int K, int out_f32,
                            void* stream);
/* y[n][c][s] = tanh(x[n*S + s][c]): fp16 channels-last (pitch ldx) -> NCHW planes, fp32 (out_f32) or fp16. */
int b2_tanh_nhwc_to_nchw(const void* x, int ldx, void* y, int N, int C, long long S, int out_f32, void* stream);

/* ---------------------------------------------------------------------------------------------
 * SE-ResNet / SE-ResNeXt (senet.py:85-204)
 * ------------------------------------------------------------------------------------------- */
/* Squeeze-and-excitation of one SE bottleneck as per-sample affine rows for b2_gemm_sample_affine_f16.  SEModule
 * (senet.py:85-104) scales x = bn3(conv3(h2)) by e = sigmoid(fc2(relu(fc1(avgpool(x))))); conv3 + bn3 is affine, so
 * avgpool(x) = s3 * (W3 . m) + t3 with m the mean of h2 over the positions of a sample, and the caller passes fc1 composed with
 * that map: w1 = W_fc1 . diag(s3) . W3 (fp32 [R][C2]), b1 = W_fc1 . t3 + b_fc1 (fp32 [R]).  Per sample n:
 *     m[c]   = sum_p h[n*S + p][c] / S                 (fp32)
 *     a[r]   = relu(sum_c w1[r][c] m[c] + b1[r])
 *     e[k]   = sigmoid(sum_r w2[k][r] a[r] + b2[k])    (w2 fp32 [C][R] = fc2.weight, b2 = fc2.bias)
 *     scale[n * ld_aff + k] = e[k] * s3[k],  shift[n * ld_aff + k] = e[k] * t3[k]      (k < C; columns >= C untouched)
 * so that relu(scale * (W3 . h2) + shift + residual) is the block output (senet.py:127-131).  h: fp16 [N*S][ldh], C2 % 8 == 0,
 * ldh % 8 == 0, 16-byte aligned.  ws: fp32 workspace of b2_se_excite_workspace_elems(N, C2, R) elements.  Three launches, fp32
 * throughout, every sum in one fixed order (no atomics): bitwise repeatable, no host synchronisation. */
size_t b2_se_excite_workspace_elems(int N, int C2, int R);
int b2_se_excite(const void* h, int ldh, int N, int S, int C2, const float* w1, const float* b1, int R, const float* w2, const float* b2,
                 int C, const float* s3, const float* t3, float* scale, float* shift, int ld_aff, float* ws, size_t ws_elems,
                 void* stream);

/* ---------------------------------------------------------------------------------------------
 * BNInception (bninception.py:27-495): inception branches written in place into the concatenated block output
 * ------------------------------------------------------------------------------------------- */
/* Column-slice destinations.  A destination (y, ldy, cols) is columns [0, cols) of the rows of pitch ldy that start at y: y is
 * the first column of the slice inside a wider row (16-byte aligned), cols % 8 == 0, ldy % 8 == 0, ldy >= cols.  The entries below
 * write exactly those columns and leave every other column of the row untouched, so the branches of an inception block
 * (torch.cat at bninception.py:288, 311, 328, 351, 374, 397, 420, 437, 460, 483) land in their slices of one [M][out] matrix. */

/* Packed layout of a split GEMM: destination d owns the 64-column store boxes [box0[d], box0[d + 1]) of the packed B / affine,
 * box0[0] = 0, box0[d + 1] = box0[d] + ceil(cols[d] / 64).  Returns the packed width 64 * box0[nd], or B2_ERR_INVALID (1 <= nd <= 4,
 * cols[d] > 0 and cols[d] % 8 == 0).  Host only. */
int b2_gemm_split_plan(int nd, const int* cols, int* box0);
/* One GEMM, up to four column-slice destinations (the 1x1 heads of an inception block that read the same input, bninception.py:266-275):
 *     D[m][n] = act(scale[n] * (A . B^T)[m][n] + shift[n]),  n < N = b2_gemm_split_plan(nd, cols)
 * packed column 64 * box0[d] + j (j < cols[d]) is column j of destination d; B rows / affine entries of the padding columns (j >= cols[d]
 * inside a destination's last box) are computed and dropped.  g: a, lda, b, ldb, Kd, M, N, scale, shift, relu as in b2_gemm_f16;
 * d, ldd, residual, out_f32, per_row, accumulate, aff_ld, d2 and mask must be zero (B2_ERR_INVALID).  Always the persistent GEMM
 * (b2_debug_last_kernel: KID 12, info = {N tile, nd, N}) with the N tile b2_gemm_f16 picks for an N-wide output (64 for N <= 64, else
 * 128): with the same N tile each destination equals the stand-alone b2_gemm_f16 of its rows of B bit for bit. */
int b2_gemm_split_f16(const b2_gemm_args* g, int nd, void* const* y, const int* ldy, const int* cols, void* stream);
/* b2_conv_ndhwc_fprop with y a column slice (y, ldy, K) as above: columns [0, K) of each output row are written, K % 8 == 0, the rest
 * of the row is untouched.  2-D convolutions (kt = 1) with an odd kh x kw filter other than 1x1 (3x3, 1x3, 3x1, 1x7, 7x1, 5x5 ...),
 * in-plane padding from 0 ("valid") to (k - 1) / 2 ("same") per axis, stride 1 or 2, on the slab kernel only
 * (b2_debug_last_kernel: KID 13).  Stem mode, mask, per-sample affine, upsampling, second output, pool_w, the generator fields and fp32
 * output are refused (B2_ERR_INVALID); B2_ERR_UNSUPPORTED when no slab tiling of the image fits. */
int b2_conv_ndhwc_fprop_slice(const b2_conv_args* a, void* stream);
/* b2_conv_ndhwc_fprop_slice with one N tile exactly K = 32 or 48 columns wide (one m64n32k16 / m64n48k16 per K step, positions along
 * M) instead of the 64-wide tile that pads those widths: the growth-rate 3x3 convolutions of DenseNet's dense layers.  Same contract
 * as b2_conv_ndhwc_fprop_slice, plus K in {32, 48} (B2_ERR_INVALID).  Each output element is accumulated in the same order as on the
 * 64-wide tile and goes through the same epilogue.  b2_debug_last_kernel: KID 13, info = {K, MT, 1, wchunks}. */
int b2_conv_ndhwc_fprop_slice_narrow(const b2_conv_args* a, void* stream);
/* Pooling between column slices: x is [N*T*H*W] rows of pitch ldx (channels [0, C) read), y is a slice (y, ldy, C) of rows
 * [N*To*Ho*Wo] with the output extent given by the caller (ceil mode).  avg = 0: max (nn.MaxPool2d, padding taps skipped);
 * avg = 1: nn.AvgPool2d(count_include_pad=True) -- fp32 sum in a fixed tap order, divided by the window clipped to the padded input,
 * one fp16 rounding.  The 3x3 stride-1 pools of the pool branches (bninception.py:61, :247) and the stride-2 ceil-mode pools whose
 * output is a block's pass-through slice (:102, :206).  Every window must start inside the input or its left padding, padding <= half
 * the window (B2_ERR_INVALID).  b2_debug_last_kernel: KID 14, info = {avg}. */
int b2_pool_ndhwc_slice(const void* x, int ldx, void* y, int ldy, int N, int T, int H, int W, int C, int kt, int kh, int kw, int st, int sh,
                        int sw, int pt, int ph, int pw, int To, int Ho, int Wo, int avg, void* stream);
/* b2_pool_ndhwc_slice's average with count_include_pad=False (nn.AvgPool2d(3, 1, 1, count_include_pad=False), the pool branches of
 * inceptionv4.py:124, :180, :238 and inceptionresnetv2.py:73): fp32 sum over the in-input taps in (dt, dh, dw) order, divided by
 * their number, one fp16 rounding.  Same argument contract as b2_pool_ndhwc_slice (every window overlaps the input).
 * b2_debug_last_kernel: KID 14, info = {2}. */
int b2_avgpool_ndhwc_slice_exclude_pad(const void* x, int ldx, void* y, int ldy, int N, int T, int H, int W, int C, int kt, int kh, int kw,
                                       int st, int sh, int sw, int pt, int ph, int pw, int To, int Ho, int Wo, void* stream);

/* ---------------------------------------------------------------------------------------------
 * DenseNet (torchvision densenet.py, wrapped by torchvision_models.py:254-380)
 * ------------------------------------------------------------------------------------------- */
/* The 1x1 convolution of a dense layer with its pre-activation applied to the A operand on chip:
 *     D[m][n] = act(scale[n] * sum_k relu(in_scale[k] * A[m][k] + in_shift[k]) * B[n][k] + shift[n])
 * A is the first Kd columns of the dense block's matrix (pitch lda, any Kd % 8 == 0): columns >= Kd are never read -- the A and
 * B tensor maps span Kd columns and TMA zero-fills the rest of the last 64-column K block -- so in_scale / in_shift must be
 * 16-byte aligned fp32 arrays of round_up(Kd, 64) entries that are ZERO past Kd (relu(0 * 0 + 0) = 0), and B zero there.  The
 * transformed operand is rounded to fp16 once before the MMA.  g: as b2_gemm_f16 with fp16 output (columns [N, ldd) written
 * as zero); residual, per_row, out_f32, accumulate, aff_ld, d2 and mask must be zero (B2_ERR_INVALID).  Always the persistent
 * GEMM's generator instance (b2_debug_last_kernel: KID 6, info = {N tile, 0, 1}). */
int b2_gemm_preact_f16(const b2_gemm_args* g, const float* in_scale, const float* in_shift, void* stream);
/* A dense transition's BatchNorm + ReLU + AvgPool2d(2, 2) (densenet.py _Transition, pooled before its 1x1 convolution):
 *     y[n][ho][wo][c] = fp16(sum_{dh, dw < 2} relu(scale[c] * x[n][2 ho + dh][2 wo + dw][c] + shift[c]) / 4)
 * fp32 sum in (dh, dw) order, one rounding; Ho = H / 2, Wo = W / 2 (floor: an odd last row / column is dropped, as nn.AvgPool2d).
 * x: rows of pitch ldx (channels [0, C) read), y: a slice (y, ldy, C).  C, ldx, ldy multiples of 8, x / y 16-byte aligned, scale /
 * shift fp32 [C].  b2_debug_last_kernel: KID 14, info = {3}. */
int b2_bn_relu_avgpool2_ndhwc(const void* x, int ldx, void* y, int ldy, int N, int H, int W, int C, const float* scale, const float* shift,
                              void* stream);
/* b2_avgpool_global_ndhwc with relu(scale[c] * x + shift[c]) applied to every element before the sum (DenseNet's norm5 + ReLU +
 * 7x7 mean, torchvision_models.py:262-264): fp32 accumulation, one fp16 rounding.  scale / shift fp32 [C].
 * b2_debug_last_kernel: KID 14, info = {4}. */
int b2_avgpool_global_affine_ndhwc(const void* x, void* y, int N, int S, int C, const float* scale, const float* shift, void* stream);

/* ---------------------------------------------------------------------------------------------
 * VGG / AlexNet (torchvision vgg.py / alexnet.py behind torchvision_models.py:195-248, 597-725)
 * ------------------------------------------------------------------------------------------- */
/* AlexNet's first convolution (nn.Conv2d(3, 64, 11, stride=4, padding=2)) as a valid 3x3 stride-1 convolution over a 4x4
 * space-to-depth image: x fp32 NCHW [N][3][H][W] -> y fp16 [N*Hs*Ws][48] with Ho = (H + 4 - 11) / 4 + 1, Hs = Ho + 2 (same for W),
 *     y[(n, hs, ws)][(dh * 4 + dw) * 3 + c] = x[n][c][4 hs + dh - 2][4 ws + dw - 2]      (0 outside the image)
 * so that conv11x11/4(x)[ho][wo] = sum_{a, b < 3} y[ho + a][wo + b] . W3[a][b] with W3[k][(dh * 4 + dw) * 3 + c][a][b] =
 * W[k][c][4 a + dh][4 b + dw] (zero where 4 a + dh or 4 b + dw reaches 11).  One rounding to fp16 per element.  H, W >= 7, y 16-byte
 * aligned.  Replaces the layout pass of the generic input path for this network. */
int b2_space_to_depth4_nchw(const float* x, void* y, int N, int H, int W, void* stream);
/* Split-K GEMM for the fully connected classifiers (torchvision_models.py:211-224, 613-626), whose M is the batch:
 *     D[M][N] = act(scale[n] * sum_{s < S} P_s[m][n] + shift[n]),   P_s = A[:, K_s] . B[:, K_s]^T over K blocks
 *                                                                 K_s = [s * nkb / S, (s + 1) * nkb / S) of 64 (nkb = ceil(Kd / 64))
 * One persistent-GEMM launch writes every P_s in fp32 into its own slice of the caller's workspace ws ([S][M][round_up(N, 8)] floats,
 * b2_gemm_splitk_workspace_elems), then one pass sums the slices in the order 0..S-1, applies the per-column affine, the ReLU
 * (g->relu) and writes fp16 (columns [N, ldd) zero) or fp32 (g->out_f32, ldd >= N, only columns [0, N) written).  No atomics: the
 * result is bitwise repeatable, and the same under CUDA-graph replay.  g: a, lda, b, ldb, M, N, Kd, scale, shift, d, ldd, relu,
 * out_f32 as in b2_gemm_f16; a residual, a mask, per_row, a per-sample affine (aff_ld / aff_rows), a second output (d2 / scale2 /
 * shift2 / aff2_*) and accumulate are refused (B2_ERR_INVALID), as is 1 > S or S > min(64, nkb).  Two launches;
 * b2_debug_last_kernel: KID 17, info = {N tile, S}, with the N tile b2_gemm_f16 picks for an output of pitch round_up(N, 8). */
size_t b2_gemm_splitk_workspace_elems(int M, int N, int splits);
int b2_gemm_splitk_f16(const b2_gemm_args* g, int splits, float* ws, size_t ws_elems, void* stream);
/* The number of splits S for an M x N x Kd product on `sm_count` SMs: 1 when the output tiles (128 rows x the N tile) fill the SMs,
 * else SMs / tiles, capped so that every split keeps at least 8 K blocks of 64 and at 16 splits; at least 1.  Host only. */
int b2_gemm_splitk_plan(int M, int N, int Kd, int sm_count);

#ifdef __cplusplus
}
#endif
#endif /* B2_PRETORCHED_H_ */
