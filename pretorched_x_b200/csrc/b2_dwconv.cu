// b2_dwconv.cu -- depthwise 3x3 convolution (groups = channels, padding 1, stride 1 or 2) with the folded BatchNorm and ReLU6
// of MobileNetV2's inverted residuals (mobilenet.py:48-70), and the in-place ReLU6 of its last 1x1 convolution.
//
// A depthwise 3x3 does 9 MACs per output element: far below the H100's ridge point, so this is a CUDA-core kernel bound by
// HBM bandwidth.  One thread owns 8 channels (one 16-byte vector, channel index fastest across the warp) of R consecutive
// output columns of one output row.  It walks the three input rows of its window; in each row it loads the
// (R - 1) * stride + 3 input columns once and feeds every output column that reads them, so within a thread each input
// vector is loaded once per row instead of once per tap.  The remaining halo overlap (the two rows shared with the output
// rows above and below, and the edge columns shared with the neighbouring run) is served by L1 / L2: each input byte
// comes from HBM once.  Every output element accumulates its taps in the fixed order (kh, kw) in fp32; the folded BN
// affine and the clamp run in fp32 before the single fp16 rounding.
//
// The RELU_IN instance is the depthwise half of Xception's separable convolutions (xception.py:50-60, 93-112): it reads
// max(x, 0) and has no affine and no activation (the BatchNorm follows the pointwise 1x1, in its GEMM epilogue), so it rounds
// the fp32 tap sum itself.  Xception needs the ReLU on load because a block's input is the signed residual sum, which the
// skip path reads raw.
//
// The K x K instances (K = 3, 5, 7; b2_dwconv_kxk_relu_in_ndhwc) are the depthwise halves of PNASNet-5's separable branches
// (pnasnet.py:49-97): the same tile (dwconv_tile) on max(x, 0), with a top / left padding and the output extent given by the caller,
// separate input and output pitches, and only the C channels of a column slice written.  A branch that opens with ZeroPad2d((1, 0,
// 1, 0)) and crops [1:, 1:] after its strided convolution (cell_4) is the same convolution at padding K / 2 - 1 with the ceil
// extent.  dwconv3x3_kernel keeps its own symbol, so the existing entries' instances, launch records and outputs are unchanged.
#include "b2_host.h"

#include <cuda_fp16.h>

namespace b2 {

static inline int div_up(long long a, long long b) { return (int)((a + b - 1) / b); }

__device__ __forceinline__ void unpack8(const uint4& v, float* f) {
  const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 p = __half22float2(h[i]);
    f[2 * i] = p.x;
    f[2 * i + 1] = p.y;
  }
}

__device__ __forceinline__ uint4 pack8(const float* f) {
  uint4 v;
  __half2* h = reinterpret_cast<__half2*>(&v);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
  return v;
}

// The depthwise tile one thread computes: 8 channels (vector c8) of R consecutive output columns (from wo0) of output row ho of
// image n, for a K x K filter of stride S whose window starts `pad` rows / columns before the input (top / left); taps outside
// the map read zero.  x: fp16 rows of ldx8 vectors; w: fp32 [K*K][C] (tap-major).  In each of the K window rows the run reads
// its J = (R - 1) * S + K input columns once and feeds every output column that reads them; every output element accumulates
// its taps in the fixed order (kh, kw) in fp32.  RELU_IN reads max(x, 0), clamp_in min(x, 6).
template <int K, int S, int R, bool RELU_IN>
__device__ __forceinline__ void dwconv_tile(const uint4* __restrict__ x, const float* __restrict__ w, long long n, int ho, int wo0,
                                            int c8, int H, int W, int C, int ldx8, int pad, int clamp_in, float (&acc)[R][8]) {
  constexpr int J = (R - 1) * S + K;
#pragma unroll
  for (int r = 0; r < R; ++r)
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[r][e] = 0.f;

  const int wi0 = wo0 * S - pad;
#pragma unroll
  for (int kh = 0; kh < K; ++kh) {
    const int hi = ho * S - pad + kh;
    if (hi < 0 || hi >= H) continue;                    // zero padding row: adds nothing
    float wk[K][8];
#pragma unroll
    for (int kw = 0; kw < K; ++kw) {
      const float4* wp = reinterpret_cast<const float4*>(w + (long long)(kh * K + kw) * C + c8 * 8);
      const float4 a = __ldg(wp), b = __ldg(wp + 1);
      wk[kw][0] = a.x; wk[kw][1] = a.y; wk[kw][2] = a.z; wk[kw][3] = a.w;
      wk[kw][4] = b.x; wk[kw][5] = b.y; wk[kw][6] = b.z; wk[kw][7] = b.w;
    }
    const uint4* xrow = x + ((n * H + hi) * (long long)W) * ldx8 + c8;
#pragma unroll
    for (int j = 0; j < J; ++j) {
      const int wi = wi0 + j;
      if (wi < 0 || wi >= W) continue;                  // zero padding column
      float xv[8];
      unpack8(__ldg(xrow + (long long)wi * ldx8), xv);
      if constexpr (RELU_IN) {
#pragma unroll
        for (int e = 0; e < 8; ++e) xv[e] = fmaxf(xv[e], 0.f);
      } else if (clamp_in) {
#pragma unroll
        for (int e = 0; e < 8; ++e) xv[e] = fminf(xv[e], 6.f);
      }
#pragma unroll
      for (int r = 0; r < R; ++r) {
        const int kw = j - r * S;                       // this column is tap kw of output column wo0 + r
        if (kw < 0 || kw >= K) continue;
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[r][e] = fmaf(xv[e], wk[kw][e], acc[r][e]);
      }
    }
  }
}

// x, y: fp16 [N*H*W][ld] resp. [N*Ho*Wo][ld] as uint4 (ld8 = ld / 8 vectors per pixel); w: fp32 [9][C] (tap-major);
// scale / shift: fp32 [C] (unused by RELU_IN).  Thread i -> (n, ho, run of R output columns, 8-channel group), channel group
// fastest.  The 3x3 padding-1 instance of dwconv_tile.
template <int S, int R, bool RELU_IN>
__global__ void __launch_bounds__(256) dwconv3x3_kernel(const uint4* __restrict__ x, const float* __restrict__ w,
                                                         const float* __restrict__ scale, const float* __restrict__ shift,
                                                         uint4* __restrict__ y, int H, int W, int Ho, int Wo, int runs, int C8,
                                                         int ld8, int clamp_in, int relu6, long long total) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c8 = (int)(i % ld8);
  long long q = i / ld8;
  const int run = (int)(q % runs); q /= runs;
  const int ho = (int)(q % Ho);
  const long long n = q / Ho;
  const int wo0 = run * R;
  const long long orow = (n * Ho + ho) * Wo;
  if (c8 >= C8) {                                       // padding channels [C, ld) are written as zero
#pragma unroll
    for (int r = 0; r < R; ++r)
      if (wo0 + r < Wo) y[(orow + wo0 + r) * ld8 + c8] = make_uint4(0, 0, 0, 0);
    return;
  }
  float acc[R][8];
  dwconv_tile<3, S, R, RELU_IN>(x, w, n, ho, wo0, c8, H, W, C8 * 8, ld8, 1, clamp_in, acc);

  if constexpr (RELU_IN) {
#pragma unroll
    for (int r = 0; r < R; ++r)
      if (wo0 + r < Wo) y[(orow + wo0 + r) * ld8 + c8] = pack8(acc[r]);
    return;
  }
  float sc[8], sh[8];
  {
    const float4* sp = reinterpret_cast<const float4*>(scale + c8 * 8);
    const float4* hp = reinterpret_cast<const float4*>(shift + c8 * 8);
    const float4 s0 = __ldg(sp), s1 = __ldg(sp + 1), h0 = __ldg(hp), h1 = __ldg(hp + 1);
    sc[0] = s0.x; sc[1] = s0.y; sc[2] = s0.z; sc[3] = s0.w; sc[4] = s1.x; sc[5] = s1.y; sc[6] = s1.z; sc[7] = s1.w;
    sh[0] = h0.x; sh[1] = h0.y; sh[2] = h0.z; sh[3] = h0.w; sh[4] = h1.x; sh[5] = h1.y; sh[6] = h1.z; sh[7] = h1.w;
  }
#pragma unroll
  for (int r = 0; r < R; ++r) {
    if (wo0 + r >= Wo) break;
    float v[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      v[e] = fmaf(acc[r][e], sc[e], sh[e]);
      if (relu6) v[e] = fminf(fmaxf(v[e], 0.f), 6.f);
    }
    y[(orow + wo0 + r) * ld8 + c8] = pack8(v);
  }
}

// The K x K instance of dwconv_tile on max(x, 0), no affine (b2_dwconv_kxk_relu_in_ndhwc): x rows of pitch ldx8 vectors, y the
// column slice (y, ldy8, C) of rows [N*Ho*Wo] -- only channel groups [0, C8) are written.  Thread i -> (n, ho, run, c8), c8 fastest.
template <int K, int S, int R>
__global__ void __launch_bounds__(256) dwconv_kxk_kernel(const uint4* __restrict__ x, const float* __restrict__ w,
                                                          uint4* __restrict__ y, int H, int W, int Ho, int Wo, int runs, int C8,
                                                          int ldx8, int ldy8, int pad, long long total) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c8 = (int)(i % C8);
  long long q = i / C8;
  const int run = (int)(q % runs); q /= runs;
  const int ho = (int)(q % Ho);
  const long long n = q / Ho;
  const int wo0 = run * R;
  const long long orow = (n * Ho + ho) * Wo;
  float acc[R][8];
  dwconv_tile<K, S, R, true>(x, w, n, ho, wo0, c8, H, W, C8 * 8, ldx8, pad, 0, acc);
#pragma unroll
  for (int r = 0; r < R; ++r)
    if (wo0 + r < Wo) y[(orow + wo0 + r) * ldy8 + c8] = pack8(acc[r]);
}

// x = min(max(x, 0), 6) over an fp16 matrix of `vecs` 16-byte vectors (zero padding channels stay zero)
__global__ void relu6_inplace_kernel(uint4* __restrict__ x, long long vecs) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= vecs) return;
  uint4 v = x[i];
  __half2* h = reinterpret_cast<__half2*>(&v);
  const __half2 lo = __float2half2_rn(0.f), hi = __float2half2_rn(6.f);
#pragma unroll
  for (int e = 0; e < 4; ++e) h[e] = __hmin2(__hmax2(h[e], lo), hi);
  x[i] = v;
}

template <int S, int R, bool RELU_IN = false>
static int launch_dwconv(const void* x, const float* w, const float* scale, const float* shift, void* y, int N, int H, int W,
                         int C, int ld, int clamp_in, int relu6, cudaStream_t stream) {
  const int Ho = (H - 1) / S + 1, Wo = (W - 1) / S + 1;
  const int runs = (Wo + R - 1) / R;
  const long long total = (long long)N * Ho * runs * (ld / 8);
  dwconv3x3_kernel<S, R, RELU_IN><<<div_up(total, 256), 256, 0, stream>>>(reinterpret_cast<const uint4*>(x), w, scale, shift,
                                                                          reinterpret_cast<uint4*>(y), H, W, Ho, Wo, runs, C / 8,
                                                                          ld / 8, clamp_in, relu6, total);
  B2_CHECK_LAUNCH("dwconv3x3_kernel");
  return B2_OK;
}

template <int K, int S, int R>
static int launch_dwconv_kxk(const void* x, int ldx, const float* w, void* y, int ldy, int N, int H, int W, int C, int pad, int Ho,
                             int Wo, cudaStream_t stream) {
  const int runs = (Wo + R - 1) / R;
  const long long total = (long long)N * Ho * runs * (C / 8);
  dwconv_kxk_kernel<K, S, R><<<div_up(total, 256), 256, 0, stream>>>(reinterpret_cast<const uint4*>(x), w, reinterpret_cast<uint4*>(y),
                                                                      H, W, Ho, Wo, runs, C / 8, ldx / 8, ldy / 8, pad, total);
  B2_CHECK_LAUNCH("dwconv_kxk_kernel");
  return B2_OK;
}

// Output columns per thread of the K x K instances: 2 at stride 2; at stride 1, 6 for K = 3 (at 4, ptxas spills 4 bytes of that
// instance) and 4 for K = 5, 7.  No instance spills (register counts in DESIGN section 3).
constexpr int kxk_run(int K, int S) { return S == 2 ? 2 : (K == 3 ? 6 : 4); }

template <int K>
static int launch_dwconv_kxk_k(const void* x, int ldx, const float* w, void* y, int ldy, int N, int H, int W, int C, int stride, int pad,
                               int Ho, int Wo, cudaStream_t st) {
  return stride == 1 ? launch_dwconv_kxk<K, 1, kxk_run(K, 1)>(x, ldx, w, y, ldy, N, H, W, C, pad, Ho, Wo, st)
                     : launch_dwconv_kxk<K, 2, kxk_run(K, 2)>(x, ldx, w, y, ldy, N, H, W, C, pad, Ho, Wo, st);
}

}  // namespace b2

using namespace b2;

extern "C" {

int b2_dwconv3x3_ndhwc(const void* x, const float* w, const float* scale, const float* shift, void* y, int N, int H, int W, int C,
                       int ld, int stride, int clamp_in, int relu6, void* stream) {
  B2_CHECK_ARG(x && w && scale && shift && y, "null tensor pointer");
  B2_CHECK_ARG(N > 0 && H > 0 && W > 0 && C > 0, "empty output (N %d, H %d, W %d, C %d)", N, H, W, C);
  B2_CHECK_ARG(C % 8 == 0, "channel count %d is not a multiple of 8", C);
  B2_CHECK_ARG(ld % 8 == 0 && ld >= C, "channel pitch %d must be a multiple of 8 and >= C %d", ld, C);
  B2_CHECK_ARG(stride == 1 || stride == 2, "stride %d is not 1 or 2", stride);
  B2_CHECK_ARG(((uintptr_t)x | (uintptr_t)y | (uintptr_t)w | (uintptr_t)scale | (uintptr_t)shift) % 16 == 0,
               "tensors must be 16-byte aligned");
  int rc;
  if ((rc = require_sm90()) != B2_OK) return rc;
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return stride == 1 ? launch_dwconv<1, 4>(x, w, scale, shift, y, N, H, W, C, ld, clamp_in, relu6, st)
                     : launch_dwconv<2, 2>(x, w, scale, shift, y, N, H, W, C, ld, clamp_in, relu6, st);
}

int b2_dwconv3x3_relu_in_ndhwc(const void* x, const float* w, void* y, int N, int H, int W, int C, int ld, void* stream) {
  B2_CHECK_ARG(x && w && y, "null tensor pointer");
  B2_CHECK_ARG(N > 0 && H > 0 && W > 0 && C > 0, "empty output (N %d, H %d, W %d, C %d)", N, H, W, C);
  B2_CHECK_ARG(C % 8 == 0, "channel count %d is not a multiple of 8", C);
  B2_CHECK_ARG(ld % 8 == 0 && ld >= C, "channel pitch %d must be a multiple of 8 and >= C %d", ld, C);
  B2_CHECK_ARG(((uintptr_t)x | (uintptr_t)y | (uintptr_t)w) % 16 == 0, "tensors must be 16-byte aligned");
  int rc;
  if ((rc = require_sm90()) != B2_OK) return rc;
  constexpr int R = 4;
  if ((rc = launch_dwconv<1, R, true>(x, w, nullptr, nullptr, y, N, H, W, C, ld, 0, 0, reinterpret_cast<cudaStream_t>(stream))) != B2_OK)
    return rc;
  set_last_kernel(KID_DWCONV_RELU_IN, 1, R);
  return B2_OK;
}

int b2_dwconv_kxk_relu_in_ndhwc(const void* x, int ldx, const float* w, void* y, int ldy, int N, int H, int W, int C, int K, int stride,
                                int pad, int Ho, int Wo, void* stream) {
  B2_CHECK_ARG(x && w && y, "null tensor pointer");
  B2_CHECK_ARG(K == 3 || K == 5 || K == 7, "kernel size %d is not 3, 5 or 7", K);
  B2_CHECK_ARG(stride == 1 || stride == 2, "stride %d is not 1 or 2", stride);
  B2_CHECK_ARG(N > 0 && H > 0 && W > 0 && C > 0 && Ho > 0 && Wo > 0, "empty tensor (N %d, H %d, W %d, C %d, Ho %d, Wo %d)", N, H, W, C,
               Ho, Wo);
  B2_CHECK_ARG(C % 8 == 0, "channel count %d is not a multiple of 8", C);
  B2_CHECK_ARG(ldx % 8 == 0 && ldx >= C && ldy % 8 == 0 && ldy >= C, "pitches (ldx %d, ldy %d) must be multiples of 8 and >= C %d", ldx,
               ldy, C);
  B2_CHECK_ARG(pad >= 0 && pad <= K / 2, "padding %d is outside [0, %d]", pad, K / 2);
  B2_CHECK_ARG((Ho - 1) * stride - pad < H && (Wo - 1) * stride - pad < W, "output extent %dx%d has windows past the %dx%d input", Ho,
               Wo, H, W);
  B2_CHECK_ARG(((uintptr_t)x | (uintptr_t)y | (uintptr_t)w) % 16 == 0, "tensors must be 16-byte aligned");
  const uintptr_t x0 = (uintptr_t)x, x1 = x0 + ((unsigned long long)N * H * W - 1) * ldx * 2 + C * 2;
  const uintptr_t y0 = (uintptr_t)y, y1 = y0 + ((unsigned long long)N * Ho * Wo - 1) * ldy * 2 + C * 2;
  B2_CHECK_ARG(y1 <= x0 || x1 <= y0, "the output overlaps the input");
  int rc;
  if ((rc = require_sm90()) != B2_OK) return rc;
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  rc = K == 3 ? launch_dwconv_kxk_k<3>(x, ldx, w, y, ldy, N, H, W, C, stride, pad, Ho, Wo, st)
     : K == 5 ? launch_dwconv_kxk_k<5>(x, ldx, w, y, ldy, N, H, W, C, stride, pad, Ho, Wo, st)
              : launch_dwconv_kxk_k<7>(x, ldx, w, y, ldy, N, H, W, C, stride, pad, Ho, Wo, st);
  if (rc != B2_OK) return rc;
  set_last_kernel(KID_DWCONV_KXK, K, stride, pad, kxk_run(K, stride));
  return B2_OK;
}

int b2_relu6_inplace_ndhwc(void* x, long long rows, int ld, void* stream) {
  B2_CHECK_ARG(x && rows > 0, "bad argument");
  B2_CHECK_ARG(ld % 8 == 0 && ld > 0, "channel pitch %d is not a multiple of 8", ld);
  B2_CHECK_ARG((uintptr_t)x % 16 == 0, "tensor must be 16-byte aligned");
  int rc;
  if ((rc = require_sm90()) != B2_OK) return rc;
  const long long vecs = rows * (ld / 8);
  relu6_inplace_kernel<<<div_up(vecs, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(reinterpret_cast<uint4*>(x), vecs);
  B2_CHECK_LAUNCH("relu6_inplace_kernel");
  return B2_OK;
}

}  // extern "C"
