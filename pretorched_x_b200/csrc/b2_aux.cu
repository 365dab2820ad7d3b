// b2_aux.cu -- HBM-bound helper kernels around the tensor-core path: weight packing, pooling, layout
// conversion, casts, the type-A shortcut, the TRN frame gather, and a CUDA-core reference convolution
// used only as an on-device cross-check in tests.  All activation kernels move 16 bytes per thread
// per access (8 fp16 channels) with the channel index fastest, so warps read/write full 128-byte lines.
#include "b2_host.h"

#include <cuda_fp16.h>
#include <float.h>

namespace b2 {

static inline int div_up(long long a, long long b) { return (int)((a + b - 1) / b); }

// ------------------------------------------------------------------------------------------
// weight packing: fp32 [K][Cin][kt][kh][kw] -> fp16 [K][taps][C]   (or the STEM7 run layout)
// ------------------------------------------------------------------------------------------
__global__ void pack_weight_kernel(const float* __restrict__ w, __half* __restrict__ out, int K, int Cin, int kt,
                                   int kh, int kw, int C, long long total) {
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int taps = kt * kh * kw;
  int c = (int)(i % C);
  long long q = i / C;
  int tap = (int)(q % taps);
  int k = (int)(q / taps);
  float v = 0.f;
  if (c < Cin) v = w[((long long)k * Cin + c) * taps + tap];
  out[i] = __float2half_rn(v);
}

// STEM7 weight image (consumed by b2_stemconv.cuh): [ntile][dt][slot][n/8][j = 16-byte K chunk (4)][n%8][e (8)]
// with K element index k = j*8 + e = px*4 + c, px 0 = zero alignment pixel, px 1..7 <-> kw tap 0..6, channels >= Cin
// zero, output channels >= K zero.  `slot` orders the vertical taps of one temporal tap as: even dh in decreasing
// order, then odd dh in decreasing order (stem_slot()), so that the taps feeding consecutive output rows from one
// input row are adjacent.  Each tap is the canonical SWIZZLE_NONE K-major smem layout of a [BN x 32] B operand
// (LBO = 128 B, SBO = 512 B): one contiguous BN*64-byte block, and consecutive taps concatenate to a taller B.
__global__ void pack_weight_stem7_kernel(const float* __restrict__ w, __half* __restrict__ out, int K, int Cin,
                                         int kt, int kh, int BN, long long total) {
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int e = (int)(i & 7);
  const int nn = (int)((i >> 3) & 7);
  const int j = (int)((i >> 6) & 3);
  long long q = i >> 8;
  const int n8 = (int)(q % (BN / 8)); q /= (BN / 8);
  const int pairs = kt * kh;
  const int pr = (int)(q % pairs);
  const int ntile = (int)(q / pairs);
  const int k = ntile * BN + n8 * 8 + nn;
  const int px = j * 2 + (e >> 2), c = e & 3;
  float v = 0.f;
  if (k < K && px >= 1 && c < Cin) {
    const int dt = pr / kh, slot = pr % kh, dw = px - 1;
    const int emax = ((kh - 1) / 2) * 2, n_even = emax / 2 + 1, omax = (kh >= 2) ? ((kh - 2) / 2) * 2 + 1 : -1;
    const int dh = (slot < n_even) ? emax - 2 * slot : omax - 2 * (slot - n_even);
    v = w[((((long long)k * Cin + c) * kt + dt) * kh + dh) * 7 + dw];
  }
  out[i] = __float2half_rn(v);
}

// ------------------------------------------------------------------------------------------
// CUDA-core reference convolution (test cross-check only)
// ------------------------------------------------------------------------------------------
struct SimtConvParams {
  const __half* x; const __half* w; const float* scale; const float* shift; const __half* residual; void* y;
  int N, T, H, W, C, K, ldy, ldr, kt, kh, kw, st, sh, sw, pt, ph, pw, To, Ho, Wo, relu, out_f32, accumulate, stem7,
      ldw;
};

__global__ void conv_simt_kernel(SimtConvParams p, long long total) {
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int k = (int)(i % p.ldy);
  long long m = i / p.ldy;
  int q = (int)m;
  const int wo = q % p.Wo; q /= p.Wo;
  const int ho = q % p.Ho; q /= p.Ho;
  const int to = q % p.To;
  const int n = q / p.To;
  float acc = 0.f;
  if (k < p.K) {
    for (int dt = 0; dt < p.kt; ++dt) {
      const int ti = to * p.st - p.pt + dt;
      if ((unsigned)ti >= (unsigned)p.T) continue;
      for (int dh = 0; dh < p.kh; ++dh) {
        const int hi = ho * p.sh - p.ph + dh;
        if ((unsigned)hi >= (unsigned)p.H) continue;
        for (int dw = 0; dw < p.kw; ++dw) {
          const int wi = wo * p.sw - p.pw + dw;
          if ((unsigned)wi >= (unsigned)p.W) continue;
          const __half* xp = p.x + ((((size_t)n * p.T + ti) * p.H + hi) * p.W + wi) * (size_t)p.C;
          const __half* wp;
          if (p.stem7) {
            // weight image [ntile][pair][n/8][j][n%8][e], BN = p.ldw
            const int BN = p.ldw, px = dw + 1;
            const int emax = ((p.kh - 1) / 2) * 2, n_even = emax / 2 + 1, omax = (p.kh >= 2) ? ((p.kh - 2) / 2) * 2 + 1 : -1;
            const int slot = (dh % 2 == 0) ? (emax - dh) / 2 : n_even + (omax - dh) / 2;
            const size_t base = ((((size_t)(k / BN) * (p.kt * p.kh) + (dt * p.kh + slot)) * (BN / 8) + (k % BN) / 8) * 4 + px / 2) * 64 +
                                (size_t)(k % 8) * 8 + (px & 1) * 4;
            for (int c = 0; c < p.C; ++c) acc += __half2float(xp[c]) * __half2float(p.w[base + c]);
          } else {
            wp = p.w + (size_t)k * p.ldw + (size_t)((dt * p.kh + dh) * p.kw + dw) * p.C;
            for (int c = 0; c < p.C; ++c) acc += __half2float(xp[c]) * __half2float(wp[c]);
          }
        }
      }
    }
    acc = acc * p.scale[k] + p.shift[k];
    if (p.residual) acc += __half2float(p.residual[(size_t)m * p.ldr + k]);
    if (p.relu) acc = fmaxf(acc, 0.f);
  }
  if (p.out_f32) {
    if (k < p.K) {
      float* yo = reinterpret_cast<float*>(p.y) + (size_t)m * p.ldy + k;
      *yo = p.accumulate ? (*yo + acc) : acc;
    }
  } else {
    reinterpret_cast<__half*>(p.y)[(size_t)m * p.ldy + k] = __float2half_rn(acc);
  }
}

// ------------------------------------------------------------------------------------------
// pooling
// ------------------------------------------------------------------------------------------
__global__ void maxpool3d_kernel(const __half* __restrict__ x, __half* __restrict__ y, int N, int T, int H, int W,
                                 int C8, int To, int Ho, int Wo, int kt, int kh, int kw, int st, int sh, int sw, int pt,
                                 int ph, int pw, long long total) {
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c8 = (int)(i % C8);
  long long q = i / C8;
  const int wo = (int)(q % Wo); q /= Wo;
  const int ho = (int)(q % Ho); q /= Ho;
  const int to = (int)(q % To);
  const int n = (int)(q / To);
  const __half2 ninf = __float2half2_rn(-65504.f);
  __half2 m0 = ninf, m1 = ninf, m2 = ninf, m3 = ninf;
  for (int dt = 0; dt < kt; ++dt) {
    const int ti = to * st - pt + dt;
    if ((unsigned)ti >= (unsigned)T) continue;
    for (int dh = 0; dh < kh; ++dh) {
      const int hi = ho * sh - ph + dh;
      if ((unsigned)hi >= (unsigned)H) continue;
      for (int dw = 0; dw < kw; ++dw) {
        const int wi = wo * sw - pw + dw;
        if ((unsigned)wi >= (unsigned)W) continue;
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(x + ((((size_t)n * T + ti) * H + hi) * W + wi) * (size_t)(C8 * 8)) + c8);
        m0 = __hmax2(m0, *reinterpret_cast<const __half2*>(&v.x));
        m1 = __hmax2(m1, *reinterpret_cast<const __half2*>(&v.y));
        m2 = __hmax2(m2, *reinterpret_cast<const __half2*>(&v.z));
        m3 = __hmax2(m3, *reinterpret_cast<const __half2*>(&v.w));
      }
    }
  }
  uint4 o;
  o.x = *reinterpret_cast<uint32_t*>(&m0); o.y = *reinterpret_cast<uint32_t*>(&m1);
  o.z = *reinterpret_cast<uint32_t*>(&m2); o.w = *reinterpret_cast<uint32_t*>(&m3);
  reinterpret_cast<uint4*>(y)[i] = o;
}

// The stem pool (3x3x3, stride 2, pad 1): branch-free so that the nine loads of a temporal tap are issued
// back to back (out-of-range taps are clamped to the window centre, which is always in range and already part
// of the maximum), giving the memory system 9 x 16 B in flight per thread instead of one dependent load at a time.
__global__ void __launch_bounds__(256)
maxpool3d_k3s2p1_kernel(const __half* __restrict__ x, __half* __restrict__ y, int T, int H, int W, int C8, int To,
                        int Ho, int Wo, long long total) {
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c8 = (int)(i % C8);
  long long q = i / C8;
  const int wo = (int)(q % Wo); q /= Wo;
  const int ho = (int)(q % Ho); q /= Ho;
  const int to = (int)(q % To);
  const long long n = q / To;
  const int tc = 2 * to, hc = 2 * ho, wc = 2 * wo;          // window centre (dt = dh = dw = 1): always valid
  const uint4* base = reinterpret_cast<const uint4*>(x) + c8;
  __half2 m0 = __float2half2_rn(-65504.f), m1 = m0, m2 = m0, m3 = m0;
#pragma unroll
  for (int dt = -1; dt <= 1; ++dt) {
    int ti = tc + dt; ti = ((unsigned)ti < (unsigned)T) ? ti : tc;
    uint4 v[9];
#pragma unroll
    for (int dh = -1; dh <= 1; ++dh) {
      int hi = hc + dh; hi = ((unsigned)hi < (unsigned)H) ? hi : hc;
#pragma unroll
      for (int dw = -1; dw <= 1; ++dw) {
        int wi = wc + dw; wi = ((unsigned)wi < (unsigned)W) ? wi : wc;
        v[(dh + 1) * 3 + dw + 1] = __ldg(base + (((n * T + ti) * H + hi) * (long long)W + wi) * C8);
      }
    }
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      m0 = __hmax2(m0, *reinterpret_cast<const __half2*>(&v[k].x));
      m1 = __hmax2(m1, *reinterpret_cast<const __half2*>(&v[k].y));
      m2 = __hmax2(m2, *reinterpret_cast<const __half2*>(&v[k].z));
      m3 = __hmax2(m3, *reinterpret_cast<const __half2*>(&v[k].w));
    }
  }
  uint4 o;
  o.x = *reinterpret_cast<uint32_t*>(&m0); o.y = *reinterpret_cast<uint32_t*>(&m1);
  o.z = *reinterpret_cast<uint32_t*>(&m2); o.w = *reinterpret_cast<uint32_t*>(&m3);
  reinterpret_cast<uint4*>(y)[i] = o;
}

// Second pass of the separable stem pool: (3, 3, 1) window, stride (2, 2, 1), padding (1, 1, 0) over a tensor whose W direction
// was already pooled by the stem convolution's epilogue (b2_conv_args.pool_w).  Same branch-free clamping, 9 loads in flight.
__global__ void __launch_bounds__(256)
maxpool3d_k331s221_kernel(const __half* __restrict__ x, __half* __restrict__ y, int T, int H, int W, int C8, int To, int Ho,
                          long long total) {
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c8 = (int)(i % C8);
  long long q = i / C8;
  const int wo = (int)(q % W); q /= W;
  const int ho = (int)(q % Ho); q /= Ho;
  const int to = (int)(q % To);
  const long long n = q / To;
  const int tc = 2 * to, hc = 2 * ho;
  const uint4* base = reinterpret_cast<const uint4*>(x) + c8;
  uint4 v[9];
#pragma unroll
  for (int dt = -1; dt <= 1; ++dt) {
    int ti = tc + dt; ti = ((unsigned)ti < (unsigned)T) ? ti : tc;
#pragma unroll
    for (int dh = -1; dh <= 1; ++dh) {
      int hi = hc + dh; hi = ((unsigned)hi < (unsigned)H) ? hi : hc;
      v[(dt + 1) * 3 + dh + 1] = __ldg(base + (((n * T + ti) * H + hi) * (long long)W + wo) * C8);
    }
  }
  __half2 m0 = __float2half2_rn(-65504.f), m1 = m0, m2 = m0, m3 = m0;
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    m0 = __hmax2(m0, *reinterpret_cast<const __half2*>(&v[k].x));
    m1 = __hmax2(m1, *reinterpret_cast<const __half2*>(&v[k].y));
    m2 = __hmax2(m2, *reinterpret_cast<const __half2*>(&v[k].z));
    m3 = __hmax2(m3, *reinterpret_cast<const __half2*>(&v[k].w));
  }
  uint4 o;
  o.x = *reinterpret_cast<uint32_t*>(&m0); o.y = *reinterpret_cast<uint32_t*>(&m1);
  o.z = *reinterpret_cast<uint32_t*>(&m2); o.w = *reinterpret_cast<uint32_t*>(&m3);
  reinterpret_cast<uint4*>(y)[i] = o;
}

// global average: grid (C8 chunks / 32, N), 1024 threads.  Lane = one 8-channel chunk (a warp reads 512 contiguous
// bytes of a pixel), warp w walks positions w, w+32, ... ; the 32 partial sums meet in shared memory in a fixed order.
__global__ void __launch_bounds__(1024) avgpool_kernel(const __half* __restrict__ x, __half* __restrict__ y, int S, int C8) {
  __shared__ float part[32][32][9];                 // [slice][lane][8 + pad]
  const int lane = threadIdx.x & 31, slice = threadIdx.x >> 5;
  const int c8 = blockIdx.x * 32 + lane;
  const int n = blockIdx.y;
  float acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  if (c8 < C8) {
    const uint4* base = reinterpret_cast<const uint4*>(x + (size_t)n * S * (C8 * 8)) + c8;
#pragma unroll 4
    for (int s = slice; s < S; s += 32) {
      const uint4 v = __ldg(base + (size_t)s * C8);
      const uint32_t u[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&u[e]));
        acc[2 * e] += f.x; acc[2 * e + 1] += f.y;
      }
    }
  }
#pragma unroll
  for (int e = 0; e < 8; ++e) part[slice][lane][e] = acc[e];
  __syncthreads();
  if (slice == 0 && c8 < C8) {
    float tot[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int w = 0; w < 32; ++w)
#pragma unroll
      for (int e = 0; e < 8; ++e) tot[e] += part[w][lane][e];
    const float inv = 1.f / (float)S;
    uint32_t o[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      __half2 h = __floats2half2_rn(tot[2 * e] * inv, tot[2 * e + 1] * inv);
      o[e] = *reinterpret_cast<uint32_t*>(&h);
    }
    reinterpret_cast<uint4*>(y + (size_t)n * (C8 * 8))[c8] = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

// ------------------------------------------------------------------------------------------
// layout conversion
// ------------------------------------------------------------------------------------------
// fp32 NCDHW -> fp16 NDHWC(pitch Cp).  One thread per pixel: reads are coalesced along W within each
// channel plane, the write is Cp*2 contiguous bytes per thread (8 B for the NDHWC4 stem input).
__device__ __forceinline__ float to_f32(float v) { return v; }
__device__ __forceinline__ float to_f32(__half v) { return __half2float(v); }

template <typename TIn>
__global__ void ncdhw_to_ndhwc_kernel(const TIn* __restrict__ x, __half* __restrict__ y, int C, long long S,
                                      int Cp, long long total_px) {
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= total_px) return;
  const long long n = i / S, s = i - n * S;
  const TIn* xp = x + n * C * S + s;
  __half* yp = y + i * Cp;
  if (Cp == 4) {
    float v[4] = {0, 0, 0, 0};
    for (int c = 0; c < C && c < 4; ++c) v[c] = to_f32(__ldg(xp + (long long)c * S));
    __half2 a = __floats2half2_rn(v[0], v[1]), b = __floats2half2_rn(v[2], v[3]);
    uint2 o; o.x = *reinterpret_cast<uint32_t*>(&a); o.y = *reinterpret_cast<uint32_t*>(&b);
    *reinterpret_cast<uint2*>(yp) = o;
  } else {
    for (int c = 0; c < Cp; ++c) yp[c] = __float2half_rn(c < C ? to_f32(__ldg(xp + (long long)c * S)) : 0.f);
  }
}

// Stem input, fp32 NCDHW with C <= 4 -> fp16 NDHWC4, four pixels per thread: one 16-byte load per channel plane and one 32-byte
// store (the per-pixel version keeps only 12 B of loads in flight per thread; S % 4 == 0 and 16-byte aligned
// planes are checked by the launcher).
__global__ void __launch_bounds__(256)
ncdhw_f32_to_ndhwc4_x4_kernel(const float* __restrict__ x, __half* __restrict__ y, int C, long long S, long long total_q) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;          // quad of pixels
  if (i >= total_q) return;
  const long long S4 = S >> 2;
  const long long n = i / S4, s4 = i - n * S4;
  const float4* xp = reinterpret_cast<const float4*>(x + n * C * S) + s4;
  float4 v[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) v[c] = (c < C) ? __ldg(xp + c * S4) : make_float4(0.f, 0.f, 0.f, 0.f);
  const float w3[4] = {0.f, 0.f, 0.f, 0.f};
  float4 v3 = make_float4(w3[0], w3[1], w3[2], w3[3]);
  if (C > 3) v3 = __ldg(xp + 3 * S4);
  const float a0[4] = {v[0].x, v[0].y, v[0].z, v[0].w}, a1[4] = {v[1].x, v[1].y, v[1].z, v[1].w};
  const float a2[4] = {v[2].x, v[2].y, v[2].z, v[2].w}, a3[4] = {v3.x, v3.y, v3.z, v3.w};
  uint32_t o[8];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const __half2 p01 = __floats2half2_rn(a0[k], a1[k]), p23 = __floats2half2_rn(a2[k], a3[k]);
    o[2 * k] = *reinterpret_cast<const uint32_t*>(&p01); o[2 * k + 1] = *reinterpret_cast<const uint32_t*>(&p23);
  }
  uint4* yp = reinterpret_cast<uint4*>(y + (n * S + s4 * 4) * 4);
  yp[0] = make_uint4(o[0], o[1], o[2], o[3]);
  yp[1] = make_uint4(o[4], o[5], o[6], o[7]);
}

// fp16 NDHWC(pitch Cp) -> fp32 NCDHW via a 32x32 smem transpose tile (positions x channels)
__global__ void ndhwc_to_ncdhw_kernel(const __half* __restrict__ x, float* __restrict__ y, int C, long long S, int Cp) {
  __shared__ float tile[32][33];
  const long long n = blockIdx.z;
  const long long s0 = (long long)blockIdx.x * 32;
  const int c0 = blockIdx.y * 32;
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    const long long s = s0 + r;
    const int c = c0 + threadIdx.x;
    tile[r][threadIdx.x] = (s < S && c < C) ? __half2float(x[(n * S + s) * Cp + c]) : 0.f;
  }
  __syncthreads();
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    const int c = c0 + r;
    const long long s = s0 + threadIdx.x;
    if (c < C && s < S) y[(n * C + c) * S + s] = tile[threadIdx.x][r];
  }
}

__global__ void cast_kernel(const float* __restrict__ x, int ldx, __half* __restrict__ y, int ldy, int rows, int cols,
                            int relu) {
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= (long long)rows * ldy) return;
  const int c = (int)(i % ldy);
  const long long r = i / ldy;
  float v = 0.f;
  if (c < cols) {
    v = x[r * ldx + c];
    if (relu) v = fmaxf(v, 0.f);
  }
  y[i] = __float2half_rn(v);
}

// type-A shortcut: y[n,to,ho,wo,0:C] = x[n,to*s,ho*s,wo*s,:], y[..., C:Cout] = 0
__global__ void shortcut_a_kernel(const __half* __restrict__ x, __half* __restrict__ y, int T, int H, int W, int C8,
                                  int s, int To, int Ho, int Wo, int Co8, long long total) {
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c8 = (int)(i % Co8);
  long long q = i / Co8;
  const int wo = (int)(q % Wo); q /= Wo;
  const int ho = (int)(q % Ho); q /= Ho;
  const int to = (int)(q % To);
  const long long n = q / To;
  uint4 v = make_uint4(0, 0, 0, 0);
  if (c8 < C8) v = __ldg(reinterpret_cast<const uint4*>(x + (((n * T + (long long)to * s) * H + (long long)ho * s) * W + (long long)wo * s) * (C8 * 8)) + c8);
  reinterpret_cast<uint4*>(y)[i] = v;
}

// y[r] = [ a[r][0:Ca8*8] | b[r][0:Cb8*8] | 0 ... ]   (torch.cat along channels, slowfast.py:143-150)
__global__ void concat_channels_kernel(const __half* __restrict__ a, int lda8, int Ca8, const __half* __restrict__ b,
                                       int ldb8, int Cb8, __half* __restrict__ y, int ldy8, long long total) {
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c8 = (int)(i % ldy8);
  const long long r = i / ldy8;
  uint4 v = make_uint4(0, 0, 0, 0);
  if (c8 < Ca8) v = __ldg(reinterpret_cast<const uint4*>(a) + r * lda8 + c8);
  else if (c8 < Ca8 + Cb8) v = __ldg(reinterpret_cast<const uint4*>(b) + r * ldb8 + (c8 - Ca8));
  reinterpret_cast<uint4*>(y)[i] = v;
}

// y[(n * n_tuples + t)][j * F + f] = x[n][idx[t * n_idx + j]][f]: all frame tuples of one scale in one pass; the output row
// index has the tuple fastest, so the hidden layer of the relation MLP comes out as [n][n_tuples * bottleneck]
__global__ void gather_frames_kernel(const __half* __restrict__ x, __half* __restrict__ y, const int* __restrict__ idx,
                                     int T, int F8, int n_idx, int n_tuples, long long total) {
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int f8 = (int)(i % F8);
  long long q = i / F8;
  const int j = (int)(q % n_idx);
  q /= n_idx;
  const int t = (int)(q % n_tuples);
  const long long n = q / n_tuples;
  reinterpret_cast<uint4*>(y)[i] = __ldg(reinterpret_cast<const uint4*>(x + (n * T + idx[t * n_idx + j]) * (long long)(F8 * 8)) + f8);
}

// ------------------------------------------------------------------------------------------
// fine-tuning backward helpers
// ------------------------------------------------------------------------------------------
// Adjoint of shortcut_a_kernel: y[n, s*to, s*ho, s*wo, 0:C] = g[n, to, ho, wo, 0:C], every other pixel and channels [C, ldy)
// zero.  y has the full-resolution extent (T, H, W); s * (To - 1) <= T - 1 for To = (T - 1) / s + 1.
__global__ void zero_insert_kernel(const __half* __restrict__ g, int ldg8, int C8, __half* __restrict__ y, int ldy8, int T, int H,
                                   int W, int s, int To, int Ho, int Wo, long long total) {
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c8 = (int)(i % ldy8);
  long long q = i / ldy8;
  const int w = (int)(q % W); q /= W;
  const int h = (int)(q % H); q /= H;
  const int t = (int)(q % T);
  const long long n = q / T;
  uint4 v = make_uint4(0, 0, 0, 0);
  if (c8 < C8 && t % s == 0 && h % s == 0 && w % s == 0 && t / s < To && h / s < Ho && w / s < Wo)
    v = __ldg(reinterpret_cast<const uint4*>(g) + (((n * To + t / s) * Ho + h / s) * Wo + w / s) * ldg8 + c8);
  reinterpret_cast<uint4*>(y)[i] = v;
}

// Column sums of an fp16 matrix in two fixed-order passes: CTA (column block of 32, row chunk) -> part[chunk][c], then
// out[c] = inv * sum_chunk part[chunk][c].
constexpr int kColsumChunks = 128;
__global__ void __launch_bounds__(256) colsum_partial_kernel(const __half* __restrict__ g, int ldg, long long rows, int C,
                                                             float* __restrict__ part) {
  __shared__ float red[8][33];
  const int c = blockIdx.x * 32 + threadIdx.x;
  const long long r0 = rows * blockIdx.y / kColsumChunks, r1 = rows * (blockIdx.y + 1) / kColsumChunks;
  float acc = 0.f;
  if (c < C)
    for (long long r = r0 + threadIdx.y; r < r1; r += 8) acc += __half2float(g[r * ldg + c]);
  red[threadIdx.y][threadIdx.x] = acc;
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
    float t = 0.f;
    for (int j = 0; j < 8; ++j) t += red[j][threadIdx.x];
    part[(long long)blockIdx.y * C + c] = t;
  }
}
__global__ void colsum_final_kernel(const float* __restrict__ part, int C, const float* __restrict__ inv, float* __restrict__ out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float t = 0.f;
  for (int j = 0; j < kColsumChunks; ++j) t += part[(long long)j * C + c];
  out[c] = t * (inv ? *inv : 1.f);
}

// Power-of-two loss scale from the largest |g| of the gradient entering the trunk: max|g| lands in [2^7, 2^8), leaving 2^8
// of fp16 headroom for growth through the blocks.  sc = [scale, 1 / scale].  Non-finite values leave the scale at 2^0 so
// that they reach the parameter gradients unchanged.
__global__ void __launch_bounds__(1024) loss_scale_kernel(const float* __restrict__ g, int rows, int cols, int ldg,
                                                          float* __restrict__ sc) {
  __shared__ float red[32];
  __shared__ int bad_any;
  if (threadIdx.x == 0) bad_any = 0;
  __syncthreads();
  float m = 0.f;
  int bad = 0;
  const long long total = (long long)rows * cols;
  for (long long i = threadIdx.x; i < total; i += blockDim.x) {
    const float v = fabsf(g[(i / cols) * ldg + i % cols]);
    if (!(v <= FLT_MAX)) bad = 1;
    else m = fmaxf(m, v);
  }
  if (bad) atomicOr(&bad_any, 1);
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) m = fmaxf(m, __shfl_down_sync(0xffffffffu, m, off));
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int j = 1; j < (int)(blockDim.x >> 5); ++j) m = fmaxf(m, red[j]);
    int e = 0;
    if (m > 0.f && !bad_any) frexpf(m, &e);              // m = f * 2^e, f in [0.5, 1)
    int k = (m > 0.f && !bad_any) ? 8 - e : 0;
    k = k > 100 ? 100 : (k < -100 ? -100 : k);
    sc[0] = ldexpf(1.f, k);
    sc[1] = ldexpf(1.f, -k);
  }
}

// Backward of the global average pool: y[n*S + p][c] = fp16(gf[n][c] * scale / S) where the pooled block output was
// positive (its closing ReLU), 0 elsewhere and in channels [C, ld).
__global__ void pool_backward_kernel(const float* __restrict__ gf, int ldf, const float* __restrict__ sc, const __half* __restrict__ out,
                                     __half* __restrict__ y, int S, int C, int ld8, long long total) {
  long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c8 = (int)(i % ld8);
  const long long r = i / ld8;
  const long long n = r / S;
  const float f = sc[0] / (float)S;
  const uint4 mk = __ldg(reinterpret_cast<const uint4*>(out) + i);
  const __half* mh = reinterpret_cast<const __half*>(&mk);
  uint4 v;
  __half* vh = reinterpret_cast<__half*>(&v);
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = c8 * 8 + j;
    vh[j] = __float2half_rn((c < C && __half2float(mh[j]) > 0.f) ? gf[n * ldf + c] * f : 0.f);
  }
  reinterpret_cast<uint4*>(y)[i] = v;
}

}  // namespace b2

using namespace b2;

extern "C" {

static int odim(int in, int k, int s, int p) { return (in + 2 * p - k) / s + 1; }

static int stem_bn(int K) { return K <= 64 ? 64 : 128; }

size_t b2_pack_conv_weight_elems(int K, int Cin, int kt, int kh, int kw, int C, int mode) {
  (void)Cin;
  if (mode == B2_CONV_STEM7) {
    const int BN = stem_bn(K);
    return (size_t)((K + BN - 1) / BN) * kt * kh * BN * 32;
  }
  return (size_t)K * kt * kh * kw * C;
}

int b2_pack_conv_weight(const float* w, void* out, int K, int Cin, int kt, int kh, int kw, int C, int mode,
                        void* stream) {
  B2_CHECK_ARG(w && out, "null pointer");
  B2_CHECK_ARG(K > 0 && Cin > 0 && kt > 0 && kh > 0 && kw > 0, "non-positive dimension");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const long long total = (long long)b2_pack_conv_weight_elems(K, Cin, kt, kh, kw, C, mode);
  if (mode == B2_CONV_STEM7) {
    B2_CHECK_ARG(kw == 7 && Cin <= 4, "STEM7 packing needs kw == 7 and Cin <= 4");
    pack_weight_stem7_kernel<<<div_up(total, 256), 256, 0, st>>>(w, reinterpret_cast<__half*>(out), K, Cin, kt, kh,
                                                                 stem_bn(K), total);
  } else {
    B2_CHECK_ARG(C >= Cin && C % 8 == 0, "packed channel pitch %d must be >= Cin and a multiple of 8", C);
    pack_weight_kernel<<<div_up(total, 256), 256, 0, st>>>(w, reinterpret_cast<__half*>(out), K, Cin, kt, kh, kw, C, total);
  }
  B2_CHECK_LAUNCH("pack_weight");
  return B2_OK;
}

int b2_conv_ndhwc_fprop_simt(const b2_conv_args* a, void* stream) {
  B2_CHECK_ARG(a && a->x && a->w && a->scale && a->shift && a->y, "null pointer");
  SimtConvParams p;
  p.x = (const __half*)a->x; p.w = (const __half*)a->w; p.scale = a->scale; p.shift = a->shift;
  p.residual = (const __half*)a->residual; p.y = a->y;
  p.N = a->N; p.T = a->T; p.H = a->H; p.W = a->W; p.C = a->C; p.K = a->K; p.ldy = a->ldy; p.ldr = a->ldr;
  p.kt = a->kt; p.kh = a->kh; p.kw = a->kw; p.st = a->st; p.sh = a->sh; p.sw = a->sw;
  p.pt = a->pt; p.ph = a->ph; p.pw = a->pw;
  p.To = odim(a->T, a->kt, a->st, a->pt); p.Ho = odim(a->H, a->kh, a->sh, a->ph); p.Wo = odim(a->W, a->kw, a->sw, a->pw);
  p.relu = a->relu; p.out_f32 = a->out_f32; p.accumulate = a->accumulate;
  p.stem7 = (a->mode == B2_CONV_STEM7);
  p.ldw = p.stem7 ? stem_bn(a->K) : a->kt * a->kh * a->kw * a->C;
  const long long total = (long long)a->N * p.To * p.Ho * p.Wo * a->ldy;
  conv_simt_kernel<<<div_up(total, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(p, total);
  B2_CHECK_LAUNCH("conv_simt");
  return B2_OK;
}

int b2_maxpool3d_ndhwc(const void* x, void* y, int N, int T, int H, int W, int C, int kt, int kh, int kw, int st,
                       int sh, int sw, int pt, int ph, int pw, void* stream) {
  B2_CHECK_ARG(x && y, "null pointer");
  B2_CHECK_ARG(C % 8 == 0, "channel pitch %d is not a multiple of 8", C);
  const int To = odim(T, kt, st, pt), Ho = odim(H, kh, sh, ph), Wo = odim(W, kw, sw, pw);
  B2_CHECK_ARG(To > 0 && Ho > 0 && Wo > 0, "empty output");
  const long long total = (long long)N * To * Ho * Wo * (C / 8);
  if (kt == 3 && kh == 3 && kw == 3 && st == 2 && sh == 2 && sw == 2 && pt == 1 && ph == 1 && pw == 1) {
    maxpool3d_k3s2p1_kernel<<<div_up(total, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
        (const __half*)x, (__half*)y, T, H, W, C / 8, To, Ho, Wo, total);
  } else if (kt == 3 && kh == 3 && kw == 1 && st == 2 && sh == 2 && sw == 1 && pt == 1 && ph == 1 && pw == 0) {
    maxpool3d_k331s221_kernel<<<div_up(total, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
        (const __half*)x, (__half*)y, T, H, W, C / 8, To, Ho, total);
  } else {
    maxpool3d_kernel<<<div_up(total, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
        (const __half*)x, (__half*)y, N, T, H, W, C / 8, To, Ho, Wo, kt, kh, kw, st, sh, sw, pt, ph, pw, total);
  }
  B2_CHECK_LAUNCH("maxpool3d");
  return B2_OK;
}

int b2_avgpool_global_ndhwc(const void* x, void* y, int N, int S, int C, void* stream) {
  B2_CHECK_ARG(x && y && N > 0 && S > 0, "bad argument");
  B2_CHECK_ARG(C % 8 == 0, "channel pitch %d is not a multiple of 8", C);
  dim3 grid(div_up(C / 8, 32), N);
  avgpool_kernel<<<grid, 1024, 0, reinterpret_cast<cudaStream_t>(stream)>>>((const __half*)x, (__half*)y, S, C / 8);
  B2_CHECK_LAUNCH("avgpool");
  return B2_OK;
}

int b2_ncdhw_f32_to_ndhwc_f16(const float* x, void* y, int N, int C, int T, int H, int W, int Cp, void* stream) {
  B2_CHECK_ARG(x && y && Cp >= C && (Cp == 4 || Cp % 8 == 0), "bad argument (Cp must be 4 or a multiple of 8, >= C)");
  const long long S = (long long)T * H * W, total = (long long)N * S;
  if (Cp == 4 && C <= 4 && S % 4 == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(y) & 15) == 0) {
    ncdhw_f32_to_ndhwc4_x4_kernel<<<div_up(total / 4, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(x, (__half*)y, C, S, total / 4);
  } else {
    ncdhw_to_ndhwc_kernel<float><<<div_up(total, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(x, (__half*)y, C, S, Cp, total);
  }
  B2_CHECK_LAUNCH("ncdhw_to_ndhwc");
  return B2_OK;
}

int b2_ncdhw_f16_to_ndhwc_f16(const void* x, void* y, int N, int C, int T, int H, int W, int Cp, void* stream) {
  B2_CHECK_ARG(x && y && Cp >= C && (Cp == 4 || Cp % 8 == 0), "bad argument (Cp must be 4 or a multiple of 8, >= C)");
  const long long S = (long long)T * H * W, total = (long long)N * S;
  ncdhw_to_ndhwc_kernel<__half><<<div_up(total, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      (const __half*)x, (__half*)y, C, S, Cp, total);
  B2_CHECK_LAUNCH("ncdhw_to_ndhwc_f16");
  return B2_OK;
}

int b2_ndhwc_f16_to_ncdhw_f32(const void* x, float* y, int N, int C, int T, int H, int W, int Cp, void* stream) {
  B2_CHECK_ARG(x && y && Cp >= C, "bad argument");
  const long long S = (long long)T * H * W;
  dim3 grid(div_up(S, 32), div_up(C, 32), N), block(32, 8);
  ndhwc_to_ncdhw_kernel<<<grid, block, 0, reinterpret_cast<cudaStream_t>(stream)>>>((const __half*)x, y, C, S, Cp);
  B2_CHECK_LAUNCH("ndhwc_to_ncdhw");
  return B2_OK;
}

int b2_cast_f32_to_f16(const float* x, int ldx, void* y, int ldy, int rows, int cols, int relu, void* stream) {
  B2_CHECK_ARG(x && y && rows > 0 && cols > 0 && ldx >= cols && ldy >= cols, "bad argument");
  const long long total = (long long)rows * ldy;
  cast_kernel<<<div_up(total, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(x, ldx, (__half*)y, ldy, rows, cols, relu);
  B2_CHECK_LAUNCH("cast");
  return B2_OK;
}

int b2_shortcut_a_ndhwc(const void* x, void* y, int N, int T, int H, int W, int C, int stride, int Cout, void* stream) {
  B2_CHECK_ARG(x && y && stride > 0, "bad argument");
  B2_CHECK_ARG(C % 8 == 0 && Cout % 8 == 0 && Cout >= C, "channel pitches must be multiples of 8 with Cout >= C");
  // F.avg_pool3d(kernel_size=1, stride): out = floor((in - 1) / stride) + 1
  const int To = (T - 1) / stride + 1, Ho = (H - 1) / stride + 1, Wo = (W - 1) / stride + 1;
  const long long total = (long long)N * To * Ho * Wo * (Cout / 8);
  shortcut_a_kernel<<<div_up(total, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      (const __half*)x, (__half*)y, T, H, W, C / 8, stride, To, Ho, Wo, Cout / 8, total);
  B2_CHECK_LAUNCH("shortcut_a");
  return B2_OK;
}

int b2_concat_channels(const void* a, int lda, int Ca, const void* b, int ldb, int Cb, void* y, int ldy, long long rows,
                       void* stream) {
  B2_CHECK_ARG(a && b && y && rows > 0, "bad argument");
  B2_CHECK_ARG(lda % 8 == 0 && ldb % 8 == 0 && ldy % 8 == 0 && Ca % 8 == 0 && Cb % 8 == 0,
               "channel counts and pitches must be multiples of 8");
  B2_CHECK_ARG(lda >= Ca && ldb >= Cb && ldy >= Ca + Cb, "pitch smaller than extent");
  const long long total = rows * (ldy / 8);
  concat_channels_kernel<<<div_up(total, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      (const __half*)a, lda / 8, Ca / 8, (const __half*)b, ldb / 8, Cb / 8, (__half*)y, ldy / 8, total);
  B2_CHECK_LAUNCH("concat_channels");
  return B2_OK;
}

int b2_gather_frame_tuples(const void* x, void* y, const int32_t* idx_dev, int N, int T, int F, int n_idx, int n_tuples,
                           void* stream) {
  B2_CHECK_ARG(x && y && idx_dev && F % 8 == 0 && n_idx > 0 && n_tuples > 0 && T > 0, "bad argument");
  const long long total = (long long)N * n_tuples * n_idx * (F / 8);
  gather_frames_kernel<<<div_up(total, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      (const __half*)x, (__half*)y, idx_dev, T, F / 8, n_idx, n_tuples, total);
  B2_CHECK_LAUNCH("gather_frames");
  return B2_OK;
}

int b2_gather_frames(const void* x, void* y, const int32_t* idx_dev, int N, int T, int F, int n_idx, void* stream) {
  return b2_gather_frame_tuples(x, y, idx_dev, N, T, F, n_idx, 1, stream);
}

int b2_zero_insert_ndhwc(const void* g, int ldg, int C, void* y, int ldy, int N, int T, int H, int W, int stride, void* stream) {
  B2_CHECK_ARG(g && y && N > 0 && T > 0 && H > 0 && W > 0 && stride > 0, "bad argument");
  B2_CHECK_ARG(C % 8 == 0 && ldg % 8 == 0 && ldy % 8 == 0 && ldg >= C && ldy >= C, "channel counts and pitches must be multiples of 8");
  const int To = (T - 1) / stride + 1, Ho = (H - 1) / stride + 1, Wo = (W - 1) / stride + 1;
  const long long total = (long long)N * T * H * W * (ldy / 8);
  zero_insert_kernel<<<div_up(total, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      (const __half*)g, ldg / 8, C / 8, (__half*)y, ldy / 8, T, H, W, stride, To, Ho, Wo, total);
  B2_CHECK_LAUNCH("zero_insert");
  return B2_OK;
}

size_t b2_colsum_workspace_elems(int C) { return (size_t)kColsumChunks * (C > 0 ? C : 0); }

int b2_colsum_f16(const void* g, int ldg, long long rows, int C, const float* inv_loss_scale, float* out, float* ws, void* stream) {
  B2_CHECK_ARG(g && out && ws && rows > 0 && C > 0 && ldg >= C, "bad argument");
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  colsum_partial_kernel<<<dim3(div_up(C, 32), kColsumChunks), dim3(32, 8), 0, st>>>((const __half*)g, ldg, rows, C, ws);
  B2_CHECK_LAUNCH("colsum_partial");
  colsum_final_kernel<<<div_up(C, 256), 256, 0, st>>>(ws, C, inv_loss_scale, out);
  B2_CHECK_LAUNCH("colsum_final");
  return B2_OK;
}

int b2_loss_scale_f32(const float* g, int rows, int cols, int ldg, float* scale_pair, void* stream) {
  B2_CHECK_ARG(g && scale_pair && rows > 0 && cols > 0 && ldg >= cols, "bad argument");
  loss_scale_kernel<<<1, 1024, 0, reinterpret_cast<cudaStream_t>(stream)>>>(g, rows, cols, ldg, scale_pair);
  B2_CHECK_LAUNCH("loss_scale");
  return B2_OK;
}

int b2_avgpool_global_backward(const float* gf, int ldf, const float* scale_pair, const void* out, void* y, int N, int S, int C,
                               int ld, void* stream) {
  B2_CHECK_ARG(gf && scale_pair && out && y && N > 0 && S > 0 && C > 0 && ldf >= C, "bad argument");
  B2_CHECK_ARG(ld % 8 == 0 && ld >= C, "channel pitch %d is not a multiple of 8 >= C", ld);
  const long long total = (long long)N * S * (ld / 8);
  pool_backward_kernel<<<div_up(total, 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      gf, ldf, scale_pair, (const __half*)out, (__half*)y, S, C, ld / 8, total);
  B2_CHECK_LAUNCH("pool_backward");
  return B2_OK;
}

}  // extern "C"
