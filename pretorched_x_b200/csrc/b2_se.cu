// b2_se.cu -- squeeze-and-excitation of SE-ResNet / SE-ResNeXt bottlenecks (senet.py:85-104) as per-sample affine rows.
//
// SEModule scales bn3(conv3(h2)) by e = sigmoid(fc2(relu(fc1(avgpool(bn3(conv3(h2))))))).  conv3 + bn3 is affine, so the pool
// commutes with it: avgpool(bn3(W3 h2)) = s3 * (W3 . mean(h2)) + t3, and fc1 composed with it is one affine map of mean(h2)
// (the caller folds W1 diag(s3) W3 and W1 t3 + b1 once).  Three launches:
//   se_mean_kernel      m[n][c]  = sum_p h2[n, p, c] / S                       fp32, fixed-order two-level sum
//   se_fc_kernel<0>     a[n][r]  = relu(sum_c w1[r][c] m[n][c] + b1[r])
//   se_fc_kernel<1>     e[n][k]  = sigmoid(sum_r w2[k][r] a[n][r] + b2[k]); scale[n][k] = e s3[k], shift[n][k] = e t3[k]
// The closing GEMM then computes relu(scale[n] * (W3 h2) + shift[n] + residual), which is relu(e * bn3(W3 h2) + residual).
// Every sum runs in one fixed order (no atomics, no split-dependent reduction): results are bitwise repeatable.
#include "b2_host.h"

#include <cuda_fp16.h>

namespace b2 {

constexpr int kSeMeanCols = 64;      // channels per mean CTA: 8 threads x 8 fp16 channels (one 16-byte load)
constexpr int kSeMeanStripes = 32;   // position stripes per mean CTA
constexpr int kSeFcJ = 64, kSeFcN = 16, kSeFcK = 32;

// grid (N, ceil(C / 64)), 256 threads: thread (stripe r, chunk j) sums positions r, r + 32, ... of channels [c0 + 8 j, c0 + 8 j + 8),
// then thread t < 64 adds the 32 stripe sums of channel c0 + t in stripe order.
__global__ void __launch_bounds__(256) se_mean_kernel(const __half* __restrict__ h, int ldh, int S, int C, float* __restrict__ m) {
  __shared__ float part[kSeMeanStripes][kSeMeanCols + 1];
  const int n = blockIdx.x, c0 = blockIdx.y * kSeMeanCols;
  const int j = threadIdx.x & 7, r = threadIdx.x >> 3;
  const int c = c0 + 8 * j;
  float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  if (c < C) {
    const __half* base = h + static_cast<size_t>(n) * S * ldh + c;
    for (int p = r; p < S; p += kSeMeanStripes) {
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(base + static_cast<size_t>(p) * ldh));
      const __half2* hv = reinterpret_cast<const __half2*>(&v);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float2 f = __half22float2(hv[q]);
        acc[2 * q] += f.x;
        acc[2 * q + 1] += f.y;
      }
    }
  }
#pragma unroll
  for (int q = 0; q < 8; ++q) part[r][8 * j + q] = acc[q];
  __syncthreads();
  if (threadIdx.x < kSeMeanCols && c0 + threadIdx.x < C) {
    float s = 0.f;
    for (int i = 0; i < kSeMeanStripes; ++i) s += part[i][threadIdx.x];
    m[static_cast<size_t>(n) * C + c0 + threadIdx.x] = s / static_cast<float>(S);
  }
}

// out[n][j] = act(sum_k x[n][k] w[j][k] + b[j]) for n < N, j < J; x fp32 [N][K], w fp32 [J][K].  CTA: 64 outputs x 16 samples,
// thread (jj = t % 64, sample quad t / 64); each output is one fmaf chain over k = 0 .. K-1.
// MODE 0: act = relu, out fp32 [N][J].  MODE 1: e = sigmoid, scale[n * ld + j] = e * s3[j], shift[n * ld + j] = e * t3[j].
template <int MODE>
__global__ void __launch_bounds__(256) se_fc_kernel(const float* __restrict__ x, const float* __restrict__ w, const float* __restrict__ b,
                                                    int N, int J, int K, float* __restrict__ out, const float* __restrict__ s3,
                                                    const float* __restrict__ t3, float* __restrict__ scale, float* __restrict__ shift,
                                                    int ld) {
  __shared__ float ws[kSeFcK][kSeFcJ + 1];
  __shared__ float xs[kSeFcN][kSeFcK];
  const int t = threadIdx.x, jj = t & (kSeFcJ - 1), quad = t >> 6;
  const int j0 = blockIdx.x * kSeFcJ, n0 = blockIdx.y * kSeFcN;
  float acc[4] = {0.f, 0.f, 0.f, 0.f};
  for (int k0 = 0; k0 < K; k0 += kSeFcK) {
#pragma unroll
    for (int q = 0; q < kSeFcJ * kSeFcK / 256; ++q) {
      const int e = t + 256 * q, rj = e / kSeFcK, ck = e % kSeFcK;
      ws[ck][rj] = (j0 + rj < J && k0 + ck < K) ? __ldg(&w[static_cast<size_t>(j0 + rj) * K + k0 + ck]) : 0.f;
    }
#pragma unroll
    for (int q = 0; q < kSeFcN * kSeFcK / 256; ++q) {
      const int e = t + 256 * q, rn = e / kSeFcK, ck = e % kSeFcK;
      xs[rn][ck] = (n0 + rn < N && k0 + ck < K) ? __ldg(&x[static_cast<size_t>(n0 + rn) * K + k0 + ck]) : 0.f;
    }
    __syncthreads();
    const int kn = min(kSeFcK, K - k0);
    for (int k = 0; k < kn; ++k) {
      const float wv = ws[k][jj];
#pragma unroll
      for (int s = 0; s < 4; ++s) acc[s] = fmaf(xs[4 * quad + s][k], wv, acc[s]);
    }
    __syncthreads();
  }
  const int j = j0 + jj;
  if (j >= J) return;
  const float bj = __ldg(&b[j]);
#pragma unroll
  for (int s = 0; s < 4; ++s) {
    const int n = n0 + 4 * quad + s;
    if (n >= N) continue;
    const float v = acc[s] + bj;
    if (MODE == 0) {
      out[static_cast<size_t>(n) * J + j] = fmaxf(v, 0.f);
    } else {
      const float e = 1.f / (1.f + expf(-v));
      scale[static_cast<size_t>(n) * ld + j] = e * __ldg(&s3[j]);
      shift[static_cast<size_t>(n) * ld + j] = e * __ldg(&t3[j]);
    }
  }
}

}  // namespace b2

using namespace b2;

extern "C" {

size_t b2_se_excite_workspace_elems(int N, int C2, int R) {
  return N > 0 && C2 > 0 && R > 0 ? (size_t)N * C2 + (size_t)N * R : 0;
}

int b2_se_excite(const void* h, int ldh, int N, int S, int C2, const float* w1, const float* b1, int R, const float* w2, const float* b2,
                 int C, const float* s3, const float* t3, float* scale, float* shift, int ld_aff, float* ws, size_t ws_elems,
                 void* stream) {
  B2_CHECK_ARG(h && w1 && b1 && w2 && b2 && s3 && t3 && scale && shift && ws, "null pointer");
  B2_CHECK_ARG(N > 0 && S > 0 && C2 > 0 && R > 0 && C > 0, "non-positive dimension");
  B2_CHECK_ARG(C2 % 8 == 0 && ldh % 8 == 0 && ldh >= C2 && (reinterpret_cast<uintptr_t>(h) & 15) == 0,
               "h must be 16-byte aligned fp16 rows with C2 %% 8 == 0 and pitch ldh %% 8 == 0, ldh >= C2 (got C2 %d, ldh %d)", C2, ldh);
  B2_CHECK_ARG(ld_aff >= C, "affine pitch %d < C %d", ld_aff, C);
  B2_CHECK_ARG(ws_elems >= b2_se_excite_workspace_elems(N, C2, R), "workspace too small");
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  float* m = ws;
  float* a = ws + (size_t)N * C2;
  se_mean_kernel<<<dim3(N, (C2 + kSeMeanCols - 1) / kSeMeanCols), 256, 0, st>>>(reinterpret_cast<const __half*>(h), ldh, S, C2, m);
  B2_CHECK_LAUNCH("se_mean_kernel");
  se_fc_kernel<0><<<dim3((R + kSeFcJ - 1) / kSeFcJ, (N + kSeFcN - 1) / kSeFcN), 256, 0, st>>>(m, w1, b1, N, R, C2, a, nullptr, nullptr,
                                                                                          nullptr, nullptr, 0);
  B2_CHECK_LAUNCH("se_fc_kernel<0>");
  se_fc_kernel<1><<<dim3((C + kSeFcJ - 1) / kSeFcJ, (N + kSeFcN - 1) / kSeFcN), 256, 0, st>>>(a, w2, b2, N, C, R, nullptr, s3, t3, scale,
                                                                                          shift, ld_aff);
  B2_CHECK_LAUNCH("se_fc_kernel<1>");
  return B2_OK;
}

}  // extern "C"
