// b2_wgrad.cu -- weight gradient of a convolution (the backward of nn.Conv3d's weight, resnet3D.py:91-143) on wgmma:
//     G[co][ci][tap] = sum_{n, p} g[n, p][co] * x[n, s * p + tap - pad][ci]
// for 1x1x1 and 3x3x3 filters at stride 1 or 2, fp16 operands, fp32 accumulation.
//
// Both operands are read in their natural channels-last layout [positions][channels]: a block of 64 output positions of g
// and the matching (shifted, strided) 64 input positions of x arrive as two SWIZZLE_128B TMA boxes and feed the MMA as
// MN-major tiles (A = g^T, B = x^T, the K dimension of the product is the position).  A position block is a whole 8 x 8
// (h, w) sub-box of one frame of one clip, so the x box of a tap is a single 5-D TMA box (elementStrides 2 for stride 2,
// out-of-range rows / columns read as zero = the padding); g positions outside the frame read as zero and contribute
// nothing.  CTA = 128 output channels x 128 input channels of one tap, two consumer warpgroups (64 output channels each,
// accumulators in registers) and one TMA producer warp.
//
// Split-K over position blocks is deterministic: split j writes its partial G to its own slice of a caller-provided
// workspace, and a second kernel sums the slices in a fixed order, divides the loss scale out and writes
//     dw[co][ci][tap] = scale[co] * G[co][ci][tap] / loss_scale        (nn.Conv3d.weight layout, fp32)
//     wdot[co]        = <w[co], G[co]> / loss_scale                    (the BatchNorm gamma gradient needs this dot product)
#include "b2_host.h"
#include "b2_ptx.cuh"

namespace b2 {

constexpr int kWgThreads = 288;           // warps 0-7: two consumer warpgroups, warp 8: TMA producer
constexpr int kWgStages = 4;
constexpr int kWgTileBytes = 8192;        // one [64 positions][64 channels] fp16 box
constexpr int kWgStageBytes = 4 * kWgTileBytes;   // g: 128 output channels, x: 128 input channels
constexpr int kWgSmem = kWgStages * kWgStageBytes + 1024 + 2 * kWgStages * 8;
constexpr int kWgReduceThreads = 256;

struct WgradParams {
  int Cout, Cin, taps, kh, kw;
  int To, Ho, Wo, hb, wb;      // output extent, 8 x 8 blocks per frame
  int nbox, splits;
  int stride, pad;
  float* ws;                   // [splits][taps][Cout][Cin]
};

// MN-major SWIZZLE_128B descriptor: 64-element rows 128 B apart, 8-row groups SBO = 1024 B apart, 64-wide MN blocks
// LBO = 8 KB apart (the second box of a 128-wide operand)
__device__ __forceinline__ uint64_t wg_desc_mn(uint32_t addr) {
  return desc_from(kSw128DescHi, ((addr & 0x3FFFFu) >> 4) | ((static_cast<uint32_t>(kWgTileBytes) >> 4) << 16));
}

__global__ void __launch_bounds__(kWgThreads, 1)
wgrad_kernel(const __grid_constant__ CUtensorMap tmG, const __grid_constant__ CUtensorMap tmX, const WgradParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_align<1024>(smem_raw);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + kWgStages * kWgStageBytes);
  uint64_t* empty = full + kWgStages;
  const int ci0 = blockIdx.x * 128, co0 = blockIdx.y * 128;
  const int tap = blockIdx.z % p.taps, split = blockIdx.z / p.taps;
  const int b0 = static_cast<int>(static_cast<long long>(p.nbox) * split / p.splits);
  const int b1 = static_cast<int>(static_cast<long long>(p.nbox) * (split + 1) / p.splits);
  const int warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) {
    for (int s = 0; s < kWgStages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 2);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == 8) {
    if ((threadIdx.x & 31) == 0) {
      tma_prefetch_desc(&tmG);
      tma_prefetch_desc(&tmX);
      const int dt = tap / (p.kh * p.kw), dh = (tap / p.kw) % p.kh, dw = tap % p.kw;
      for (int b = b0, i = 0; b < b1; ++b, ++i) {
        const int s = i % kWgStages;
        if (i >= kWgStages) mbar_wait(&empty[s], ((i / kWgStages) - 1) & 1);
        int q = b;
        const int wbi = q % p.wb; q /= p.wb;
        const int hbi = q % p.hb; q /= p.hb;
        const int t = q % p.To;
        const int n = q / p.To;
        const int h0 = hbi * 8, w0 = wbi * 8;
        const int xt = t * p.stride + dt - p.pad, xh = h0 * p.stride + dh - p.pad, xw = w0 * p.stride + dw - p.pad;
        uint8_t* st = smem + s * kWgStageBytes;
        mbar_expect_tx(&full[s], kWgStageBytes);
        tma_load_5d(st, &tmG, &full[s], co0, w0, h0, t, n);
        tma_load_5d(st + kWgTileBytes, &tmG, &full[s], co0 + 64, w0, h0, t, n);
        tma_load_5d(st + 2 * kWgTileBytes, &tmX, &full[s], ci0, xw, xh, xt, n);
        tma_load_5d(st + 3 * kWgTileBytes, &tmX, &full[s], ci0 + 64, xw, xh, xt, n);
      }
    }
    return;
  }

  const int wg = warp >> 2;
  float acc[64];
#pragma unroll
  for (int j = 0; j < 64; ++j) acc[j] = 0.f;
  for (int b = b0, i = 0; b < b1; ++b, ++i) {
    const int s = i % kWgStages;
    mbar_wait(&full[s], (i / kWgStages) & 1);
    const uint32_t st = smem_u32(smem + s * kWgStageBytes);
    const uint64_t da = wg_desc_mn(st + wg * kWgTileBytes), db = wg_desc_mn(st + 2 * kWgTileBytes);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_n128_ss_mn(acc, da + k * 128, db + k * 128);   // 16 positions = 2 KB per K step
    wgmma_commit();
    wgmma_wait0();
    if ((threadIdx.x & 127) == 0) mbar_arrive(&empty[s]);
  }

  // fragment -> workspace slice: thread t holds rows 16 (t / 32) + (t % 32) / 4 (+ 8), column pairs 8 j + 2 (t % 4)
  const int wt = threadIdx.x & 127;
  const int row = co0 + wg * 64 + (wt >> 5) * 16 + ((wt & 31) >> 2);
  float* out = p.ws + (static_cast<size_t>(split) * p.taps + tap) * p.Cout * p.Cin;
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int col = ci0 + 8 * j + 2 * (wt & 3);
    if (col >= p.Cin) continue;
    if (row < p.Cout) *reinterpret_cast<float2*>(out + static_cast<size_t>(row) * p.Cin + col) = make_float2(acc[4 * j], acc[4 * j + 1]);
    if (row + 8 < p.Cout)
      *reinterpret_cast<float2*>(out + static_cast<size_t>(row + 8) * p.Cin + col) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
  }
}

// One CTA per output channel: fixed-order sum over the split slices, loss scale and BN scale applied, <w, G> reduced in a
// fixed order (warp shuffles, then the 8 warp sums by one thread).
__global__ void __launch_bounds__(kWgReduceThreads)
wgrad_reduce_kernel(const float* __restrict__ ws, int splits, int Cout, int Cin, int taps, const float* __restrict__ w,
                    const float* __restrict__ scale, const float* __restrict__ inv_loss_scale, float* __restrict__ dw,
                    float* __restrict__ wdot) {
  __shared__ float part[kWgReduceThreads / 32];
  const int co = blockIdx.x;
  const float inv = inv_loss_scale ? *inv_loss_scale : 1.f;
  const float sc = scale ? scale[co] : 1.f;
  const int n = Cin * taps;
  const size_t slice = static_cast<size_t>(Cout) * Cin;
  float dot = 0.f;
  for (int i = threadIdx.x; i < n; i += kWgReduceThreads) {
    const int tap = i / Cin, ci = i - tap * Cin;       // ci fastest: consecutive threads read consecutive workspace words
    const float* src = ws + static_cast<size_t>(tap) * slice + static_cast<size_t>(co) * Cin + ci;
    float g = 0.f;
    for (int j = 0; j < splits; ++j) g += src[static_cast<size_t>(j) * taps * slice];
    g *= inv;
    const size_t o = static_cast<size_t>(co) * n + static_cast<size_t>(ci) * taps + tap;
    dw[o] = sc * g;
    if (w) dot += w[o] * g;
  }
  if (!wdot) return;
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) dot += __shfl_down_sync(0xffffffffu, dot, off);
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = dot;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int j = 0; j < kWgReduceThreads / 32; ++j) t += part[j];
    wdot[co] = t;
  }
}

struct WgradPlan {
  int To, Ho, Wo, nbox, tiles, splits;
};

static WgradPlan wgrad_plan(int N, int T, int H, int W, int Cin, int Cout, int k, int stride, int pad) {
  WgradPlan q;
  q.To = (T + 2 * pad - k) / stride + 1;
  q.Ho = (H + 2 * pad - k) / stride + 1;
  q.Wo = (W + 2 * pad - k) / stride + 1;
  q.nbox = N * q.To * ((q.Ho + 7) / 8) * ((q.Wo + 7) / 8);
  q.tiles = ((Cin + 127) / 128) * ((Cout + 127) / 128) * k * k * k;
  // enough CTAs for two waves over the SMs, at least 4 position blocks per split (pipeline fill), at most 64 slices
  int s = (2 * sm_count() + q.tiles - 1) / q.tiles;
  s = s < q.nbox / 4 ? s : q.nbox / 4;
  s = s < 64 ? s : 64;
  q.splits = s > 1 ? s : 1;
  return q;
}

}  // namespace b2

using namespace b2;

extern "C" {

size_t b2_conv_wgrad_workspace_elems(int N, int T, int H, int W, int Cin, int Cout, int k, int stride, int pad) {
  if (N <= 0 || T <= 0 || H <= 0 || W <= 0 || Cin <= 0 || Cout <= 0 || k <= 0 || stride <= 0) return 0;
  const WgradPlan q = wgrad_plan(N, T, H, W, Cin, Cout, k, stride, pad);
  return static_cast<size_t>(q.splits) * k * k * k * Cout * Cin;
}

int b2_conv_wgrad(const void* g, int ldg, const void* x, int ldx, const float* w, const float* scale, const float* inv_loss_scale,
                  float* dw, float* wdot, float* ws, size_t ws_elems, int N, int T, int H, int W, int Cin, int Cout, int k,
                  int stride, int pad, void* stream) {
  B2_CHECK_ARG(g && x && dw && ws, "null pointer");
  B2_CHECK_ARG(!wdot || w, "wdot needs the weight");
  B2_CHECK_ARG(N > 0 && T > 0 && H > 0 && W > 0 && Cin > 0 && Cout > 0, "non-positive dimension");
  B2_CHECK_ARG((k == 1 && pad == 0) || (k == 3 && pad == 1), "filters are 1x1x1 (padding 0) or 3x3x3 (padding 1), got k=%d pad=%d", k, pad);
  B2_CHECK_ARG(stride == 1 || stride == 2, "stride %d is not 1 or 2", stride);
  B2_CHECK_ARG(Cin % 8 == 0 && Cout % 8 == 0 && ldg >= Cout && ldx >= Cin, "channel counts must be multiples of 8 within their pitches");
  const WgradPlan q = wgrad_plan(N, T, H, W, Cin, Cout, k, stride, pad);
  B2_CHECK_ARG(q.To > 0 && q.Ho > 0 && q.Wo > 0, "empty output");
  B2_CHECK_ARG(ws_elems >= static_cast<size_t>(q.splits) * k * k * k * Cout * Cin, "workspace too small (see b2_conv_wgrad_workspace_elems)");
  int rc;
  if ((rc = require_sm90()) != B2_OK) return rc;
  CUtensorMap tmG, tmX;
  if ((rc = make_tmap_ndhwc_5d(&tmG, g, (uint64_t)Cout, (uint64_t)ldg, (uint64_t)q.Wo, (uint64_t)q.Ho, (uint64_t)q.To, (uint64_t)N,
                               8, 8, 1)) != B2_OK)
    return rc;
  if ((rc = make_tmap_ndhwc_5d(&tmX, x, (uint64_t)Cin, (uint64_t)ldx, (uint64_t)W, (uint64_t)H, (uint64_t)T, (uint64_t)N, 8, 8,
                               (uint32_t)stride)) != B2_OK)
    return rc;
  WgradParams p;
  p.Cout = Cout; p.Cin = Cin; p.taps = k * k * k; p.kh = k; p.kw = k;
  p.To = q.To; p.Ho = q.Ho; p.Wo = q.Wo; p.hb = (q.Ho + 7) / 8; p.wb = (q.Wo + 7) / 8;
  p.nbox = q.nbox; p.splits = q.splits; p.stride = stride; p.pad = pad; p.ws = ws;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  B2_OPT_IN_SMEM(wgrad_kernel, kWgSmem);
  dim3 grid((Cin + 127) / 128, (Cout + 127) / 128, p.taps * q.splits);
  wgrad_kernel<<<grid, kWgThreads, kWgSmem, st>>>(tmG, tmX, p);
  B2_CHECK_LAUNCH("wgrad");
  wgrad_reduce_kernel<<<Cout, kWgReduceThreads, 0, st>>>(ws, q.splits, Cout, Cin, p.taps, w, scale, inv_loss_scale, dw, wdot);
  B2_CHECK_LAUNCH("wgrad_reduce");
  return B2_OK;
}

}  // extern "C"
