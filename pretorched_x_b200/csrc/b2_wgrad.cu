// b2_wgrad.cu -- weight gradient of a convolution (the backward of nn.Conv3d's / nn.Conv2d's weight, resnet3D.py:91-143 and
// torchvision's BasicBlock / Bottleneck) on wgmma:
//     G[co][ci][dt, dh, dw] = sum_{n, t, h, w} g[n, t, h, w][co] * x[n, st * t + dt - pt, s * h + dh - p, s * w + dw - p][ci]
// for kt x kh x kw filters with kt, kh = kw in {1, 3} (1x1x1, 1x3x3 -- a 2-D filter as a clip with T = 1 --, 3x3x3), temporal
// stride st and in-plane stride s in {1, 2}, fp16 operands, fp32 accumulation.
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
  int st, s, pt, p;            // temporal / in-plane stride and padding
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
        const int xt = t * p.st + dt - p.pt, xh = h0 * p.s + dh - p.p, xw = w0 * p.s + dw - p.p;
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

static WgradPlan wgrad_plan(int N, int T, int H, int W, int Cin, int Cout, int kt, int kh, int kw, int st, int s_hw, int pt,
                            int p_hw) {
  WgradPlan q;
  q.To = (T + 2 * pt - kt) / st + 1;
  q.Ho = (H + 2 * p_hw - kh) / s_hw + 1;
  q.Wo = (W + 2 * p_hw - kw) / s_hw + 1;
  q.nbox = N * q.To * ((q.Ho + 7) / 8) * ((q.Wo + 7) / 8);
  q.tiles = ((Cin + 127) / 128) * ((Cout + 127) / 128) * kt * kh * kw;
  // enough CTAs for two waves over the SMs, at least 4 position blocks per split (pipeline fill), at most 64 slices
  int s = (2 * sm_count() + q.tiles - 1) / q.tiles;
  s = s < q.nbox / 4 ? s : q.nbox / 4;
  s = s < 64 ? s : 64;
  q.splits = s > 1 ? s : 1;
  return q;
}

// ---------------------------------------------------------------------------------------------------------------------------
// Grouped weight gradient (C == K, 4 / 8 / 16 / 32 channels per group, 1 x 3 x 3 filters): every group lies inside one 64-channel
// slice, so only the diagonal 64 x 64 block of each slice and tap is computed -- one consumer warpgroup, A = g^T, B = x^T over
// the same position blocks and TMA boxes as wgrad_kernel -- 64 / cg times the algorithmic multiply-accumulates instead of the
// K x C (= groups times) of the dense product.  Workspace [splits][taps][C][64] (column = input channel within the slice); the
// reduce keeps the group's own cg columns:
//     dw[k][c_local][tap] = scale[k] * G[k][g cg + c_local][tap] / loss_scale,  wdot[k] = <w[k], G[k]> / loss_scale
// ---------------------------------------------------------------------------------------------------------------------------
constexpr int kWgdThreads = 160;          // warps 0-3: one consumer warpgroup, warp 4: TMA producer
constexpr int kWgdStageBytes = 2 * kWgTileBytes;
constexpr int kWgdSmem = kWgStages * kWgdStageBytes + 1024 + 2 * kWgStages * 8;

__global__ void __launch_bounds__(kWgdThreads, 1)
wgrad_diag_kernel(const __grid_constant__ CUtensorMap tmG, const __grid_constant__ CUtensorMap tmX, const WgradParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_align<1024>(smem_raw);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + kWgStages * kWgdStageBytes);
  uint64_t* empty = full + kWgStages;
  const int c0 = blockIdx.x * 64;
  const int tap = blockIdx.y % p.taps, split = blockIdx.y / p.taps;
  const int b0 = static_cast<int>(static_cast<long long>(p.nbox) * split / p.splits);
  const int b1 = static_cast<int>(static_cast<long long>(p.nbox) * (split + 1) / p.splits);
  const int warp = threadIdx.x >> 5;
  if (threadIdx.x == 0) {
    for (int s = 0; s < kWgStages; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], 1);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == 4) {
    if ((threadIdx.x & 31) == 0) {
      tma_prefetch_desc(&tmG);
      tma_prefetch_desc(&tmX);
      const int dh = tap / p.kw, dw = tap % p.kw;
      for (int b = b0, i = 0; b < b1; ++b, ++i) {
        const int s = i % kWgStages;
        if (i >= kWgStages) mbar_wait(&empty[s], ((i / kWgStages) - 1) & 1);
        int q = b;
        const int wbi = q % p.wb; q /= p.wb;
        const int hbi = q % p.hb; q /= p.hb;
        const int t = q % p.To;
        const int n = q / p.To;
        const int h0 = hbi * 8, w0 = wbi * 8;
        uint8_t* st = smem + s * kWgdStageBytes;
        mbar_expect_tx(&full[s], kWgdStageBytes);
        tma_load_5d(st, &tmG, &full[s], c0, w0, h0, t, n);
        tma_load_5d(st + kWgTileBytes, &tmX, &full[s], c0, w0 * p.s + dw - p.p, h0 * p.s + dh - p.p, t, n);
      }
    }
    return;
  }

  float acc[32];
#pragma unroll
  for (int j = 0; j < 32; ++j) acc[j] = 0.f;
  for (int b = b0, i = 0; b < b1; ++b, ++i) {
    const int s = i % kWgStages;
    mbar_wait(&full[s], (i / kWgStages) & 1);
    const uint32_t st = smem_u32(smem + s * kWgdStageBytes);
    const uint64_t da = wg_desc_mn(st), db = wg_desc_mn(st + kWgTileBytes);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) wgmma_n64_ss_mn(acc, da + k * 128, db + k * 128);
    wgmma_commit();
    wgmma_wait0();
    if (threadIdx.x == 0) mbar_arrive(&empty[s]);
  }

  const int wt = threadIdx.x;
  const int row = c0 + (wt >> 5) * 16 + ((wt & 31) >> 2);
  float* out = p.ws + (static_cast<size_t>(split) * p.taps + tap) * p.Cout * 64;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int col = 8 * j + 2 * (wt & 3);
    *reinterpret_cast<float2*>(out + static_cast<size_t>(row) * 64 + col) = make_float2(acc[4 * j], acc[4 * j + 1]);
    *reinterpret_cast<float2*>(out + static_cast<size_t>(row + 8) * 64 + col) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
  }
}

// One CTA per output channel, fixed-order sums as wgrad_reduce_kernel, over the cg x taps entries of the channel's own group.
__global__ void __launch_bounds__(kWgReduceThreads)
wgrad_diag_reduce_kernel(const float* __restrict__ ws, int splits, int C, int cg, int taps, const float* __restrict__ w,
                         const float* __restrict__ scale, const float* __restrict__ inv_loss_scale, float* __restrict__ dw,
                         float* __restrict__ wdot) {
  __shared__ float part[kWgReduceThreads / 32];
  const int k = blockIdx.x;
  const float inv = inv_loss_scale ? *inv_loss_scale : 1.f;
  const float sc = scale ? scale[k] : 1.f;
  const int n = cg * taps;
  const int base = (k & 63) / cg * cg;                 // the group's first input channel within the 64-channel slice
  const size_t slice = static_cast<size_t>(C) * 64;
  float dot = 0.f;
  for (int i = threadIdx.x; i < n; i += kWgReduceThreads) {
    const int tap = i / cg, cl = i - tap * cg;
    const float* src = ws + static_cast<size_t>(tap) * slice + static_cast<size_t>(k) * 64 + base + cl;
    float g = 0.f;
    for (int j = 0; j < splits; ++j) g += src[static_cast<size_t>(j) * taps * slice];
    g *= inv;
    const size_t o = static_cast<size_t>(k) * n + static_cast<size_t>(cl) * taps + tap;
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
    wdot[k] = t;
  }
}

static WgradPlan wgrad_diag_plan(int N, int T, int H, int W, int C, int s) {
  WgradPlan q = wgrad_plan(N, T, H, W, C, C, 1, 3, 3, 1, s, 0, 1);
  q.tiles = (C / 64) * 9;
  int sp = (2 * sm_count() + q.tiles - 1) / q.tiles;
  sp = sp < q.nbox / 4 ? sp : q.nbox / 4;
  sp = sp < 64 ? sp : 64;
  q.splits = sp > 1 ? sp : 1;
  return q;
}

static bool wgrad_diag_ok(int N, int T, int H, int W, int C, int groups, int s) {
  return N > 0 && T > 0 && H > 0 && W > 0 && groups > 0 && C % 64 == 0 && C % groups == 0 && (s == 1 || s == 2) &&
         (C / groups == 4 || C / groups == 8 || C / groups == 16 || C / groups == 32);
}

}  // namespace b2

using namespace b2;

extern "C" {

size_t b2_conv_wgrad_thw_workspace_elems(int N, int T, int H, int W, int Cin, int Cout, int kt, int kh, int kw, int st, int s,
                                         int pt, int p) {
  if (N <= 0 || T <= 0 || H <= 0 || W <= 0 || Cin <= 0 || Cout <= 0 || kt <= 0 || kh <= 0 || kw <= 0 || st <= 0 || s <= 0) return 0;
  const WgradPlan q = wgrad_plan(N, T, H, W, Cin, Cout, kt, kh, kw, st, s, pt, p);
  return static_cast<size_t>(q.splits) * kt * kh * kw * Cout * Cin;
}

int b2_conv_wgrad_thw(const void* g, int ldg, const void* x, int ldx, const float* w, const float* scale, const float* inv_loss_scale,
                      float* dw, float* wdot, float* ws, size_t ws_elems, int N, int T, int H, int W, int Cin, int Cout, int kt,
                      int kh, int kw, int st, int s, int pt, int p, void* stream) {
  B2_CHECK_ARG(g && x && dw && ws, "null pointer");
  B2_CHECK_ARG(!wdot || w, "wdot needs the weight");
  B2_CHECK_ARG(N > 0 && T > 0 && H > 0 && W > 0 && Cin > 0 && Cout > 0, "non-positive dimension");
  B2_CHECK_ARG((kt == 1 || kt == 3) && (kh == 1 || kh == 3) && kw == kh && pt == kt / 2 && p == kh / 2,
               "filters are kt x k x k with kt, k in {1, 3} and padding (kt / 2, k / 2, k / 2), got %dx%dx%d padding (%d, %d)", kt, kh,
               kw, pt, p);
  B2_CHECK_ARG((st == 1 || st == 2) && (s == 1 || s == 2), "strides (%d, %d) are not 1 or 2", st, s);
  B2_CHECK_ARG(Cin % 8 == 0 && Cout % 8 == 0 && ldg >= Cout && ldx >= Cin, "channel counts must be multiples of 8 within their pitches");
  const WgradPlan q = wgrad_plan(N, T, H, W, Cin, Cout, kt, kh, kw, st, s, pt, p);
  const int taps = kt * kh * kw;
  B2_CHECK_ARG(q.To > 0 && q.Ho > 0 && q.Wo > 0, "empty output");
  B2_CHECK_ARG(ws_elems >= static_cast<size_t>(q.splits) * taps * Cout * Cin, "workspace too small (see b2_conv_wgrad_thw_workspace_elems)");
  int rc;
  if ((rc = require_sm90()) != B2_OK) return rc;
  CUtensorMap tmG, tmX;
  if ((rc = make_tmap_ndhwc_5d(&tmG, g, (uint64_t)Cout, (uint64_t)ldg, (uint64_t)q.Wo, (uint64_t)q.Ho, (uint64_t)q.To, (uint64_t)N,
                               8, 8, 1)) != B2_OK)
    return rc;
  // the temporal stride needs no element stride: the x box is one frame deep and its frame index is computed per box
  if ((rc = make_tmap_ndhwc_5d(&tmX, x, (uint64_t)Cin, (uint64_t)ldx, (uint64_t)W, (uint64_t)H, (uint64_t)T, (uint64_t)N, 8, 8,
                               (uint32_t)s)) != B2_OK)
    return rc;
  WgradParams prm;
  prm.Cout = Cout; prm.Cin = Cin; prm.taps = taps; prm.kh = kh; prm.kw = kw;
  prm.To = q.To; prm.Ho = q.Ho; prm.Wo = q.Wo; prm.hb = (q.Ho + 7) / 8; prm.wb = (q.Wo + 7) / 8;
  prm.nbox = q.nbox; prm.splits = q.splits; prm.st = st; prm.s = s; prm.pt = pt; prm.p = p; prm.ws = ws;
  cudaStream_t stm = reinterpret_cast<cudaStream_t>(stream);
  B2_OPT_IN_SMEM(wgrad_kernel, kWgSmem);
  dim3 grid((Cin + 127) / 128, (Cout + 127) / 128, taps * q.splits);
  wgrad_kernel<<<grid, kWgThreads, kWgSmem, stm>>>(tmG, tmX, prm);
  B2_CHECK_LAUNCH("wgrad");
  wgrad_reduce_kernel<<<Cout, kWgReduceThreads, 0, stm>>>(ws, q.splits, Cout, Cin, taps, w, scale, inv_loss_scale, dw, wdot);
  B2_CHECK_LAUNCH("wgrad_reduce");
  return B2_OK;
}

size_t b2_conv_wgrad_grouped_workspace_elems(int N, int T, int H, int W, int C, int groups, int s) {
  if (!wgrad_diag_ok(N, T, H, W, C, groups, s)) return 0;
  return static_cast<size_t>(wgrad_diag_plan(N, T, H, W, C, s).splits) * 9 * C * 64;
}

int b2_conv_wgrad_grouped_plan(int N, int T, int H, int W, int C, int groups, int s, long long* executed_macs, long long* algorithmic_macs,
                               int* splits) {
  B2_CHECK_ARG(executed_macs && algorithmic_macs && splits, "null pointer");
  if (!wgrad_diag_ok(N, T, H, W, C, groups, s))
    return set_error(B2_ERR_UNSUPPORTED, "grouped weight gradient needs C %% 64 == 0, 4 / 8 / 16 / 32 channels per group, stride 1 or 2");
  const WgradPlan q = wgrad_diag_plan(N, T, H, W, C, s);
  *executed_macs = static_cast<long long>(q.nbox) * 64 * 9 * (C / 64) * 64 * 64;
  *algorithmic_macs = static_cast<long long>(N) * T * q.Ho * q.Wo * 9 * C * (C / groups);
  *splits = q.splits;
  return B2_OK;
}

int b2_conv_wgrad_grouped(const void* g, int ldg, const void* x, int ldx, const float* w, const float* scale, const float* inv_loss_scale,
                          float* dw, float* wdot, float* ws, size_t ws_elems, int N, int T, int H, int W, int C, int groups, int s,
                          void* stream) {
  set_last_kernel(KID_NONE);
  B2_CHECK_ARG(g && x && dw && ws, "null pointer");
  B2_CHECK_ARG(!wdot || w, "wdot needs the weight");
  if (!wgrad_diag_ok(N, T, H, W, C, groups, s))
    return set_error(B2_ERR_UNSUPPORTED, "grouped weight gradient needs C %% 64 == 0, 4 / 8 / 16 / 32 channels per group and stride 1 "
                                         "or 2 (got C=%d groups=%d stride %d)", C, groups, s);
  B2_CHECK_ARG(ldg >= C && ldx >= C && ldg % 8 == 0 && ldx % 8 == 0, "pitches must be multiples of 8 and >= C");
  const WgradPlan q = wgrad_diag_plan(N, T, H, W, C, s);
  B2_CHECK_ARG(q.Ho > 0 && q.Wo > 0, "empty output");
  B2_CHECK_ARG(ws_elems >= static_cast<size_t>(q.splits) * 9 * C * 64, "workspace too small (see b2_conv_wgrad_grouped_workspace_elems)");
  int rc;
  if ((rc = require_sm90()) != B2_OK) return rc;
  CUtensorMap tmG, tmX;
  if ((rc = make_tmap_ndhwc_5d(&tmG, g, (uint64_t)C, (uint64_t)ldg, (uint64_t)q.Wo, (uint64_t)q.Ho, (uint64_t)T, (uint64_t)N, 8, 8, 1)) !=
      B2_OK)
    return rc;
  if ((rc = make_tmap_ndhwc_5d(&tmX, x, (uint64_t)C, (uint64_t)ldx, (uint64_t)W, (uint64_t)H, (uint64_t)T, (uint64_t)N, 8, 8,
                               (uint32_t)s)) != B2_OK)
    return rc;
  WgradParams prm;
  prm.Cout = C; prm.Cin = C; prm.taps = 9; prm.kh = 3; prm.kw = 3;
  prm.To = T; prm.Ho = q.Ho; prm.Wo = q.Wo; prm.hb = (q.Ho + 7) / 8; prm.wb = (q.Wo + 7) / 8;
  prm.nbox = q.nbox; prm.splits = q.splits; prm.st = 1; prm.s = s; prm.pt = 0; prm.p = 1; prm.ws = ws;
  cudaStream_t stm = reinterpret_cast<cudaStream_t>(stream);
  B2_OPT_IN_SMEM(wgrad_diag_kernel, kWgdSmem);
  wgrad_diag_kernel<<<dim3(C / 64, 9 * q.splits), kWgdThreads, kWgdSmem, stm>>>(tmG, tmX, prm);
  B2_CHECK_LAUNCH("wgrad_diag");
  wgrad_diag_reduce_kernel<<<C, kWgReduceThreads, 0, stm>>>(ws, q.splits, C, C / groups, 9, w, scale, inv_loss_scale, dw, wdot);
  B2_CHECK_LAUNCH("wgrad_diag_reduce");
  set_last_kernel(KID_WGRAD_GROUPED, C / groups, q.splits, q.nbox);
  return B2_OK;
}

size_t b2_conv_wgrad_workspace_elems(int N, int T, int H, int W, int Cin, int Cout, int k, int stride, int pad) {
  return b2_conv_wgrad_thw_workspace_elems(N, T, H, W, Cin, Cout, k, k, k, stride, stride, pad, pad);
}

int b2_conv_wgrad(const void* g, int ldg, const void* x, int ldx, const float* w, const float* scale, const float* inv_loss_scale,
                  float* dw, float* wdot, float* ws, size_t ws_elems, int N, int T, int H, int W, int Cin, int Cout, int k,
                  int stride, int pad, void* stream) {
  B2_CHECK_ARG((k == 1 && pad == 0) || (k == 3 && pad == 1), "filters are 1x1x1 (padding 0) or 3x3x3 (padding 1), got k=%d pad=%d", k, pad);
  return b2_conv_wgrad_thw(g, ldg, x, ldx, w, scale, inv_loss_scale, dw, wdot, ws, ws_elems, N, T, H, W, Cin, Cout, k, k, k, stride,
                           stride, pad, pad, stream);
}

}  // extern "C"
