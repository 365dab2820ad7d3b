// b2_tstack.cuh -- purely temporal (kt,1,1) stride-1 "same" convolution with <= 64 output channels: the second half of every
// SpatioTemporalConv of R(2+1)D whose output is 64 wide (r2plus1d.py:85-88 -- the stem's (7,1,1) C110->64 and the twelve
// (3,1,1) C144->64 of layer1 in R(2+1)D-34), with the outer BN / residual / ReLU in the epilogue.
//
// Why its own kernel.  With Cout = 64 a 128 x 64 x 16 MMA is bound by the A-operand feed from shared memory, not by math, so the
// slab kernel -- one N = 64 MMA per (temporal tap, K step) -- pays that feed once per tap.  An input frame f contributes to the output frames f-pt .. f+pt through the
// taps dt = kt-1 .. 0 with the SAME A tile (128 positions x 64 channels of frame f), so here the accumulators of G = 2 consecutive
// output frames sit side by side in the accumulator tile ([slot][64 columns]) and the weights are stacked [W(dt=kt-1); ...; W(dt=0)]
// (64 rows each): the slots an input frame feeds are a CONTIGUOUS row range of that stack and a contiguous column range of the
// accumulator tile, and one MMA of N = 64 x (slots fed) <= 128 replaces up to two N = 64 MMAs on the same A tile.
// b2_slabts.cuh does the same for 3 x kh x kw filters but streams a 24 KB weight stack per (tap, input frame) from L2, which is what
// made it lose on 1x1 in-plane filters.  Here the in-plane filter is 1x1: the whole filter is
// kt x ceil(C/64) blocks of 8 KB (72 KB for C144, 112 KB for C110 x 7 taps) and stays RESIDENT in shared memory, loaded once per CTA
// before griddepcontrol.wait (weights do not depend on the previous kernel); A tiles are plain [128 positions][64 channels] TMA boxes
// (no halo, rows past the end of a frame zero-filled).  The accumulator tile (128 x 128 fp32, 66 KB) shares the 227 KB of shared
// memory with the resident filter (up to 112 KB) and a 2-stage A ring, which is what bounds G and leaves room for one set only.
//
//   warp 12      TMA producer: resident weights once, then the A tiles of (item, input frame, channel chunk) through the ring
//   warps 8-11   MMA warpgroup: per input frame one MMA of N = 64 x slots per K step; all MMAs accumulate
//                (the epilogue hands the accumulators back zeroed, so slots may start from different input frames)
//   warps 0-7    epilogue: thread = one position (accumulator row) x 32 channels; affine (+ residual) (+ ReLU), 16-byte stores
#pragma once

#include "b2_ptx.cuh"

namespace b2 {

constexpr int kTkThreads = 416;
constexpr int kTkMmaWarp0 = 8;
constexpr int kTkTmaWarp = 12;
constexpr int kTkStages = 2;                 // A-tile ring depth
constexpr int kTkABytes = 128 * 128;         // one A tile: 128 positions x 64 fp16 channels, SWIZZLE_128B
constexpr int kTkG = 2;                      // output frames (accumulator slots) per work item
constexpr int kTkSetCols = kTkG * 64;        // accumulator columns
constexpr int kTkWBlock = 64 * 128;          // one (channel chunk, temporal tap) weight block: 64 output rows x 128 B

struct TstackParams {
  int T, HW, C;            // frames per clip, positions per frame, channel pitch of x
  int kt, pt;              // temporal taps and padding (stride 1, 2 * pt == kt - 1: To == T)
  int cchunks;             // ceil(C / 64)
  int groups;              // ceil(T / kTkG) frame groups per clip
  int tiles_q;             // ceil(HW / 128) position tiles per frame
  int items_total;         // N * groups * tiles_q
  int Ncols, ldy, ldr, relu;
  const float* scale;
  const float* shift;
  const __half* residual;  // nullable, dense [M][ldr]
  __half* y;               // dense [M][ldy]
  FastDiv fd_tiles_q, fd_groups;
};

struct TstackItem {
  int q0;                  // first position of the tile inside its frame
  int plane_o0;            // first output plane (n * T + to0) of the group
  int plane_i0;            // input plane of relative frame 0 (= to0 - pt; may lie before the clip: such frames are skipped)
  int nf;                  // output frames of the group that exist (1 .. kTkG)
  int fr_lo, fr_hi;        // relative input frames inside the clip
};

__device__ __forceinline__ TstackItem tstack_item(const TstackParams& p, int item) {
  TstackItem w;
  const int pg = fdiv(item, p.fd_tiles_q);            // (clip, frame group); position tile fastest
  w.q0 = (item - pg * p.tiles_q) * 128;
  const int n = fdiv(pg, p.fd_groups), g = pg - n * p.groups;
  const int to0 = g * kTkG;
  w.nf = min(kTkG, p.T - to0);
  w.plane_o0 = n * p.T + to0;
  w.plane_i0 = n * p.T + to0 - p.pt;
  w.fr_lo = max(0, p.pt - to0);                        // absolute frame to0 - pt + fr >= 0
  w.fr_hi = min(w.nf + p.kt - 2, p.T - 1 - to0 + p.pt);   // last frame any slot reads, clipped to the clip
  return w;
}

__global__ void __launch_bounds__(kTkThreads, 1)
tstack_kernel(const __grid_constant__ CUtensorMap tmX,   // input as (C, HW, 1, N*T), box (64, 128, 1, 1)
              const __grid_constant__ CUtensorMap tmB,   // weights [K][kt*C], box (64 columns, 64 rows)
              const TstackParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_align<1024>(smem_raw);
  uint8_t* a_base = smem;
  uint8_t* w_base = smem + kTkStages * kTkABytes;
  uint8_t* tail = w_base + p.cchunks * p.kt * kTkWBlock;
  uint64_t* a_full = reinterpret_cast<uint64_t*>(tail);
  uint64_t* a_empty = a_full + kTkStages;
  uint64_t* w_full = a_empty + kTkStages;             // [1]
  uint64_t* acc_full = w_full + 1;                    // [1]
  uint64_t* acc_empty = acc_full + 1;                 // [1]
  float* s_scale = reinterpret_cast<float*>(tail + 128);   // barriers occupy the first 64 bytes
  float* s_shift = s_scale + 64;
  const AccTile at{reinterpret_cast<float*>(tail + 128 + 512), acc_ld(kTkSetCols)};

  const int tid = threadIdx.x, warp = tid >> 5;

  if (tid == 128) {
    for (int s = 0; s < kTkStages; ++s) { mbar_init(&a_full[s], 1); mbar_init(&a_empty[s], 1); }
    mbar_init(&w_full[0], 1);
    mbar_init(acc_full, 1); mbar_init(acc_empty, 256);
    fence_mbar_init();
    tma_prefetch_desc(&tmX);
    tma_prefetch_desc(&tmB);
  }
  if (tid < 64) {
    s_scale[tid] = (tid < p.Ncols) ? __ldg(&p.scale[tid]) : 0.f;
    s_shift[tid] = (tid < p.Ncols) ? __ldg(&p.shift[tid]) : 0.f;
  }
  __syncthreads();
  pdl_launch_dependents();
  if (warp == kTkTmaWarp) {
    // resident filter: block (cc, r) holds W(dt = kt-1-r) for channels [64 cc, 64 cc + 64); rows >= K and columns past the
    // tensor's extent are zero-filled by TMA (columns past C inside a tap hold the next tap's weights: the activation side
    // zero-fills channels >= C and the K loop stops at the last 16-channel step that holds real channels)
    if (elect_one()) {
      mbar_expect_tx(&w_full[0], static_cast<uint32_t>(p.cchunks * p.kt * kTkWBlock));
      for (int cc = 0; cc < p.cchunks; ++cc)
        for (int dt = 0; dt < p.kt; ++dt)
          tma_load_2d(w_base + (cc * p.kt + (p.kt - 1 - dt)) * kTkWBlock, &tmB, &w_full[0], dt * p.C + cc * 64, 0);
    }
    __syncwarp();
  }
  pdl_wait();                       // everything above touched only weights / on-chip state

  if (warp == kTkTmaWarp) {
    // ================================ TMA producer ======================================
    int it = 0;
    for (int item = blockIdx.x; item < p.items_total; item += gridDim.x) {
      const TstackItem w = tstack_item(p, item);
      for (int fr = w.fr_lo; fr <= w.fr_hi; ++fr) {
        for (int cc = 0; cc < p.cchunks; ++cc, ++it) {
          const int s = it % kTkStages;
          mbar_wait(&a_empty[s], ((it / kTkStages) & 1) ^ 1);
          if (elect_one()) {
            mbar_expect_tx(&a_full[s], static_cast<uint32_t>(kTkABytes));
            tma_load_4d(a_base + s * kTkABytes, &tmX, &a_full[s], cc * 64, w.q0, 0, w.plane_i0 + fr);
          }
          __syncwarp();
        }
      }
    }
  } else if (warp >= kTkMmaWarp0) {
    // ================================ MMA warpgroup =====================================
    const uint32_t a0s = smem_u32(a_base), w0s = smem_u32(w_base);
    mbar_wait(&w_full[0], 0);
    int it = 0, lt = 0;
    for (int item = blockIdx.x; item < p.items_total; item += gridDim.x, ++lt) {
      const TstackItem w = tstack_item(p, item);
      mbar_wait(acc_empty, lt & 1);                        // the epilogue has drained AND re-zeroed the accumulators
      for (int fr = w.fr_lo; fr <= w.fr_hi; ++fr) {
        const int s_lo = max(0, fr - (p.kt - 1)), s_hi = min(w.nf - 1, fr);   // output slots this input frame feeds (>= 1)
        const int r0 = p.kt - 1 - (fr - s_lo);                              // first block of the stack: dt = fr - s_lo
        for (int cc = 0; cc < p.cchunks; ++cc, ++it) {
          const int ksteps = min(4, (p.C - cc * 64 + 15) >> 4);              // 16-channel K steps that hold real channels
          const int s = it % kTkStages;
          mbar_wait(&a_full[s], (it / kTkStages) & 1);
          const uint32_t a_lo = sw128_desc_lo(a0s + s * kTkABytes);
          const uint32_t b_lo = sw128_desc_lo(w0s + (cc * p.kt + r0) * kTkWBlock);
          wg_mma(at, s_lo * 64, (s_hi - s_lo + 1) * 64, wg_sw128(desc_from(kSw128DescHi, a_lo), desc_from(kSw128DescHi, b_lo)), ksteps,
                 true);
          wg_sync();
          wg_arrive(&a_empty[s]);
          if (fr == w.fr_hi && cc == p.cchunks - 1) wg_arrive(acc_full);
        }
      }
    }
  } else {
    // ================================ epilogue ==========================================
    // thread = accumulator row; the two warpgroups split the 64 channels of a slot
    const int erow = (warp & 3) * 32 + (tid & 31);
    const int egroup = warp >= 4 ? 1 : 0;
    const int c0 = egroup * 32;
    for (int c = c0; c < kTkSetCols; c += 64) acc_zero32(at, erow, c);     // the accumulators start at zero (this group's chunks)
    mbar_arrive(acc_empty);
    float sc[32], sh[32];
#pragma unroll
    for (int c = 0; c < 32; ++c) { sc[c] = s_scale[c0 + c]; sh[c] = s_shift[c0 + c]; }
    const int ncols_here = min(64, p.ldy);
    int lt = 0;
    for (int item = blockIdx.x; item < p.items_total; item += gridDim.x, ++lt) {
      const TstackItem w = tstack_item(p, item);
      const bool ok = w.q0 + erow < p.HW;
      const size_t row0 = static_cast<size_t>(w.plane_o0) * p.HW + w.q0 + erow;     // slot s: + s * HW
      // residual rows of both slots are requested before the accumulators are complete
      uint4 rres[kTkG][4];
      auto load_res = [&](int s) {
        if (p.residual && ok && s < w.nf) {
          const __half* rrow = p.residual + (row0 + static_cast<size_t>(s) * p.HW) * p.ldr + c0;
#pragma unroll
          for (int c8 = 0; c8 < 4; ++c8)
            if (c0 + c8 * 8 < ncols_here) rres[s][c8] = __ldg(reinterpret_cast<const uint4*>(rrow + c8 * 8));
        }
      };
      load_res(0);
      load_res(1);
      mbar_wait(acc_full, lt & 1);
#pragma unroll
      for (int s = 0; s < kTkG; ++s) {
        if (s < w.nf) {                                      // warp-uniform
          uint32_t v[32];
          acc_ld32(at, erow, s * 64 + c0, v);
          if (ok) {
            __half* yrow = p.y + (row0 + static_cast<size_t>(s) * p.HW) * p.ldy + c0;
#pragma unroll
            for (int c8 = 0; c8 < 4; ++c8) {
              if (c0 + c8 * 8 < ncols_here) {
                uint32_t rr[4] = {0u, 0u, 0u, 0u};
                if (p.residual) {
                  const uint4 rv = rres[s][c8];
                  rr[0] = rv.x; rr[1] = rv.y; rr[2] = rv.z; rr[3] = rv.w;
                }
                uint32_t o[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                  const int c = c8 * 8 + e * 2;
                  const float2 rf = unpack_half2(rr[e]);
                  float a0 = fmaf(__uint_as_float(v[c]), sc[c], sh[c]) + rf.x;       // residual added in fp32 before the single rounding
                  float a1 = fmaf(__uint_as_float(v[c + 1]), sc[c + 1], sh[c + 1]) + rf.y;
                  if (p.relu) { a0 = fmaxf(a0, 0.f); a1 = fmaxf(a1, 0.f); }
                  o[e] = pack_half2(a0, a1);
                }
                *reinterpret_cast<uint4*>(yrow + c8 * 8) = make_uint4(o[0], o[1], o[2], o[3]);
              }
            }
          }
        }
      }
      for (int c = c0; c < kTkSetCols; c += 64) acc_zero32(at, erow, c);   // hand the accumulators back zeroed (this group's chunks)
      mbar_arrive(acc_empty);
    }
  }
}

}  // namespace b2
