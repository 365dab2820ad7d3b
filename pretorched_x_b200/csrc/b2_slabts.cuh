// b2_slabts.cuh -- 3 x kh x kw "same" convolution with <= 64 output channels, temporal-group form of the slab kernel.
//
// The slab kernel (b2_slabconv.cuh) reads the A tile of every (dt, dh, dw) tap from shared memory for an MMA of N = Cout columns.
// With Cout = 64 a 128 x 64 x 16 MMA moves 4 KB of A + 2 KB of B per 32 math cycles: it is shared-memory-operand bound.  An input frame f contributes to the three output
// frames f-1, f, f+1 through the temporal taps dt = 2, 1, 0 with the SAME in-plane shift, so here a work item owns a group of three
// consecutive output frames (to0, to0+1, to0+2) of one spatial tile and walks the five input frames to0-1 .. to0+3:
//     input frame (relative) fr = 0..4 feeds output slots s in [max(0, fr-2), min(2, fr)] with temporal tap dt = fr - s,
// and since the weight stage holds the taps stacked as [W(dt=2); W(dt=1); W(dt=0)] (192 rows), the slots fed by one input frame are
// a CONTIGUOUS row range of that stack and a contiguous column range of the accumulator [tile][slot][64]: one MMA of N = 64, 128 or
// 192 per (in-plane tap, K step) instead of one N = 64 MMA per (temporal tap, in-plane tap, K step).  Five A tiles are read where the
// plain form reads nine, and the operand bytes per MMA column drop from 96 to 53 (N = 192): 304 instead of 432 shared-memory cycles
// per in-plane tap.  Accumulators start from zero, so every MMA accumulates and slots may receive their first contribution from
// different input frames.
//
// Same building blocks as the slab kernel: 4-D TMA halo slabs (SWIZZLE_128B, zero-filled padding), shifted descriptors for the
// in-plane taps, persistent CTAs, TMA producer warp / two consumer warpgroups with register accumulators / 3 epilogue warps.  The
// 3 x 64 accumulator columns of one M tile take 192 of the kSlabAccCols register columns, so an item is a single M tile (MT = 1).
// Stride 1, kt = 3, pt = 1, plain per-channel affine.
#pragma once

#include "b2_slabconv.cuh"

namespace b2 {

constexpr int kTsGroup = 3;          // output frames per work item
constexpr int kTsBN = 64;            // output-channel tile
constexpr int kTsWBytes = 3 * kTsBN * 128;   // weight stage: [W(dt=2); W(dt=1); W(dt=0)], 64 rows x 128 B each

struct SlabTsItem {
  int q0, wc, plane_o0, plane_i0, r_lo;             // plane_o0: first output plane of the group; plane_i0: input plane of relative frame 0
  int nf;                                           // valid output frames in the group (1..3)
  int fr_lo, fr_hi;                                 // valid relative input frames (inside the clip)
  int n_slabs;
};

// SlabParams fields reused: T, C, To, Ho, Wo, khw, cchunks, PW, WC, wchunks, halo_l, R, sub_* [0], reach, slab_bytes, P, Ncols,
// tiles_q, items_total, scale, shift, residual, ldr, y, ldy, relu, naff, fd_tiles_q, fd_wchunks, fd_PW; fd_To divides by the number
// of frame groups per clip (ceil(To / 3)), tiles_n == 1.
__device__ __forceinline__ SlabTsItem slabts_item(const SlabParams& p, int item) {
  SlabTsItem w;
  int t = fdiv(item, p.fd_tiles_q);
  const int tq = item - t * p.tiles_q; item = t;
  const int pg = fdiv(item, p.fd_wchunks);           // (clip, frame group)
  w.wc = item - pg * p.wchunks;
  const int n = fdiv(pg, p.fd_To), g = pg - n * p.fd_To.d;
  const int to0 = g * kTsGroup;
  w.nf = min(kTsGroup, p.To - to0);
  w.plane_o0 = n * p.To + to0;
  w.plane_i0 = n * p.T + to0 - 1;                    // relative input frame 0 = to0 - pt
  w.fr_lo = max(0, 1 - to0);
  w.fr_hi = min(w.nf + 1, p.T - to0);                // absolute frame to0 - 1 + fr < T
  w.n_slabs = p.cchunks * (w.fr_hi - w.fr_lo + 1);
  w.q0 = tq * 128;
  const int lo = w.q0 - p.reach;
  w.r_lo = (lo >= 0) ? fdiv(lo, p.fd_PW) : -fdiv(-lo + p.PW - 1, p.fd_PW);
  return w;
}

static_assert(kTsGroup * kTsBN <= kSlabAccCols, "slabts: one M tile of accumulators per item");

__global__ void __launch_bounds__(kSlabThreads, 1)
slabts_kernel(const __grid_constant__ CUtensorMap tmX,   // input as (C, W, H, N*T), box (64, PW, R, 1)
              const __grid_constant__ CUtensorMap tmB,   // weights [Ncols][taps*C], box (64, 64)
              const SlabParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_align<1024>(smem_raw);
  uint8_t* slab_base = smem;
  uint8_t* w_base = smem + kSlabSStages * p.slab_bytes;
  uint8_t* tail = w_base + kSlabWStages * kTsWBytes;
  uint64_t* slab_full = reinterpret_cast<uint64_t*>(tail);
  uint64_t* slab_empty = slab_full + kSlabSStages;
  uint64_t* w_full = slab_empty + kSlabSStages;
  uint64_t* w_empty = w_full + kSlabWStages;
  uint64_t* acc_full = w_empty + kSlabWStages;
  uint64_t* acc_empty = acc_full + 1;
  float* s_scale = reinterpret_cast<float*>(tail + 256);
  float* s_shift = s_scale + p.naff;

  const int tid = threadIdx.x, warp = tid >> 5;
  constexpr int tile_cols = kTsGroup * kTsBN;        // accumulator columns of the item's M tile: [slot][64]
  const AccTile at{s_shift + p.naff, acc_ld(tile_cols)};

  if (tid == 0) {
    for (int s = 0; s < kSlabSStages; ++s) { mbar_init(&slab_full[s], 1); mbar_init(&slab_empty[s], kSlabConsumerWarps); }
    for (int s = 0; s < kSlabWStages; ++s) { mbar_init(&w_full[s], 1); mbar_init(&w_empty[s], kSlabConsumerWarps); }
    mbar_init(acc_full, 32 * kSlabConsumerWarps);
    mbar_init(acc_empty, 32 * kSlabEpiWarps);
    fence_mbar_init();
    tma_prefetch_desc(&tmX);
    tma_prefetch_desc(&tmB);
  }
  for (int i = tid; i < p.naff; i += kSlabThreads) {
    s_scale[i] = (i < p.Ncols) ? __ldg(&p.scale[i]) : 0.f;
    s_shift[i] = (i < p.Ncols) ? __ldg(&p.shift[i]) : 0.f;
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();

  if (warp == kSlabTmaWarp) {
    // ================================ TMA producer ======================================
    int wit = 0, sg = 0;
    int item = blockIdx.x;
    if (item < p.items_total) {
      SlabTsItem cur = slabts_item(p, item);
      int nxt_item = item, nxt_si = 0;
      SlabTsItem nxt = cur;
      // slab index si of an item enumerates (cc, fr) with fr fastest
      auto load_next = [&]() {
        const int nfr = nxt.fr_hi - nxt.fr_lo + 1;
        const int cc = nxt_si / nfr, fr = nxt.fr_lo + (nxt_si - cc * nfr);
        const int s = sg % kSlabSStages;
        mbar_wait(&slab_empty[s], ((sg / kSlabSStages) & 1) ^ 1);
        if (elect_one()) {
          mbar_expect_tx(&slab_full[s], static_cast<uint32_t>(p.R * p.PW * 128));
          tma_load_4d(slab_base + s * p.slab_bytes, &tmX, &slab_full[s], cc * 64, p.sub_w0[0] + nxt.wc * p.WC, nxt.r_lo + p.sub_h0[0],
                      nxt.plane_i0 + fr);
        }
        __syncwarp();
        ++sg;
        if (++nxt_si == nxt.n_slabs) {
          nxt_si = 0;
          nxt_item += gridDim.x;
          if (nxt_item < p.items_total) nxt = slabts_item(p, nxt_item);
        }
      };
      load_next();
      const int ntaps = p.sub_ntaps[0];
      for (; item < p.items_total; item += gridDim.x) {
        cur = slabts_item(p, item);
        const int nfr = cur.fr_hi - cur.fr_lo + 1;
        for (int si = 0; si < cur.n_slabs; ++si) {
          const int cc = si / nfr;
          const int pf = min(kSlabWStages, ntaps - 1);      // (ntaps >= 9: the previous slab has retired by then, see b2_slabconv.cuh)
          for (int ti = 0; ti < ntaps; ++ti, ++wit) {
            if (ti == pf && nxt_item < p.items_total) load_next();
            const int ws = wit % kSlabWStages;
            mbar_wait(&w_empty[ws], ((wit / kSlabWStages) & 1) ^ 1);
            const int tap_hw = p.sub_tap[0][ti];
            if (elect_one()) {
              mbar_expect_tx(&w_full[ws], static_cast<uint32_t>(kTsWBytes));
#pragma unroll
              for (int dt = 0; dt < 3; ++dt)      // stacked [W(dt=2); W(dt=1); W(dt=0)]: temporal tap dt lands in row block 2 - dt
                tma_load_2d(w_base + ws * kTsWBytes + (2 - dt) * (kTsBN * 128), &tmB, &w_full[ws], (dt * p.khw + tap_hw) * p.C + cc * 64, 0);
            }
            __syncwarp();
          }
        }
      }
    }
  } else if (warp < kSlabEpiWarp0) {
    // ================================ consumer warpgroups ===============================
    // warpgroup wg owns rows [64 wg, 64 wg + 64) of the tile; slot s of the accumulator sits at fragment columns [64 s, 64 s + 64)
    float acc[tile_cols / 2];
    const int wg = tid >> 7;
    const bool lead = (tid & 31) == 0;
    const uint32_t slab0 = smem_u32(slab_base), w0s = smem_u32(w_base);
    const uint32_t a_wg = static_cast<uint32_t>(wg) * (64u * 128u >> 4);
    const int ntaps = p.sub_ntaps[0];
    int wit = 0, sg = 0, lt = 0;
    for (int item = blockIdx.x; item < p.items_total; item += gridDim.x, ++lt) {
      const SlabTsItem w = slabts_item(p, item);
#pragma unroll
      for (int k = 0; k < tile_cols / 2; ++k) acc[k] = 0.f;
      reg_fence(acc);
      int prev_ws = -1, prev_s = -1;
      const int nfr = w.fr_hi - w.fr_lo + 1;
      for (int si = 0; si < w.n_slabs; ++si, ++sg) {
        const int cc = si / nfr, fr = w.fr_lo + (si - cc * nfr);
        const int s_lo = warp_uniform(max(0, fr - 2)), s_hi = warp_uniform(min(w.nf - 1, fr));          // output slots this input frame feeds
        const uint32_t b_row = static_cast<uint32_t>(2 - (fr - s_lo));      // first row block of the stack: dt = fr - s_lo
        const int ksteps = warp_uniform(min(4, (p.C - cc * 64 + 15) >> 4));
        const int s = sg % kSlabSStages;
        mbar_wait(&slab_full[s], (sg / kSlabSStages) & 1);
        const uint32_t slab_addr = slab0 + s * p.slab_bytes;
        for (int ti = 0; ti < ntaps; ++ti, ++wit) {
          const int ws = wit % kSlabWStages;
          mbar_wait(&w_full[ws], (wit / kSlabWStages) & 1);
          const int pix0 = w.q0 + p.sub_off[0][ti] - w.r_lo * p.PW;
          const uint64_t b = desc_from(kSw128DescHi, sw128_desc_lo(w0s + ws * kTsWBytes + b_row * (kTsBN * 128)));
          const uint64_t a = desc_from(kSw128DescHi, sw128_desc_lo(slab_addr + static_cast<uint32_t>(pix0) * 128u) + a_wg);
          wgmma_fence();
          // one N = 64 MMA per slot the frame feeds, B = the stack row block of its temporal tap.  (A single MMA over the slot range,
          // N = 64, 128 or 192 on overlapping fragment windows, makes ptxas serialise the kernel's whole wgmma pipeline for want of
          // registers; with the accumulators in registers the A re-reads cost less than that.)
          if (s_lo == 0) slab_mma<64>(acc, a, b, ksteps);
          if (s_lo <= 1 && s_hi >= 1) slab_mma<64>(acc + 32, a, b + (kTsBN * 128 >> 4) * (1 - s_lo), ksteps);
          if (s_hi == 2) slab_mma<64>(acc + 64, a, b + (kTsBN * 128 >> 4) * (2 - s_lo), ksteps);
          wgmma_commit();
          wgmma_wait1();
          if (lead && prev_ws >= 0) {
            mbar_arrive(&w_empty[prev_ws]);
            if (prev_s >= 0) mbar_arrive(&slab_empty[prev_s]);
          }
          prev_ws = ws;
          prev_s = (ti == ntaps - 1) ? s : -1;
        }
      }
      wgmma_wait0();
      reg_fence(acc);
      if (lead) {
        mbar_arrive(&w_empty[prev_ws]);
        mbar_arrive(&slab_empty[prev_s]);
      }
      mbar_wait(acc_empty, (lt & 1) ^ 1);
      frag_io<tile_cols>(at, wg * 64, 0, acc, false, false);
      mbar_arrive(acc_full);
    }
  } else {
    // ================================ epilogue ==========================================
    const size_t plane_rows = static_cast<size_t>(p.Ho) * p.Wo;
    const int ncols_here = min(kTsBN, p.ldy);
    int lt = 0;
    for (int item = blockIdx.x; item < p.items_total; item += gridDim.x, ++lt) {
      const SlabTsItem w = slabts_item(p, item);
      mbar_wait(acc_full, lt & 1);
#pragma unroll 1
      for (int erow = tid - kSlabEpiWarp0 * 32; erow < 128; erow += 32 * kSlabEpiWarps) {   // two passes over the tile rows
        const int q = w.q0 + erow;
        const int h = fdiv(q, p.fd_PW), wp = q - h * p.PW;
        const int wo = w.wc * p.WC + wp - p.halo_l;
        const bool ok = (q < p.P) && (wp >= p.halo_l) && (wp < p.halo_l + p.WC) && (wo < p.Wo);
        const size_t row = (static_cast<size_t>(w.plane_o0) * p.Ho + h) * p.Wo + wo;
#pragma unroll 1
        for (int jc = 0; jc < 2; ++jc) {                     // 64 channels = two 32-column chunks
          const int c0 = jc * 32;
          float sc[32], sh[32];
#pragma unroll
          for (int c = 0; c < 32; ++c) { sc[c] = s_scale[c0 + c]; sh[c] = s_shift[c0 + c]; }
#pragma unroll 1
          for (int s = 0; s < w.nf; ++s) {
            uint32_t v[32];
            acc_ld32(at, erow, s * kTsBN + c0, v);
            if (ok) {
              const size_t r = row + s * plane_rows;
              __half* yrow = p.y + r * p.ldy + c0;
              const __half* rrow = p.residual ? p.residual + r * p.ldr + c0 : nullptr;
#pragma unroll
              for (int c8 = 0; c8 < 4; ++c8) {
                if (c0 + c8 * 8 < ncols_here) {
                  uint32_t rr[4] = {0u, 0u, 0u, 0u};
                  if (rrow) {
                    const uint4 rv = __ldg(reinterpret_cast<const uint4*>(rrow + c8 * 8));
                    rr[0] = rv.x; rr[1] = rv.y; rr[2] = rv.z; rr[3] = rv.w;
                  }
                  uint32_t o[4];
#pragma unroll
                  for (int e = 0; e < 4; ++e) {
                    const int c = c8 * 8 + e * 2;
                    const float2 rf = unpack_half2(rr[e]);
                    float a0 = fmaf(__uint_as_float(v[c]), sc[c], sh[c]) + rf.x;
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
      }
      mbar_arrive(acc_empty);
    }
  }
}

}  // namespace b2
