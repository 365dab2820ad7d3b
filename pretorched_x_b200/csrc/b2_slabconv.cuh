// b2_slabconv.cuh -- convolution (3x3x3, 1x3x3, 3x1x1, 7x1x1, 1x7, 5x5 ...; spatial stride 1 or 2; temporal padding "same", in-plane
// padding from 0 to "same") as an implicit GEMM whose A operand is never re-fetched per filter tap.
//
// The generic gather kernel (b2_igemm.cuh) moves 16 KB of activations from L2 for every (tap, 64-channel)
// K block: 27 x for a 3x3x3 filter, which makes those layers L2-bandwidth bound at ~20% of tensor peak.
// Here one TMA box load brings a *slab* -- R input rows x (W + 2*pw) pixels x 64 channels, halo columns and
// out-of-range rows zero-filled by the TMA unit -- into shared memory once per (temporal tap, channel chunk).
// Pixels of the slab are 128-byte rows of a K-major SWIZZLE_128B tile, so the A operand of tap (dh, dw) is
// simply the same tile with its descriptor start address advanced by (dh*(W+2pw) + dw) * 128 bytes (the
// swizzle is a function of absolute smem address bits, verified by tools/probe_umma.py).  All kh*kw in-plane
// taps therefore run out of one slab: L2 traffic for activations drops by ~kh*kw.
//
// Stride 2: the taps of a 3x3 window fall into four input phases (row parity x column parity).  Each phase is a
// dense sub-image that TMA delivers directly (elementStrides = 2 along W and H), so a strided convolution is four
// small slabs per temporal tap, each serving the taps of its phase with the same shifted-descriptor trick
// (1 + 2 + 2 + 4 taps for 3x3); the 1x1x1 stride-2 shortcut projection is the one-phase, one-tap special case.
//
// Output positions are enumerated in *padded-row* coordinates q = h*(W+2pw) + w' of one (n,t) plane; a work item
// is MT consecutive 128-position M tiles (MT accumulators share every weight tile) x one N tile, and the
// positions that fall on halo columns are discarded.  Rows longer than a TMA box are cut into W chunks (each with
// its own halo); a purely temporal (kt,1,1) filter is run as a (1,kt,1) filter over the image "frames x (H*W)",
// so its slab holds MT+kt-1 frames of one position chunk and every temporal tap is a whole-row shift of it.
// CTAs are persistent (one per SM): the producer runs ahead into the next item's slabs.  Two consumer warpgroups keep the
// item's fp32 accumulators in registers (each owns 64 rows of every M tile) from its first K block to its last, then store
// them once into an accumulator tile in shared memory (AccTile, b2_ptx.cuh) and go on with the next item while the three
// epilogue warps (one tile row per thread and pass) apply the affine / residual / ReLU and write y.
#pragma once

#include "b2_ptx.cuh"
#include "b2_groupconv.cuh"

namespace b2 {

constexpr int kSlabThreads = 384;   // warps 0-7: two consumer (MMA) warpgroups, 8-10: epilogue, 11: TMA producer
constexpr int kSlabConsumerWarps = 8;
constexpr int kSlabEpiWarp0 = 8;
constexpr int kSlabEpiWarps = 3;
constexpr int kSlabTmaWarp = 11;
// Accumulator columns of one work item (MT x N tile) held in registers: each consumer thread keeps kSlabAccCols / 2 fp32 for the
// whole item.  Twelve warps are three per SM sub-partition, whose 64 KB register file then allows 168 registers per thread (a
// thirteenth warp would cut that to 128).  The tile planner (slab_pick_tiles in b2_conv_api.cu) never picks MT * N
// above kSlabAccCols; the consumer loops size their register arrays from it.
constexpr int kSlabAccCols = 192;
constexpr int kSlabWStages = 4;     // weight-tile ring depth
constexpr int kSlabSStages = 2;     // slab ring depth

constexpr int kSlabMaxSub = 4;      // sub-images (input phases) per temporal tap: 1 for stride 1, up to 4 for stride 2
constexpr int kSlabMaxTaps = 49;    // in-plane taps per sub-image (7x7 for stride 1)

struct SlabParams {
  int T, C;                // input frames per clip, channel pitch
  int To, Ho, Wo;          // output dims per clip
  int kt, khw;             // temporal taps, in-plane taps (kh*kw)
  int st, ss;              // temporal / spatial stride
  int pt;                  // temporal padding
  int cchunks;             // ceil(C / 64)
  int PW;                  // padded output-row length: WC + halo_l + halo_r
  int WC, wchunks;         // output columns per W chunk (= Wo when the row fits one TMA box) and chunks per row
  int halo_l;              // halo columns left of output column 0
  int R;                   // slab rows (sub-image rows per TMA box)
  // sub-image table: slab row 0 / col 0 of sub-image s is input pixel (ss*r_lo + sub_h0[s], sub_w0[s]); its taps read
  // slab pixel q + sub_off[s][i] and use in-plane weight tap sub_tap[s][i]
  int n_sub;
  int sub_h0[kSlabMaxSub], sub_w0[kSlabMaxSub], sub_ntaps[kSlabMaxSub];
  short sub_off[kSlabMaxSub][kSlabMaxTaps];
  unsigned char sub_tap[kSlabMaxSub][kSlabMaxTaps];
  int reach;               // max |sub_off|
  int slab_bytes;          // R * PW * 128, rounded up to 1024
  int MT;                  // M tiles per work item (MT * N tile <= kSlabAccCols)
  // runtime N tile (slabconv_kernel<0> only; the <64>/<128> instances use their template value): Cout = 144, 288,
  // 576 ... of the (2+1)D factorisation would waste up to 44% of the MMA columns on 128-wide tiles; N = 32 / 48 for the
  // growth-rate outputs of a dense layer (b2_conv_ndhwc_fprop_slice_narrow), which a 64-wide tile half / a quarter pads
  int bn;                  // N per MMA / per tile, multiple of 16, <= 256
  int wbytes;              // weight stage stride in smem: bn * 128 rounded up to 1024
  int accs;                // accumulator column stride between the MT accumulators: bn rounded up to 32
  int P;                   // Ho * PW: padded positions per output plane
  int Ncols;               // logical output channels
  int tiles_n, tiles_q, items_total;
  const float* scale;
  const float* shift;
  const __half* residual;  // nullable, dense [M][ldr]; only columns < Ncols are read
  int ldr;
  // slabconv_kernel<64, G> (grouped) only, nullable: fp16 [M][ldm]; the output is zeroed where mask <= 0 (the ReLU derivative of
  // the fine-tuning backward, b2_conv_grouped_ndhwc_dgrad)
  const __half* mask;
  int ldm;
  __half* y;               // dense [M][ldy]
  int ldy;
  int relu;
  int naff;                // scale/shift entries staged in smem (>= every column an epilogue chunk can touch)
  int aff_ld;              // > 0: scale/shift are per-sample [N][aff_ld] arrays read from global memory per work item
  // Fused nearest-2x upsampling (3x3 conv of an upsampled image == four 2x2 "phase" convs of the low-res image): the
  // geometry above is that of the LOW-res image, a work item additionally carries an output phase (py, px); phase ph
  // uses the tap table row sub_*[ph] (4 taps, weights [K][ph*4 + i][C]) and writes output pixel (2h + py, 2w + px) of a
  // (2 Ho) x (2 Wo) plane.  n_sub stays 1: all phases read the same slab.
  int up;
  // Multi-plane items (mp >= 2, planes of at most 128 padded positions, no temporal taps that differ between planes): the MT accumulators
  // of an item belong to mp CONSECUTIVE PLANES instead of consecutive tiles of one plane, so small planes (7x7: one 38%-full tile)
  // share every weight tile mp ways -- these layers stream their whole filter per work item and are bound by that L2 traffic.  One
  // 4-D TMA box brings the mp slabs ([plane][R][PW] in shared memory); tile j's A operand starts j * plane_stride bytes further.
  int mp, plane_stride, planes_total;
  FastDiv fd_tiles_n, fd_tiles_q, fd_wchunks, fd_To, fd_PW;   // dividers of the item decode (set by launch_slab)
  int ldo;                 // slabconv_kernel<BN, TMT, kSlabSlice> only: row pitch of y (>= ldy, the columns written)
  int qitem;               // slab_t_kernel only: padded positions of one work item (whole output rows for BN = 128, 2 NP for 64)
};

// scale/shift live in smem for all (padded) output channels: SlabParams::naff = round_up(ldy, 32) + 32 entries each; the
// accumulator tile (MT * accs columns) through which the consumers hand each item to the epilogue follows them

struct SlabItem {
  int n0, q0, wc, plane_o, plane_i0, r_lo, dt_lo, n_dt, n_slabs, mt_valid;   // plane_i0: input plane of temporal tap 0
  int phase;                                                                  // output phase 2*py + px (SlabParams::up), else 0
};
__device__ __forceinline__ SlabItem slab_item(const SlabParams& p, int item, int BN) {
  SlabItem w;
  int t = fdiv(item, p.fd_tiles_n);
  const int tn = item - t * p.tiles_n; item = t;
  w.phase = 0;
  if (p.up) { w.phase = item & 3; item >>= 2; }
  t = fdiv(item, p.fd_tiles_q);
  const int tq = item - t * p.tiles_q; item = t;
  w.plane_o = fdiv(item, p.fd_wchunks);
  w.wc = item - w.plane_o * p.wchunks;
  if (p.mp > 1) w.plane_o *= p.mp;                  // first plane of the group
  w.n0 = tn * BN;
  w.q0 = tq * (p.MT * 128);
  const int n = fdiv(w.plane_o, p.fd_To), to = w.plane_o - n * p.To;
  const int t0 = to * p.st - p.pt;                  // input frame of temporal tap 0
  w.plane_i0 = n * p.T + t0;
  const int lo = w.q0 - p.reach;                    // lowest padded position any tap of this item touches
  w.r_lo = (lo >= 0) ? fdiv(lo, p.fd_PW) : -fdiv(-lo + p.PW - 1, p.fd_PW);
  w.dt_lo = max(0, -t0);                            // temporal taps that stay inside the clip
  const int dt_hi = min(p.kt - 1, p.T - 1 - t0);
  w.n_dt = dt_hi - w.dt_lo + 1;
  w.n_slabs = p.cchunks * w.n_dt * p.n_sub;
  const int mv = (p.P - w.q0 + 127) / 128;          // M tiles that contain at least one position of the plane
  w.mt_valid = mv > p.MT ? p.MT : mv;
  if (p.mp > 1) w.mt_valid = min(p.mp, p.planes_total - w.plane_o);   // planes of the group that exist
  return w;
}

// eight consecutive accumulator columns of one row of an AccTile (16-byte aligned)
__device__ __forceinline__ void acc_ld8(const float* src, float (&v)[8]) {
  const float4 a = reinterpret_cast<const float4*>(src)[0], b = reinterpret_cast<const float4*>(src)[1];
  v[0] = a.x; v[1] = a.y; v[2] = a.z; v[3] = a.w; v[4] = b.x; v[5] = b.y; v[6] = b.z; v[7] = b.w;
}

// K steps of one (tap, 64-channel block) for an N-column tile whose fragments start at d: one wgmma per K step; the last channel
// chunk of C = 144, 288, 232 ... skips its all-zero K steps
template <int N>
__device__ __forceinline__ void slab_mma(float* d, uint64_t a, uint64_t b, int ksteps) {
#pragma unroll
  for (int k = 0; k < 4; ++k)
    if (k < ksteps) wgmma_ss<N>(d, a + 2 * k, b + 2 * k);    // K step: +32 B on both start addresses
}

// 64-wide tile, transposed product.  With at most 64 output channels the weight stage is exactly one m64 A operand, so each
// warpgroup computes D^T[64 channels][positions] = W[64][K] . X^T with the slab rows as a K-major B operand.  One m64n(64 c)k16
// per K step reads 2 KB of A and c 2 KB of B from shared memory where c m64n64k16 read c (2 KB + 2 KB): at c = 2, 96 instead of
// 128 bytes per tensor cycle, so the SM's 128 B/cycle shared-memory port no longer bounds the MMAs.  The item's MT * 128 positions
// v = 128 j + r (tile j, row r) are split into two contiguous halves: warpgroup wg owns v in [wg MT 64, wg MT 64 + MT 64), its
// 64-position chunk c at fragment columns [64 c, 64 c + 64).
//   TMT = MT = 2: one m64n128k16 per K step over the whole half.
//   TMT = 0 (MT = 1, and multi-plane items, whose tiles lie plane_stride apart in the slab): one m64n64k16 per chunk.
// Every chunk is issued, also where a ragged item (mt_valid < MT) has no valid position in it: slab_rows sizes the slab for
// MT * 128 positions from every item start, so those rows are inside it (multi-plane items read the same rows the M-tile
// orientation did), their columns of D are discarded by the epilogue, and skipping them -- or issuing narrower forms on the
// same accumulators -- makes ptxas serialise the wgmma pipeline (C7515).
__device__ __forceinline__ int slab_t64_v0(int wg, int MT, int c) { return (wg * MT + c) * 64; }
__device__ __forceinline__ uint32_t slab_t64_off16(int v0, uint32_t tile_stride16) {   // slab start of position v0, 16-byte units
  return static_cast<uint32_t>(v0 >> 7) * tile_stride16 + static_cast<uint32_t>(v0 & 127) * 8u;
}

// Consumer warpgroups of slabconv_kernel for an N tile of N columns.  Warpgroup wg owns rows [64 wg, 64 wg + 64) of every M tile of
// an item; tile j sits at fragment columns [j N, j N + N) of each thread's registers from the item's first K block to its last
// (N = 64: the transposed product above).  The MMAs of one tap form one commit group, one group stays in flight, and a ring slot is
// released when the group that read it retires.  G != 0 (N = 64): the grouped convolution of b2_groupconv.cuh -- positions stay
// along M and each K step of a tap goes into its own G-column range of the fragment.
template <int N, int TMT, int G = 0>
__device__ __forceinline__ void slab_consumer(const SlabParams& p, const AccTile& at, int accs, uint32_t slab0, uint32_t w0s,
                                              int w_bytes, uint64_t* slab_full, uint64_t* slab_empty, uint64_t* w_full,
                                              uint64_t* w_empty, uint64_t* acc_full, uint64_t* acc_empty) {
  constexpr int kMaxMT = kSlabAccCols / N < 4 ? kSlabAccCols / N : 4;
  float acc[kMaxMT * N / 2];
  const int wg = warp_uniform(threadIdx.x >> 7);
  const bool lead = (threadIdx.x & 31) == 0;                 // one arrival per consumer warp on the ring barriers
  const uint32_t a_wg = static_cast<uint32_t>(wg) * (64u * 128u >> 4);   // this warpgroup's 64 rows, in 16-byte units
  const uint32_t tile_stride16 = (p.mp > 1 ? static_cast<uint32_t>(p.plane_stride) : 128u * 128u) >> 4;   // A start of tile j
  const int MT = TMT ? TMT : p.MT;
  int wit = 0, sg = 0, lt = 0;
  for (int item = blockIdx.x; item < p.items_total; item += gridDim.x, ++lt) {
    const SlabItem w = slab_item(p, item, N);
#pragma unroll
    for (int k = 0; k < kMaxMT * N / 2; ++k) acc[k] = 0.f;
    reg_fence(acc);
    int prev_ws = -1, prev_s = -1;                           // ring slots read by the group in flight
    const int mt_valid = warp_uniform(w.mt_valid);
    for (int si = 0; si < w.n_slabs; ++si, ++sg) {
      const int sub = p.up ? w.phase : si % p.n_sub;
      const int ntaps = p.sub_ntaps[sub];
      const int cc = (si / p.n_sub) / w.n_dt;
      const int ksteps = warp_uniform(min(4, (p.C - cc * 64 + 15) >> 4));       // 16-channel K steps that hold real channels
      const int s = sg % kSlabSStages;
      mbar_wait(&slab_full[s], (sg / kSlabSStages) & 1);
      const uint32_t slab_addr = slab0 + s * p.slab_bytes;
      for (int ti = 0; ti < ntaps; ++ti, ++wit) {
        const int ws = wit % kSlabWStages;
        mbar_wait(&w_full[ws], (wit / kSlabWStages) & 1);
        // slab-local pixel index of padded output position q0 under this tap
        const int pix0 = w.q0 + p.sub_off[sub][ti] - w.r_lo * p.PW;
        const uint64_t b = desc_from(kSw128DescHi, sw128_desc_lo(w0s + ws * w_bytes));
        const uint32_t a_lo0 = sw128_desc_lo(slab_addr + static_cast<uint32_t>(pix0) * 128u);
        wgmma_fence();
        if constexpr (N == 64 && G == 0) {
          // the weight stage is A, slab rows are B (the descriptor formats are the same K-major SWIZZLE_128B)
          if constexpr (TMT == 0) {
#pragma unroll
            for (int c = 0; c < kMaxMT; ++c)
              if (c < MT)
                slab_mma<64>(acc + c * 32, b, desc_from(kSw128DescHi, a_lo0 + slab_t64_off16(slab_t64_v0(wg, MT, c), tile_stride16)),
                             ksteps);
          } else {
            static_assert(TMT * 64 <= kSlabAccCols, "one warpgroup's half of the item in registers");
            slab_mma<TMT * 64>(acc, b, desc_from(kSw128DescHi, a_lo0 + slab_t64_off16(slab_t64_v0(wg, MT, 0), tile_stride16)),
                               ksteps);
          }
        } else {
#pragma unroll
          for (int j = 0; j < kMaxMT; ++j) {
            if (j < mt_valid) {
              const uint64_t a = desc_from(kSw128DescHi, a_lo0 + a_wg + j * tile_stride16);
              if constexpr (G != 0) group_mma<G>(acc + j * (N / 2), a, b);
              else slab_mma<N>(acc + j * (N / 2), a, b, ksteps);
            }
          }
        }
        wgmma_commit();
        wgmma_wait1();                                       // the previous tap's group has retired: release what it read
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
    if (lead) {                                              // every item has a slab and a tap ("same" padding keeps tap 0 inside)
      mbar_arrive(&w_empty[prev_ws]);
      mbar_arrive(&slab_empty[prev_s]);
    }
    // hand the item to the epilogue: one store of the fragments into the accumulator tile, then straight on to the next item
    mbar_wait(acc_empty, (lt & 1) ^ 1);
    if constexpr (N == 64 && G == 0) {
      // transposed into the [position][channel] tile: fragment (channel ch (+8), positions v, v + 1) goes to row v & 127 of tile
      // v >> 7.  A pitch of 4 (mod 32) floats puts the 8 channels x 4 even positions of one store in 32 distinct banks.
      // (32-bit shared addresses stepped from one base: the 96 accumulators leave no room for a 64-bit pointer per store)
      const int t = threadIdx.x & 127;
      const uint32_t ld4 = static_cast<uint32_t>(at.ld) * 4u;
      const uint32_t base = smem_u32(at.p) + static_cast<uint32_t>((t >> 5) * 16 + ((t & 31) >> 2) + 2 * (t & 3) * at.ld) * 4u;
#pragma unroll
      for (int c = 0; c < kMaxMT; ++c) {
        if (c < MT) {
          const int v0 = slab_t64_v0(wg, MT, c);
          uint32_t a = base + static_cast<uint32_t>((v0 & 127) * at.ld + (v0 >> 7) * accs) * 4u;
#pragma unroll
          for (int jb = 0; jb < 8; ++jb, a += 8u * ld4) {
            const float* f = acc + c * 32 + 4 * jb;
            st_shared_f32(a, f[0]);
            st_shared_f32(a + 32u, f[2]);
            st_shared_f32(a + ld4, f[1]);
            st_shared_f32(a + ld4 + 32u, f[3]);
          }
        }
      }
    } else {
#pragma unroll
      for (int j = 0; j < kMaxMT; ++j)
        if (j < mt_valid) frag_io<N>(at, wg * 64, j * accs, *reinterpret_cast<float(*)[N / 2]>(acc + j * (N / 2)), false, false);
    }
    mbar_arrive(acc_full);
  }
}

// TMA producer of the slab kernels (one warp); item_at(item) decodes a work item (slab_item, or slab_t_item of b2_slab_t128.cuh).
// Walks (item, slab) pairs; the slab after the current one -- possibly the first slab of the NEXT item -- is
// requested after weight tap min(kSlabWStages, ntaps - 1) of the current slab: from tap kSlabWStages on, the weight ring
// guarantees the consumers have retired the slab that occupied the target slot, so that wait never stalls weight issue;
// a slab with fewer taps issues all of its weights first (the previous slab is released only once this one's first tap runs).
template <int G, class ItemAt>
__device__ __forceinline__ void slab_producer(const SlabParams& p, const CUtensorMap* tmX, const CUtensorMap* tmB, uint8_t* slab_base,
                                              uint8_t* w_base, int kWBytes, int bn, uint64_t* slab_full, uint64_t* slab_empty,
                                              uint64_t* w_full, uint64_t* w_empty, ItemAt item_at) {
  int wit = 0, sg = 0;                     // global weight-tile / slab counters (ring phases persist across items)
  int item = blockIdx.x;
  if (item < p.items_total) {
    SlabItem cur = item_at(item);
    int nxt_item = item, nxt_si = 0;       // (item, slab) of the next slab to load
    SlabItem nxt = cur;
    // slab index si of an item enumerates (cc, dt, sub) with sub fastest
    auto load_next = [&]() {
      const int sub = nxt_si % p.n_sub;
      const int r2 = nxt_si / p.n_sub;
      const int cc = r2 / nxt.n_dt, dt = nxt.dt_lo + (r2 - cc * nxt.n_dt);
      const int s = sg % kSlabSStages;
      mbar_wait(&slab_empty[s], ((sg / kSlabSStages) & 1) ^ 1);
      if (elect_one()) {
        mbar_expect_tx(&slab_full[s], static_cast<uint32_t>(p.R * p.PW * 128 * (p.mp > 1 ? p.mp : 1)));
        tma_load_4d(slab_base + s * p.slab_bytes, tmX, &slab_full[s], G ? nxt.n0 : cc * 64,
                    p.sub_w0[sub] + p.ss * nxt.wc * p.WC, p.ss * nxt.r_lo + p.sub_h0[sub], nxt.plane_i0 + dt);
      }
      __syncwarp();
      ++sg;
      if (++nxt_si == nxt.n_slabs) {       // advance to the first slab of the following item
        nxt_si = 0;
        nxt_item += gridDim.x;
        if (nxt_item < p.items_total) nxt = item_at(nxt_item);
      }
    };
    load_next();
    for (; item < p.items_total; item += gridDim.x) {
      cur = item_at(item);
      for (int si = 0; si < cur.n_slabs; ++si) {
        const int sub = p.up ? cur.phase : si % p.n_sub;          // tap-table row (== slab index unless p.up)
        const int r2 = si / p.n_sub;
        const int cc = r2 / cur.n_dt, dt = cur.dt_lo + (r2 - cc * cur.n_dt);
        const int ntaps = p.sub_ntaps[sub];
        const int pf = min(kSlabWStages, ntaps - 1);
        for (int ti = 0; ti < ntaps; ++ti, ++wit) {
          const int ws = wit % kSlabWStages;
          mbar_wait(&w_empty[ws], ((wit / kSlabWStages) & 1) ^ 1);
          const int tap = dt * p.khw + p.sub_tap[sub][ti];
          if (elect_one()) {
            mbar_expect_tx(&w_full[ws], static_cast<uint32_t>(G ? G * 128 : bn * 128));
            if constexpr (G != 0) tma_load_2d(w_base + ws * kWBytes, tmB, &w_full[ws], 0, ((cur.n0 >> 6) * p.kt * p.khw + tap) * G);
            else tma_load_2d(w_base + ws * kWBytes, tmB, &w_full[ws], tap * p.C + cc * 64, cur.n0);
          }
          __syncwarp();
          if (ti == pf && nxt_item < p.items_total) load_next();
        }
      }
    }
  }
}

// BN = 0: N tile taken from SlabParams::bn at run time.  TMT: the 64-wide tile's MMA form (slab_consumer; 0 for the other tiles).
// G = 16 / 32 (BN = 64): grouped convolution with C == K (b2_groupconv.cuh).  N tile tn is the 64-channel slice tn of input AND
// output, the item has one channel chunk (SlabParams::cchunks = 1) whose TMA channel coordinate is the slice's, and a weight stage
// is the G-row tile of (slice, tap).
// G = kSlabSlice: dense filter, y is a column slice of a wider row -- the epilogue writes columns [0, ldy) of rows of pitch
// SlabParams::ldo and nothing else, so an inception branch lands in place in its block's concatenated output.
constexpr int kSlabSlice = -1;
template <int BN, int TMT = 0, int G_ = 0>
__global__ void __launch_bounds__(kSlabThreads, 1)
slabconv_kernel(const __grid_constant__ CUtensorMap tmX,   // input as (C, W, H, N*T), box (64, PW, R, 1)
                const __grid_constant__ CUtensorMap tmB,   // weights [Ncols][taps*C], box (64, BN); G: [slices*taps*G][64], box (64, G)
                const SlabParams p) {
  constexpr int G = G_ > 0 ? G_ : 0;            // channels per group of the grouped form, 0 otherwise
  static_assert(G == 0 || (BN == 64 && TMT == 0), "the grouped form runs on the 64-wide tile with positions along M");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_align<1024>(smem_raw);
  const int bn = BN ? BN : p.bn;
  const int kWBytes = G ? G * 128 : BN ? BN * 128 : p.wbytes;      // stage stride; a stage receives bn * 128 (G * 128) bytes
  const int accs = BN ? BN : p.accs;
  uint8_t* slab_base = smem;
  uint8_t* w_base = smem + kSlabSStages * p.slab_bytes;
  uint8_t* tail = w_base + kSlabWStages * kWBytes;
  uint64_t* slab_full = reinterpret_cast<uint64_t*>(tail);
  uint64_t* slab_empty = slab_full + kSlabSStages;
  uint64_t* w_full = slab_empty + kSlabSStages;
  uint64_t* w_empty = w_full + kSlabWStages;
  uint64_t* acc_full = w_empty + kSlabWStages;
  uint64_t* acc_empty = acc_full + 1;
  float* s_scale = reinterpret_cast<float*>(tail + 256);     // barriers occupy the first 128 bytes
  float* s_shift = s_scale + p.naff;

  const int tid = threadIdx.x, warp = tid >> 5;
  const AccTile at{s_shift + p.naff, acc_ld(p.MT * accs)};

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
    s_scale[i] = (i < p.Ncols && !p.aff_ld) ? __ldg(&p.scale[i]) : 0.f;
    s_shift[i] = (i < p.Ncols && !p.aff_ld) ? __ldg(&p.shift[i]) : 0.f;
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();                       // everything above touched only weights / on-chip state

  if (warp == kSlabTmaWarp) {
    // ================================ TMA producer ======================================
    slab_producer<G>(p, &tmX, &tmB, slab_base, w_base, kWBytes, bn, slab_full, slab_empty, w_full, w_empty,
                     [&](int it) { return slab_item(p, it, bn); });
  } else if (warp < kSlabEpiWarp0) {
    // ================================ consumer warpgroups ===============================
    const uint32_t slab0 = smem_u32(slab_base), w0s = smem_u32(w_base);
    if constexpr (BN != 0) {
      slab_consumer<BN, TMT, G>(p, at, accs, slab0, w0s, kWBytes, slab_full, slab_empty, w_full, w_empty, acc_full, acc_empty);
    } else {
      // runtime N: one compiled main loop per width the tile planner can pick (launch_slab rejects any other)
      switch (bn) {
#define B2_SLAB_N(n) case n: slab_consumer<n, 0>(p, at, accs, slab0, w0s, kWBytes, slab_full, slab_empty, w_full, w_empty, acc_full, acc_empty); break;
        B2_SLAB_N(16) B2_SLAB_N(32) B2_SLAB_N(48) B2_SLAB_N(144) B2_SLAB_N(160) B2_SLAB_N(176) B2_SLAB_N(192)
#undef B2_SLAB_N
        default: __trap();
      }
    }
  } else {
    // ================================ epilogue ==========================================
    int lt = 0;
    for (int item = blockIdx.x; item < p.items_total; item += gridDim.x, ++lt) {
      const SlabItem w = slab_item(p, item, bn);
      mbar_wait(acc_full, lt & 1);
      const int ncols_here = min(bn, p.ldy - w.n0);     // columns of this tile that exist in y (incl. zero padding)
      // thread = accumulator row; the 96 epilogue threads cover the 128 tile rows in two passes
#pragma unroll 1
      for (int erow = tid - kSlabEpiWarp0 * 32; erow < 128; erow += 32 * kSlabEpiWarps) {
        // output row of this thread in each of the item's M tiles
        size_t row[4];
        bool ok[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int q = p.mp > 1 ? erow : w.q0 + j * 128 + erow;          // multi-plane items: tile j is plane plane_o + j
          const int h = fdiv(q, p.fd_PW), wp = q - h * p.PW;
          const int wo = w.wc * p.WC + wp - p.halo_l;       // output column
          ok[j] = (j < w.mt_valid) && (q < p.P) && (wp >= p.halo_l) && (wp < p.halo_l + p.WC) && (wo < p.Wo);
          const size_t plane = static_cast<size_t>(w.plane_o) + (p.mp > 1 ? j : 0);
          row[j] = p.up ? (plane * (2 * p.Ho) + 2 * h + (w.phase >> 1)) * (2 * p.Wo) + 2 * wo + (w.phase & 1)
                        : (plane * p.Ho + h) * p.Wo + wo;
        }
#pragma unroll 1
        for (int jc = 0; jc * 32 < ncols_here; ++jc) {
          // folded-BN scale/shift of these 32 channels: registers, reused by every M tile of the item
          float sc[32], sh[32];
          const int c0 = w.n0 + jc * 32;
          if (p.aff_ld) {
            // per-sample affine (class-conditional BN of the consumer): the item lies in one image, every lane reads the
            // same 32 + 32 floats (L1 broadcast) as 16-byte vectors; launch_slab checks the 16-byte alignment
            const float* gs = p.scale + static_cast<size_t>(fdiv(w.plane_o, p.fd_To)) * p.aff_ld + c0;
            const float* gt = p.shift + static_cast<size_t>(fdiv(w.plane_o, p.fd_To)) * p.aff_ld + c0;
#pragma unroll
            for (int g = 0; g < 8; ++g) {
              float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
              if (c0 + 4 * g + 4 <= p.Ncols) {
                a = __ldg(reinterpret_cast<const float4*>(gs) + g);
                b = __ldg(reinterpret_cast<const float4*>(gt) + g);
              } else if (c0 + 4 * g < p.Ncols) {              // ragged tail of a channel count that is not a multiple of 4
                float* ap = reinterpret_cast<float*>(&a); float* bp = reinterpret_cast<float*>(&b);
                for (int e = 0; e < 4; ++e)
                  if (c0 + 4 * g + e < p.Ncols) { ap[e] = __ldg(gs + 4 * g + e); bp[e] = __ldg(gt + 4 * g + e); }
              }
              sc[4 * g] = a.x; sc[4 * g + 1] = a.y; sc[4 * g + 2] = a.z; sc[4 * g + 3] = a.w;
              sh[4 * g] = b.x; sh[4 * g + 1] = b.y; sh[4 * g + 2] = b.z; sh[4 * g + 3] = b.w;
            }
          } else {
#pragma unroll
            for (int c = 0; c < 32; ++c) {
              sc[c] = s_scale[c0 + c];
              sh[c] = s_shift[c0 + c];
            }
          }
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            if (j < w.mt_valid) {                            // warp-uniform
              // (the HBM latency of the residual row is hidden behind the consumers' next item, not behind the next M tile: one
              // register set of residuals is what the budget leaves next to the scale / shift registers)
              uint4 rres[4];
              if (p.residual && ok[j]) {
                const __half* rrow = p.residual + row[j] * p.ldr + c0;
#pragma unroll
                for (int c8 = 0; c8 < 4; ++c8)
                  if (jc * 32 + c8 * 8 < ncols_here) rres[c8] = ld_res8(rrow + c8 * 8, c0 + c8 * 8, p.Ncols);   // columns >= K: zero
              }
              // accumulators are read 8 columns at a time next to their use: with the scale / shift and residual registers a
              // whole 32-column row segment would not fit the register budget
              const float* arow = at.p + static_cast<size_t>(erow) * at.ld + j * accs + jc * 32;
              if (ok[j]) {
                __half* yrow = p.y + row[j] * (G_ == kSlabSlice ? p.ldo : p.ldy) + c0;
                if (p.residual) {                              // uniform: residual added in fp32 before the single rounding
#pragma unroll
                  for (int c8 = 0; c8 < 4; ++c8) {
                    if (jc * 32 + c8 * 8 < ncols_here) {
                      const uint4 rv = rres[c8];
                      const uint32_t rr[4] = {rv.x, rv.y, rv.z, rv.w};
                      float v[8];
                      acc_ld8(arow + c8 * 8, v);
                      uint32_t o[4];
#pragma unroll
                      for (int e = 0; e < 4; ++e) {
                        const int c = c8 * 8 + e * 2;
                        const float2 rf = unpack_half2(rr[e]);
                        float a0 = fmaf(v[2 * e], sc[c], sh[c]) + rf.x;
                        float a1 = fmaf(v[2 * e + 1], sc[c + 1], sh[c + 1]) + rf.y;
                        if (p.relu) { a0 = fmaxf(a0, 0.f); a1 = fmaxf(a1, 0.f); }
                        o[e] = pack_half2(a0, a1);
                      }
                      *reinterpret_cast<uint4*>(yrow + c8 * 8) = make_uint4(o[0], o[1], o[2], o[3]);
                    }
                  }
                } else {                                       // no residual: affine, round, ReLU on the packed pairs
                  const __half2 zero2 = __floats2half2_rn(0.f, 0.f);
#pragma unroll
                  for (int c8 = 0; c8 < 4; ++c8) {
                    if (jc * 32 + c8 * 8 < ncols_here) {
                      float v[8];
                      acc_ld8(arow + c8 * 8, v);
                      uint4 ov;
                      uint32_t* o = reinterpret_cast<uint32_t*>(&ov);
#pragma unroll
                      for (int e = 0; e < 4; ++e) {
                        const int c = c8 * 8 + e * 2;
                        __half2 hv = __floats2half2_rn(fmaf(v[2 * e], sc[c], sh[c]),
                                                       fmaf(v[2 * e + 1], sc[c + 1], sh[c + 1]));
                        if (p.relu) hv = __hmax2(hv, zero2);
                        o[e] = *reinterpret_cast<uint32_t*>(&hv);
                      }
                      if constexpr (G_ > 0) {
                        if (p.mask) {                          // uniform
                          const uint4 mv = *reinterpret_cast<const uint4*>(p.mask + static_cast<size_t>(row[j]) * p.ldm + c0 + c8 * 8);
                          const uint32_t mm[4] = {mv.x, mv.y, mv.z, mv.w};
#pragma unroll
                          for (int e = 0; e < 4; ++e) o[e] &= __hgt2_mask(*reinterpret_cast<const __half2*>(&mm[e]), zero2);
                        }
                      }
                      *reinterpret_cast<uint4*>(yrow + c8 * 8) = ov;
                    }
                  }
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
