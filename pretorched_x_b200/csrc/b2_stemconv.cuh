// b2_stemconv.cuh -- stem convolutions (kt x kh x 7, stride (1, 2, 2), padding (pt, ph, 3), Cin <= 4) as an
// implicit GEMM whose im2col matrix is never built: it is *described*.
//
// Input is NDHWC4 (8 bytes per pixel).  For a fixed temporal/vertical tap (dt, dh) the 7 horizontal taps of
// output pixel wo read the 8 consecutive pixels [2wo-4, 2wo+4) (pixel 2wo-4 carries a zero weight; it only keeps
// the run 16-byte aligned): 32 fp16 = 64 contiguous bytes, and the run of output pixel wo+1 starts exactly
// 16 bytes later.  A K-major SWIZZLE_NONE wgmma operand is addressed as
//     byte(row r, 16-byte chunk j) = start + (r % 8) * 16 + (r / 8) * SBO + j * LBO,
// so with LBO = 16 and SBO = 128 the 128 x 32 im2col tile of one input row is an overlapping (Toeplitz) view of
// the raw row sitting in shared memory (verified by tools/probe_umma.py, mode 1): no thread touches the data on
// its way to the tensor core.
//
// Input-row-stationary schedule.  Slab row i (input row 2*ho0 - ph + i) feeds local output row g through vertical
// tap dh = i - 2g, i.e. up to G consecutive output rows.  The per-row accumulators sit side by side in each consumer
// thread's registers (row g at fragment columns [BN*g, BN*g + BN)) and the weight image stores the taps of one parity class
// in *decreasing* dh order, so all of those contributions are ONE wgmma: A = the Toeplitz tile of slab row i, B =
// [W(dh_max); W(dh_max-2); ...] (N = BN x #taps <= G * BN), D = the fragments of the touched output rows.  Every A tile is
// read from shared memory once per slab row instead of once per (output row, dh).
//
// Register accumulators.  Two consumer warpgroups own 64 of the 128 tile rows each (pair mode: one plane each) and keep
// G * BN / 2 fp32 accumulators per thread for a whole work item.  A temporal tap's MMAs are issued back to back and committed
// as one group; wait_group 1 keeps one tap in flight while the next one is issued, and a ring slot is released once the
// group that read it has retired.  Each element sees the same sequence of fp32 accumulations as a per-row, per-N-tile
// schedule would: temporal tap, slab row ascending, K step ascending.
//
// Persistent CTAs (one per SM) walk (plane, row-group, column-tile) work items.  At the end of an item the consumers apply
// the BN affine (+ ReLU) to their fragments and write fp16 into one of two staging tiles ([128 rows][G * BN + 8]); the
// epilogue warps (one tile row per thread) take the W direction of the max-pool there and do the global stores while the
// consumers run the next item.
// Warps 0-7: consumer warpgroups, 8-11: epilogue, 12: TMA/bulk-copy producer.
#pragma once

#include "b2_ptx.cuh"

namespace b2 {

constexpr int kStemThreads = 416;       // warps 0-7: two consumer warpgroups, 8-11: epilogue, 12: producer
constexpr int kStemEpiWarp0 = 8;
constexpr int kStemTmaWarp = 12;
constexpr int kStemAccCols = 128;       // accumulator columns of one item: G * BN
constexpr int kStemPitch = 2048;        // bytes per slab row: 256 pixels [2*w0-4, 2*w0+252) of 8 bytes
constexpr int kStemRowPx = 256;         // TMA box width (the maximum box extent), one 8-byte element per pixel
constexpr int kStemTileW = 120;         // output columns per item: rows r < 124 of the 128-row MMA tile see complete runs
constexpr int kStemMaxStages = 4;
constexpr int kStemMaxRows = 16;        // slab rows = 2*(G-1) + kh
constexpr int kStemStgLd = kStemAccCols + 8;                 // staging tile pitch in halves (272 B: conflict-free both ways)
constexpr int kStemStgBytes = 128 * kStemStgLd * 2;          // one fp16 staging tile
// barriers, scale / shift, W-pool exchange slots, two staging tiles
constexpr int kStemTailBytes = 128 + 2048 + 512 + 2 * kStemStgBytes;

struct StemParams {
  int T, H, W;             // input dims per clip (W even)
  int To, Ho, Wo;
  int kt, kh;              // kw == 7, strides (1, 2, 2)
  int pt, ph;
  int G;                   // output rows per item (G * BN == kStemAccCols)
  int rows;                // slab rows = 2*(G-1) + kh
  int stage_bytes;         // slab + weights of one temporal tap, multiple of 128
  int w_bytes;             // kh * BN * 64: weight image of one temporal tap for one N tile
  int nstages;
  int Ncols;
  int tiles_w, tiles_h, ntiles_n, items_total;
  // per slab row: first / last local output row it feeds, and the image slot of the tap used by the first one
  signed char row_glo[kStemMaxRows], row_ghi[kStemMaxRows], row_slot[kStemMaxRows];
  const __half* wimg;      // packed weight image, see b2_pack_conv_weight (STEM7)
  const float* scale;
  const float* shift;
  __half* y;               // [N*To*Ho*Wo][ldy]
  int ldy;
  int relu;
  // pool_w: the MaxPool that follows the stem (k = 3, stride 2, padding 1 along W) is applied in the epilogue: y holds Wp = (Wo - 1) / 2 + 1
  // columns per row, pooled column wp = max over output columns {2wp - 1, 2wp, 2wp + 1}.  Exact because max-pooling is
  // separable; the H / T directions are pooled by a second pass over a tensor half the size (needs relu and one column tile per row).
  int pool_w, Wp;
  // pair: narrow images (Wo <= 60, kt == 1): an item covers TWO consecutive (n, t) planes.  The tensor map is declared with the
  // plane index as its SECOND dimension, so a box (128 pixels, 2 planes, rows) lands in shared memory as [row][plane][1024 B]: the
  // Toeplitz view of slab row i then shows plane 0 in tile rows 0..63 and plane 1 in rows 64..127 (rows r and r + 64 are exactly
  // 64 x 16 B = 1024 B apart), and 112 of the 128 MMA rows carry output pixels instead of 56.
  int pair, planes_total;
};

// slot of vertical tap dh inside one temporal tap of the weight image: even taps in decreasing order, then odd taps
__host__ __device__ inline int stem_slot(int dh, int kh) {
  const int emax = ((kh - 1) / 2) * 2;              // largest even tap
  const int n_even = emax / 2 + 1;
  const int omax = (kh >= 2) ? ((kh - 2) / 2) * 2 + 1 : -1;
  return (dh % 2 == 0) ? (emax - dh) / 2 : n_even + (omax - dh) / 2;
}

__device__ __forceinline__ void bulk_load_1d(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}


struct StemItem {
  int w0, ho0, ntile, plane_o, to, n;
};
__device__ __forceinline__ StemItem stem_item(const StemParams& p, int item) {
  StemItem it;
  const int tw = item % p.tiles_w; item /= p.tiles_w;
  const int th = item % p.tiles_h; item /= p.tiles_h;
  it.ntile = item % p.ntiles_n;
  it.plane_o = item / p.ntiles_n;
  it.w0 = tw * kStemTileW;
  it.ho0 = th * p.G;
  it.to = it.plane_o % p.To;
  it.n = it.plane_o / p.To;
  return it;
}

// One slab row's contribution (two K steps of 16) to the N = N_ fragment columns starting at d.  A: SWIZZLE_NONE Toeplitz view,
// K step 32 B; B: the stacked tap images, K step 256 B.
template <int N_>
__device__ __forceinline__ void stem_mma(float* d, uint64_t a, uint64_t b) {
  static_assert(N_ == 64 || N_ == 128, "stem MMA width");
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    if constexpr (N_ == 64) wgmma_n64<0>(*reinterpret_cast<float(*)[32]>(d), a + 2 * k, b + 16 * k);
    else wgmma_n128_ss(*reinterpret_cast<float(*)[64]>(d), a + 2 * k, b + 16 * k);
  }
}

// kOneSlot: tall filters (BN = 128 with kh >= 8, BN = 64 with kh >= 13) leave room for a single ring slot.  A separate instance,
// because a wait_group 0 inside the tap loop makes ptxas serialise the wgmma pipeline of the common, multi-slot one.
template <int BN, bool kOneSlot>
__global__ void __launch_bounds__(kStemThreads, 1)
stemconv_kernel(const __grid_constant__ CUtensorMap tmX,   // input as 8-byte pixels (W, H, N*T), box (256, rows, 1), no swizzle
                const StemParams p) {
  constexpr int G = kStemAccCols / BN;
  static_assert(G * BN == kStemAccCols && (G == 1 || G == 2), "stem tile");
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_align<128>(smem_raw);
  uint8_t* tail = smem + p.nstages * p.stage_bytes;
  uint64_t* full = reinterpret_cast<uint64_t*>(tail);          // [kStemMaxStages]
  uint64_t* empty = full + kStemMaxStages;
  uint64_t* stg_full = empty + kStemMaxStages;                 // [2]
  uint64_t* stg_empty = stg_full + 2;                          // [2]
  float* s_scale = reinterpret_cast<float*>(tail + 128);       // [256] (ntiles_n * BN <= 256 is enforced by the host)
  float* s_shift = s_scale + 256;
  uint32_t* s_xchg = reinterpret_cast<uint32_t*>(s_shift + 256);   // [2][4][16]: lane 31 of each epilogue warp, for the W pool
  __half* s_stg = reinterpret_cast<__half*>(s_xchg + 128);         // [2][128][kStemStgLd]

  const int tid = threadIdx.x, warp = tid >> 5;
  const int slab_bytes = p.rows * kStemPitch;

  if (tid == 0) {
    for (int s = 0; s < p.nstages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 256); }
    for (int i = 0; i < 2; ++i) { mbar_init(&stg_full[i], 256); mbar_init(&stg_empty[i], 128); }
    fence_mbar_init();
    tma_prefetch_desc(&tmX);
  }
  for (int i = tid; i < 256; i += kStemThreads) {
    s_scale[i] = (i < p.Ncols) ? __ldg(&p.scale[i]) : 0.f;
    s_shift[i] = (i < p.Ncols) ? __ldg(&p.shift[i]) : 0.f;
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();                       // everything above touched only weights / on-chip state

  if (warp == kStemTmaWarp) {
    // ================================ producer ==========================================
    int it = 0;
    for (int item = blockIdx.x; item < p.items_total; item += gridDim.x) {
      const StemItem w = stem_item(p, item);
      const int dt_lo = max(0, p.pt - w.to), dt_hi = min(p.kt - 1, p.T - 1 - w.to + p.pt);
      for (int dt = dt_lo; dt <= dt_hi; ++dt, ++it) {
        const int s = it % p.nstages;
        mbar_wait(&empty[s], ((it / p.nstages) & 1) ^ 1);
        if (elect_one()) {
          mbar_expect_tx(&full[s], static_cast<uint32_t>(slab_bytes + p.w_bytes));
          uint8_t* dst = smem + s * p.stage_bytes;
          if (p.pair) tma_load_3d(dst, &tmX, &full[s], 2 * w.w0 - 4, 2 * w.plane_o, 2 * w.ho0 - p.ph);
          else tma_load_3d(dst, &tmX, &full[s], 2 * w.w0 - 4, 2 * w.ho0 - p.ph, w.n * p.T + w.to + dt - p.pt);
          const __half* wsrc = p.wimg + (static_cast<size_t>(w.ntile) * p.kt + dt) * (p.w_bytes / 2);
          bulk_load_1d(dst + slab_bytes, wsrc, static_cast<uint32_t>(p.w_bytes), &full[s]);
        }
        __syncwarp();
      }
    }
  } else if (warp < kStemEpiWarp0) {
    // ================================ consumer warpgroups ===============================
    // SWIZZLE_NONE K-major descriptors: hi = SBO >> 4; lo = addr >> 4 | (LBO >> 4) << 16.  A: SBO 128 B, LBO 16 B; the
    // warpgroup's 64 tile rows start 64 x 16 B = 1 KB into the slab row.  B: SBO 512 B (8 rows), LBO 128 B.
    constexpr uint32_t a_hi = 128u >> 4, b_hi = 512u >> 4;
    constexpr uint32_t kTapBytes = BN * 64;            // weight image of one (dt, dh) tap: BN rows x 32 k
    const int wg = warp >> 2;
    const uint32_t base = smem_u32(smem) + static_cast<uint32_t>(wg) * 1024u;
    // fragment position: rows r0 and r0 + 8 of the tile, column pairs 8 j + c0
    const int r0 = wg * 64 + (warp & 3) * 16 + ((tid & 31) >> 2);
    const int c0 = 2 * (tid & 3);
    float acc[G * BN / 2];
    int it = 0, lt = 0;
    for (int item = blockIdx.x; item < p.items_total; item += gridDim.x, ++lt) {
      const StemItem w = stem_item(p, item);
      const int dt_lo = max(0, p.pt - w.to), dt_hi = min(p.kt - 1, p.T - 1 - w.to + p.pt);
#pragma unroll
      for (int k = 0; k < G * BN / 2; ++k) acc[k] = 0.f;
      reg_fence(acc);
      int prev_s = -1;
      for (int dt = dt_lo; dt <= dt_hi; ++dt, ++it) {
        const int s = it % p.nstages;
        mbar_wait(&full[s], (it / p.nstages) & 1);
        const uint32_t slab = base + s * p.stage_bytes;
        const uint32_t wbase = smem_u32(smem) + s * p.stage_bytes + slab_bytes;
        wgmma_fence();
#pragma unroll 1
        for (int i = 0; i < p.rows; ++i) {
          const int g_lo = p.row_glo[i], g_hi = p.row_ghi[i];
          if (g_lo > g_hi) continue;
          const uint32_t a_lo = ((slab + static_cast<uint32_t>(i) * kStemPitch) >> 4) | ((16u >> 4) << 16);
          const uint32_t b_lo = ((wbase + static_cast<uint32_t>(p.row_slot[i]) * kTapBytes) >> 4) | ((128u >> 4) << 16);
          const uint64_t a = desc_from(a_hi, a_lo), b = desc_from(b_hi, b_lo);
          if constexpr (G == 1) {
            stem_mma<BN>(acc, a, b);
          } else {
            if (g_lo != g_hi) stem_mma<2 * BN>(acc, a, b);
            else if (g_lo == 0) stem_mma<BN>(acc, a, b);
            else stem_mma<BN>(acc + BN / 2, a, b);
          }
        }
        wgmma_commit();
        if constexpr (kOneSlot) {                       // the next tap is loaded into this same slot: release it now
          wgmma_wait0();
          mbar_arrive(&empty[s]);
        } else {
          wgmma_wait1();                                // the previous tap's group has retired: its ring slot is free
          if (prev_s >= 0) mbar_arrive(&empty[prev_s]);
          prev_s = s;
        }
      }
      wgmma_wait0();
      reg_fence(acc);
      if constexpr (!kOneSlot) mbar_arrive(&empty[prev_s]);   // every item has a tap inside the clip (pt < kt, checked by the host)

      // ---- BN affine (+ ReLU) -> fp16 staging tile ----
      const int sb = lt & 1;
      mbar_wait(&stg_empty[sb], ((lt >> 1) & 1) ^ 1);
      __half* stg = s_stg + sb * (128 * kStemStgLd);
      const int n0 = w.ntile * BN;
#pragma unroll
      for (int g = 0; g < G; ++g) {
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int c = 8 * j + c0;
          const float2 sc = *reinterpret_cast<const float2*>(&s_scale[n0 + c]);
          const float2 sh = *reinterpret_cast<const float2*>(&s_shift[n0 + c]);
          const float* v = acc + g * (BN / 2) + 4 * j;
          float a0 = v[0] * sc.x + sh.x, a1 = v[1] * sc.y + sh.y;
          float b0 = v[2] * sc.x + sh.x, b1 = v[3] * sc.y + sh.y;
          if (p.relu) { a0 = fmaxf(a0, 0.f); a1 = fmaxf(a1, 0.f); b0 = fmaxf(b0, 0.f); b1 = fmaxf(b1, 0.f); }
          *reinterpret_cast<uint32_t*>(stg + r0 * kStemStgLd + g * BN + c) = pack_half2(a0, a1);
          *reinterpret_cast<uint32_t*>(stg + (r0 + 8) * kStemStgLd + g * BN + c) = pack_half2(b0, b1);
        }
      }
      mbar_arrive(&stg_full[sb]);
    }
  } else {
    // ================================ epilogue ==========================================
    // thread = tile row (pixel) erow
    const int ew = warp - kStemEpiWarp0;
    const int erow = tid - kStemEpiWarp0 * 32;
    const int lane = tid & 31;
    int lt = 0, xit = 0;
    for (int item = blockIdx.x; item < p.items_total; item += gridDim.x, ++lt) {
      const StemItem w = stem_item(p, item);
      const int g_valid = min(p.G, p.Ho - w.ho0);
      const int sb = lt & 1;
      const int n0 = w.ntile * BN;
      const int ncols_here = min(BN, p.ldy - n0);
      const int wo = p.pair ? (erow & 63) : w.w0 + erow;
      const int plane_out = p.pair ? 2 * w.plane_o + (erow >> 6) : w.plane_o;
      const bool col_ok = p.pair ? (wo < p.Wo && plane_out < p.planes_total) : ((erow < kStemTileW) && (wo < p.Wo));
      mbar_wait(&stg_full[sb], (lt >> 1) & 1);
      const __half* srow = s_stg + sb * (128 * kStemStgLd) + erow * kStemStgLd;
      if (p.pool_w) {
        // ---- max over the 3-wide / stride-2 window along W before anything is written ----
        // thread erow holds output column wo = erow (one column tile per row); even columns 2wp produce pooled column wp from
        // their own value and both neighbours: lanes +-1 by shuffle, the left neighbour of lane 0 through shared memory.
        // Post-ReLU values are >= 0, so a missing neighbour (image border, column >= Wo) contributes 0 without changing the max.
        for (int g = 0; g < g_valid; ++g) {
          const size_t prow = (static_cast<size_t>(w.plane_o) * p.Ho + (w.ho0 + g)) * p.Wp + (erow >> 1);
          __half* yrow = p.y + prow * p.ldy + n0;
#pragma unroll 1
          for (int jc = 0; jc < BN / 32; ++jc, ++xit) {
            uint32_t h[16];
            const uint4* src = reinterpret_cast<const uint4*>(srow + g * BN + jc * 32);
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              const uint4 u = src[q];
              h[4 * q] = col_ok ? u.x : 0u; h[4 * q + 1] = col_ok ? u.y : 0u;
              h[4 * q + 2] = col_ok ? u.z : 0u; h[4 * q + 3] = col_ok ? u.w : 0u;
            }
            uint32_t* xb = s_xchg + ((xit & 1) * 4 + ew) * 16;
            if (lane == 31) {
#pragma unroll
              for (int e = 0; e < 16; ++e) xb[e] = h[e];
            }
            asm volatile("bar.sync 1, 128;" ::: "memory");       // the four epilogue warps (double-buffered slots: one barrier per chunk)
            uint32_t m[16];
#pragma unroll
            for (int e = 0; e < 16; ++e) {
              uint32_t l = __shfl_up_sync(0xffffffffu, h[e], 1);
              const uint32_t r = __shfl_down_sync(0xffffffffu, h[e], 1);
              if (lane == 0) l = (ew > 0) ? (xb - 16)[e] : 0u;         // lane 31 of the previous warp; column -1 does not exist
              __half2 mm = __hmax2(*reinterpret_cast<const __half2*>(&h[e]), *reinterpret_cast<const __half2*>(&l));
              mm = __hmax2(mm, *reinterpret_cast<const __half2*>(&r));
              m[e] = *reinterpret_cast<const uint32_t*>(&mm);
            }
            if (col_ok && (erow & 1) == 0) {
#pragma unroll
              for (int c8 = 0; c8 < 4; ++c8) {
                const int col = jc * 32 + c8 * 8;
                if (col < ncols_here)
                  *reinterpret_cast<uint4*>(yrow + col) = make_uint4(m[c8 * 4], m[c8 * 4 + 1], m[c8 * 4 + 2], m[c8 * 4 + 3]);
              }
            }
          }
        }
      } else if (col_ok) {
        for (int g = 0; g < g_valid; ++g) {
          const size_t row = (static_cast<size_t>(plane_out) * p.Ho + (w.ho0 + g)) * p.Wo + wo;
          __half* yrow = p.y + row * p.ldy + n0;
          const uint4* src = reinterpret_cast<const uint4*>(srow + g * BN);
#pragma unroll
          for (int c8 = 0; c8 < BN / 8; ++c8)
            if (c8 * 8 < ncols_here) *reinterpret_cast<uint4*>(yrow + c8 * 8) = src[c8];
        }
      }
      mbar_arrive(&stg_empty[sb]);
    }
  }
}

}  // namespace b2
