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
// tap dh = i - 2g, i.e. up to G consecutive output rows.  The per-row accumulators sit side by side in the accumulator
// tile (row g at column BN*g) and the weight image stores the taps of one parity class in *decreasing* dh order, so
// all of those contributions are ONE MMA: A = the Toeplitz tile of slab row i, B = [W(dh_max); W(dh_max-2); ...]
// (N = BN x #taps, up to kStemAccCols), D = the accumulator columns of the touched output rows.  Every A tile is read
// from shared memory once per slab row instead of once per (output row, dh).  Accumulators start from zero (stored
// by the epilogue warps), so every MMA accumulates.
//
// Persistent CTAs (one per SM) walk (plane, row-group, column-tile) work items; two accumulator sets in shared memory
// let the epilogue of item i (BN + ReLU -> fp16 NDHWC) overlap the MMAs of item i+1.
// Warps 0-7: epilogue (the two warpgroups split the 32-column chunks), 8-11: MMA warpgroup, 12: TMA/bulk-copy producer.
#pragma once

#include "b2_ptx.cuh"

namespace b2 {

constexpr int kStemThreads = 416;       // warps 0-7: epilogue (even / odd 32-column chunks), 8-11: MMA warpgroup, 12: producer
constexpr int kStemMmaWarp0 = 8;
constexpr int kStemTmaWarp = 12;
constexpr int kStemAccCols = 128;       // one accumulator set: G * BN columns
constexpr int kStemPitch = 2048;        // bytes per slab row: 256 pixels [2*w0-4, 2*w0+252) of 8 bytes
constexpr int kStemRowPx = 256;         // TMA box width (the maximum box extent), one 8-byte element per pixel
constexpr int kStemTileW = 120;         // output columns per item: rows r < 124 of the 128-row MMA tile see complete runs
constexpr int kStemMaxStages = 4;
constexpr int kStemMaxRows = 16;        // slab rows = 2*(G-1) + kh <= 2*3 + 9

struct StemParams {
  int T, H, W;             // input dims per clip (W even)
  int To, Ho, Wo;
  int kt, kh;              // kw == 7, strides (1, 2, 2)
  int pt, ph;
  int G;                   // output rows per item (G * BN <= kStemAccCols)
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

template <int BN>
__global__ void __launch_bounds__(kStemThreads, 1)
stemconv_kernel(const __grid_constant__ CUtensorMap tmX,   // input as 8-byte pixels (W, H, N*T), box (256, rows, 1), no swizzle
                const StemParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_align<128>(smem_raw);
  uint8_t* tail = smem + p.nstages * p.stage_bytes;
  uint64_t* full = reinterpret_cast<uint64_t*>(tail);          // [kStemMaxStages]
  uint64_t* empty = full + kStemMaxStages;
  uint64_t* acc_full = empty + kStemMaxStages;                 // [2]
  uint64_t* acc_empty = acc_full + 2;                          // [2]
  float* s_scale = reinterpret_cast<float*>(tail + 128);       // [256] (ntiles_n * BN <= 256 is enforced by the host)
  float* s_shift = s_scale + 256;
  uint32_t* s_xchg = reinterpret_cast<uint32_t*>(s_shift + 256);   // [2 groups][2][4][16]: lane 31 of each epilogue warp, for the W pool
  const AccTile at{reinterpret_cast<float*>(s_xchg + 256), acc_ld(2 * kStemAccCols)};

  const int tid = threadIdx.x, warp = tid >> 5;
  const int slab_bytes = p.rows * kStemPitch;
  constexpr int kAccCols = kStemAccCols;

  if (tid == 128) {
    for (int s = 0; s < p.nstages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 1); }
    for (int i = 0; i < 2; ++i) { mbar_init(&acc_full[i], 1); mbar_init(&acc_empty[i], 256); }
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
  } else if (warp >= kStemMmaWarp0) {
    // ================================ MMA warpgroup =====================================
    // SWIZZLE_NONE K-major descriptors: hi = SBO >> 4; lo = addr >> 4 | (LBO >> 4) << 16.  A: SBO 128 B (64 rows = 1 KB),
    // K step 32 B; B: SBO 512 B (16 rows = 1 KB), LBO 128 B, K step 256 B.
    constexpr uint32_t a_hi = 128u >> 4, b_hi = 512u >> 4;
    constexpr uint32_t kTapBytes = BN * 64;            // weight image of one (dt, dh) tap: BN rows x 32 k
    const uint32_t base = smem_u32(smem);
    int it = 0, lt = 0;
    for (int item = blockIdx.x; item < p.items_total; item += gridDim.x, ++lt) {
      const StemItem w = stem_item(p, item);
      const int dt_lo = max(0, p.pt - w.to), dt_hi = min(p.kt - 1, p.T - 1 - w.to + p.pt);
      const int g_valid = min(p.G, p.Ho - w.ho0);
      const int ab = lt & 1;
      mbar_wait(&acc_empty[ab], (lt >> 1) & 1);            // the epilogue has drained and re-zeroed this set
      const int acc = ab * kAccCols;
      for (int dt = dt_lo; dt <= dt_hi; ++dt, ++it) {
        const int s = it % p.nstages;
        mbar_wait(&full[s], (it / p.nstages) & 1);
        const uint32_t slab = base + s * p.stage_bytes;
        const uint32_t wbase = slab + slab_bytes;
        for (int i = 0; i < p.rows; ++i) {
          const int g_lo = p.row_glo[i];
          const int g_hi = min(static_cast<int>(p.row_ghi[i]), g_valid - 1);
          if (g_lo > g_hi) continue;
          const uint32_t a_lo = ((slab + static_cast<uint32_t>(i) * kStemPitch) >> 4) | ((16u >> 4) << 16);
          const uint32_t b_lo = ((wbase + static_cast<uint32_t>(p.row_slot[i]) * kTapBytes) >> 4) | ((128u >> 4) << 16);
          const WgOperands ops{desc_from(a_hi, a_lo), desc_from(b_hi, b_lo), 2u, 64u, 16u, 256u, 64u};
          wg_mma(at, acc + g_lo * BN, (g_hi - g_lo + 1) * BN, ops, 2, true);
        }
        wg_sync();
        wg_arrive(&empty[s]);
        if (dt == dt_hi) wg_arrive(&acc_full[ab]);
      }
    }
  } else {
    // ================================ epilogue ==========================================
    // pixel (accumulator row) index of this thread, and its warpgroup's column chunks
    const int ew = warp & 3, egroup = warp >= 4 ? 1 : 0;
    const int erow = ew * 32 + (tid & 31);
    for (int c = egroup * 32; c < 2 * kAccCols; c += 64) acc_zero32(at, erow, c);   // both accumulator sets start at zero
    mbar_arrive(&acc_empty[0]);
    mbar_arrive(&acc_empty[1]);
    int lt = 0;
    for (int item = blockIdx.x; item < p.items_total; item += gridDim.x, ++lt) {
      const StemItem w = stem_item(p, item);
      const int g_valid = min(p.G, p.Ho - w.ho0);
      const int ab = lt & 1;
      const int n0 = w.ntile * BN;
      const int ncols_here = min(BN, p.ldy - n0);
      const int wo = p.pair ? (erow & 63) : w.w0 + erow;
      const int plane_out = p.pair ? 2 * w.plane_o + (erow >> 6) : w.plane_o;
      const bool col_ok = p.pair ? (wo < p.Wo && plane_out < p.planes_total) : ((erow < kStemTileW) && (wo < p.Wo));
      mbar_wait(&acc_full[ab], (lt >> 1) & 1);
      const int acc = ab * kAccCols;
      if (p.pool_w) {
        // ---- BN + ReLU, then max over the 3-wide / stride-2 window along W before anything is written ----
        // thread tid holds output column wo = tid (one column tile per row); even columns 2wp produce pooled column wp from
        // their own value and both neighbours: lanes +-1 by shuffle, the left neighbour of lane 0 through shared memory.
        // Post-ReLU values are >= 0, so a missing neighbour (image border, column >= Wo) contributes 0 without changing the max.
        const int lane = tid & 31;
        int xit = 0;
        for (int g = 0; g < g_valid; ++g) {
          const size_t prow = (static_cast<size_t>(w.plane_o) * p.Ho + (w.ho0 + g)) * p.Wp + (erow >> 1);
          __half* yrow = p.y + prow * p.ldy + n0;
#pragma unroll 1
          for (int jc = egroup; jc < BN / 32; jc += 2, ++xit) {
            uint32_t v[32];
            acc_ld32(at, erow, acc + g * BN + jc * 32, v);
            uint32_t h[16];
#pragma unroll
            for (int e = 0; e < 16; ++e) {
              const int ci = n0 + jc * 32 + e * 2;
              const float a0 = fmaxf(__uint_as_float(v[e * 2]) * s_scale[ci] + s_shift[ci], 0.f);
              const float a1 = fmaxf(__uint_as_float(v[e * 2 + 1]) * s_scale[ci + 1] + s_shift[ci + 1], 0.f);
              h[e] = col_ok ? pack_half2(a0, a1) : 0u;
            }
            uint32_t* xb = s_xchg + (((egroup * 2 + (xit & 1)) * 4) + ew) * 16;
            if (lane == 31) {
#pragma unroll
              for (int e = 0; e < 16; ++e) xb[e] = h[e];
            }
            if (egroup) asm volatile("bar.sync 2, 128;" ::: "memory");       // the four warps of this warpgroup (double-buffered slots:
            else asm volatile("bar.sync 1, 128;" ::: "memory");             // one barrier per chunk)
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
      } else
      for (int g = 0; g < g_valid; ++g) {
        const size_t row = (static_cast<size_t>(plane_out) * p.Ho + (w.ho0 + g)) * p.Wo + wo;
        __half* yrow = p.y + row * p.ldy + n0;
#pragma unroll 1
        for (int jc = egroup; jc < BN / 32; jc += 2) {
          uint32_t v[32];
          acc_ld32(at, erow, acc + g * BN + jc * 32, v);
          if (col_ok) {
#pragma unroll
            for (int c8 = 0; c8 < 4; ++c8) {
              const int col = jc * 32 + c8 * 8;
              if (col < ncols_here) {
                uint32_t o[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                  const int ci = n0 + col + e * 2;
                  float a0 = __uint_as_float(v[c8 * 8 + e * 2]) * s_scale[ci] + s_shift[ci];
                  float a1 = __uint_as_float(v[c8 * 8 + e * 2 + 1]) * s_scale[ci + 1] + s_shift[ci + 1];
                  if (p.relu) { a0 = fmaxf(a0, 0.f); a1 = fmaxf(a1, 0.f); }
                  o[e] = pack_half2(a0, a1);
                }
                *reinterpret_cast<uint4*>(yrow + col) = make_uint4(o[0], o[1], o[2], o[3]);
              }
            }
          }
        }
      }
      for (int c = egroup * 32; c < kAccCols; c += 64) acc_zero32(at, erow, acc + c);   // hand the set back zeroed (this group's chunks)
      mbar_arrive(&acc_empty[ab]);
    }
  }
}

}  // namespace b2
