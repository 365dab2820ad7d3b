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
// G * BN / 2 fp32 accumulators per thread for a whole work item.  Instances: BN = 128 with G = 1, BN = 64 with G = 2 or G = 4
// (128 accumulators per thread).  A temporal tap's MMAs are issued back to back and committed
// as one group; wait_group 1 keeps one tap in flight while the next one is issued, and a ring slot is released once the
// group that read it has retired.  Each element sees the same sequence of fp32 accumulations as a per-row, per-N-tile
// schedule would: temporal tap, slab row ascending, K step ascending.
//
// Persistent CTAs (one per SM) walk (plane, row-group, column-tile) work items.  At the end of an item the consumers apply
// the BN affine (+ ReLU) to their fragments and write fp16 into a staging tile ([rows][G * BN + 8]); the epilogue warps (one
// tile row per thread) take the W direction of the max-pool there and do the global stores while the consumers run the next item.
// Warps 0-7: consumer warpgroups, 8-11: epilogue, 12: TMA/bulk-copy producer.
//
// G = 4 (BN = 64, never pair mode; N = 64 MMAs, see stem_row_mma): 128 accumulators per consumer thread do not fit the 152
// registers a 416-thread CTA leaves, so the CTA has 512 threads (warps 13-15 complete the producer warpgroup and exit) and
// setmaxnreg moves registers from the producer (40) and epilogue (56) warpgroups to the consumers (208).  Its shared memory holds three 54 KB ring stages (13 slab rows + the 28 KB weight
// image of a 7-tall filter) and ONE staging tile of the 120 tile rows that carry output columns: the epilogue drains an item in
// a small fraction of the next item's main loop.
//
// Transposed G = 4 (kT; rows of at most 112 output columns): the same CTA, ring, producer and epilogue warps compute
// D^T[64 channels][112 positions] = W . X^T per output row.  A (m64) is the tap image of (dt, dh), read with the descriptor the
// other instances use for B; B is the Toeplitz view of one slab row at N = 112 (tools/probe_umma.py, mode 4), so a whole output
// row is one MMA and no tile row is padding.  Consumer warpgroup wg owns output rows 2 wg and 2 wg + 1 (56 fp32 each per thread)
// and issues one N = 112 MMA pair per (slab row, owned row): 2 KB of A + 3.5 KB of B per 56 tensor cycles, against 2 KB + 2 KB per
// 32 for a 64-row N = 64 piece.  The fragments are stored transposed (stmatrix .trans) into the [position][channel] staging
// tile, so the epilogue is shared.  Every element keeps the accumulation order of the other instances.
#pragma once

#include "b2_ptx.cuh"

namespace b2 {

constexpr int kStemEpiWarp0 = 8;
constexpr int kStemTmaWarp = 12;
constexpr int kStemPitch = 2048;        // bytes per slab row: 256 pixels [2*w0-4, 2*w0+252) of 8 bytes
constexpr int kStemRowPx = 256;         // TMA box width (the maximum box extent), one 8-byte element per pixel
constexpr int kStemTileW = 120;         // output columns per item: rows r < 124 of the 128-row MMA tile see complete runs
constexpr int kStemTileT = 112;         // output columns of the transposed instance, the N of its MMAs: position n reads the bytes
                                        // [16 n, 16 n + 64) of a 2 KB slab row
constexpr int kStemMaxStages = 4;
constexpr int kStemMaxRows = 16;        // slab rows = 2*(G-1) + kh
// per instance (G output rows per item, BN output channels per N tile)
__host__ __device__ constexpr int stem_threads(int G) { return G == 4 ? 512 : 416; }
__host__ __device__ constexpr int stem_stg_ld(int G, int BN) { return G * BN + 8; }   // pitch in halves: 16 B past a multiple of
                                                                                       // 128 B, conflict-free both ways
__host__ __device__ constexpr int stem_stg_rows(int G) { return G == 4 ? kStemTileW : 128; }
__host__ __device__ constexpr int stem_stg_bufs(int G) { return G == 4 ? 1 : 2; }
// barriers, scale / shift, W-pool exchange slots, staging tiles
__host__ __device__ constexpr int stem_tail_bytes(int G, int BN) {
  return 128 + 2048 + 512 + stem_stg_bufs(G) * stem_stg_rows(G) * stem_stg_ld(G, BN) * 2;
}

struct StemParams {
  int T, H, W;             // input dims per clip (W even)
  int To, Ho, Wo;
  int kt, kh;              // kw == 7, strides (1, 2, 2)
  int pt, ph;
  int G;                   // output rows per item: 1 (BN = 128), 2 or 4 (BN = 64)
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

// Row plan: slab row i feeds local output rows g_lo..g_hi (dh = i - 2g, 0 <= dh < kh); the taps it uses for them are dh(g_lo),
// dh(g_lo) - 2, ..., consecutive slots of the weight image starting at slot_lo.  g_lo > g_hi: the row feeds nothing.
__host__ inline void stem_row_plan(int G, int kh, int i, int* g_lo, int* g_hi, int* slot_lo) {
  int lo = i - (kh - 1);
  lo = lo > 0 ? (lo + 1) / 2 : 0;
  int hi = i / 2;
  if (hi > G - 1) hi = G - 1;
  *g_lo = lo; *g_hi = hi;
  *slot_lo = lo <= hi ? stem_slot(i - 2 * lo, kh) : 0;
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
  for (int k = 0; k < 2; ++k) wgmma_ss<N_>(d, a + 2 * k, b + 16 * k);
}
// The transposed form: A = one tap image (K step 256 B), B = the Toeplitz view of a slab row at N = 112 (K step 32 B).
__device__ __forceinline__ void stem_mma_t(float* d, uint64_t w, uint64_t x) {
#pragma unroll
  for (int k = 0; k < 2; ++k) wgmma_ss<kStemTileT>(d, w + 16 * k, x + 2 * k);
}

// Slab row feeding local output rows g_lo..g_hi (row g's fragments at acc + g * BN / 2).  G <= 2: one MMA over all of them; the
// register offset and width must be compile-time constants, hence one case per (g_lo, g_hi).  G = 4: one N = 64 MMA per output
// row.  Wider windows (N = 256 / 192 over the touched rows, or N = 128 pairs at fragment offsets 0 and 64 next to N = 64 ones)
// make ptxas serialise the wgmma pipeline (C7511) or, for N > 128, need more registers than a 512-thread launch allows at
// compile time; four equal, disjoint windows do neither.
template <int BN, int G>
__device__ __forceinline__ void stem_row_mma(float* acc, int g_lo, int g_hi, uint64_t a, uint64_t b) {
  if constexpr (G == 1) {
    stem_mma<BN>(acc, a, b);
  } else if constexpr (G == 2) {
    if (g_lo != g_hi) stem_mma<2 * BN>(acc, a, b);
    else if (g_lo == 0) stem_mma<BN>(acc, a, b);
    else stem_mma<BN>(acc + BN / 2, a, b);
  } else {
    static_assert(G == 4 && BN == 64, "stem tile");
    const uint64_t bs = BN * 64 / 16;                 // one tap image (BN rows x 64 B) in descriptor units
#pragma unroll
    for (int g = 0; g < 4; ++g)
      if (g >= g_lo && g <= g_hi) stem_mma<64>(acc + 32 * g, a, b + (g - g_lo) * bs);
  }
}

// kOneSlot: tall filters (BN = 128 with kh >= 8, BN = 64 with kh >= 13) leave room for a single ring slot.  A separate instance,
// because a wait_group 0 inside the tap loop makes ptxas serialise the wgmma pipeline of the common, multi-slot one.
// kT: the transposed four-row instance (G = 4, Wo <= kStemTileT).
template <int BN, int G, bool kOneSlot, bool kT>
__global__ void __launch_bounds__(stem_threads(G), 1)
stemconv_kernel(const __grid_constant__ CUtensorMap tmX,   // input as 8-byte pixels (W, H, N*T), box (256, rows, 1), no swizzle
                const StemParams p) {
  static_assert((BN == 128 && G == 1) || (BN == 64 && (G == 2 || G == 4)), "stem tile");
  static_assert(!kT || (BN == 64 && G == 4 && !kOneSlot), "transposed stem tile");
  constexpr int kThreads = stem_threads(G);
  constexpr int kStgLd = stem_stg_ld(G, BN), kStgRows = stem_stg_rows(G), kStgBufs = stem_stg_bufs(G);
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_align<128>(smem_raw);
  uint8_t* tail = smem + p.nstages * p.stage_bytes;
  uint64_t* full = reinterpret_cast<uint64_t*>(tail);          // [kStemMaxStages]
  uint64_t* empty = full + kStemMaxStages;
  uint64_t* stg_full = empty + kStemMaxStages;                 // [kStgBufs]
  uint64_t* stg_empty = stg_full + 2;                          // [kStgBufs]
  float* s_scale = reinterpret_cast<float*>(tail + 128);       // [256] (ntiles_n * BN <= 256 is enforced by the host)
  float* s_shift = s_scale + 256;
  uint32_t* s_xchg = reinterpret_cast<uint32_t*>(s_shift + 256);   // [2][4][16]: lane 31 of each epilogue warp, for the W pool
  __half* s_stg = reinterpret_cast<__half*>(s_xchg + 128);         // [kStgBufs][kStgRows][kStgLd]

  const int tid = threadIdx.x, warp = tid >> 5;
  const int slab_bytes = p.rows * kStemPitch;

  if (tid == 0) {
    for (int s = 0; s < p.nstages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 256); }
    for (int i = 0; i < kStgBufs; ++i) { mbar_init(&stg_full[i], 256); mbar_init(&stg_empty[i], 128); }
    fence_mbar_init();
    tma_prefetch_desc(&tmX);
  }
  for (int i = tid; i < 256; i += kThreads) {
    s_scale[i] = (i < p.Ncols) ? __ldg(&p.scale[i]) : 0.f;
    s_shift[i] = (i < p.Ncols) ? __ldg(&p.shift[i]) : 0.f;
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();                       // everything above touched only weights / on-chip state

  if (G == 4 ? warp >= kStemTmaWarp : warp == kStemTmaWarp) {   // G = 4: the whole producer warpgroup runs setmaxnreg
    // ================================ producer ==========================================
    if constexpr (G == 4) setmaxnreg_dec<40>();
    if (warp != kStemTmaWarp) return;
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
    if constexpr (G == 4) setmaxnreg_inc<208>();
    // SWIZZLE_NONE K-major descriptors: hi = SBO >> 4; lo = addr >> 4 | (LBO >> 4) << 16.  Toeplitz view of a slab row (A; kT: B):
    // SBO 128 B, LBO 16 B; outside kT the warpgroup's 64 tile rows start 64 x 16 B = 1 KB into the slab row.  Weight image (B;
    // kT: A): SBO 512 B (8 rows), LBO 128 B.
    constexpr uint32_t x_hi = 128u >> 4, w_hi = 512u >> 4;
    constexpr uint32_t kTapBytes = BN * 64;            // weight image of one (dt, dh) tap: BN rows x 32 k
    const int wg = warp >> 2;
    const uint32_t base = smem_u32(smem) + (kT ? 0u : static_cast<uint32_t>(wg) * 1024u);
    // fragment position: rows r0 and r0 + 8 of the tile, column pairs 8 j + c0
    const int r0 = wg * 64 + (warp & 3) * 16 + ((tid & 31) >> 2);
    const int c0 = 2 * (tid & 3);
    constexpr int kAcc = kT ? kStemTileT : G * BN / 2;   // kT: output rows 2 wg and 2 wg + 1, kStemTileT / 2 fp32 each
    float acc[kAcc];
    int it = 0, lt = 0;
    for (int item = blockIdx.x; item < p.items_total; item += gridDim.x, ++lt) {
      const StemItem w = stem_item(p, item);
      const int dt_lo = max(0, p.pt - w.to), dt_hi = min(p.kt - 1, p.T - 1 - w.to + p.pt);
#pragma unroll
      for (int k = 0; k < kAcc; ++k) acc[k] = 0.f;
      reg_fence(acc);
      int prev_s = -1;
      for (int dt = dt_lo; dt <= dt_hi; ++dt, ++it) {
        const int s = it % p.nstages;
        mbar_wait(&full[s], (it / p.nstages) & 1);
        const uint32_t slab = base + s * p.stage_bytes;
        const uint32_t wbase = smem_u32(smem) + s * p.stage_bytes + slab_bytes;
        wgmma_fence();
        if constexpr (kT) {
          // slab row i feeds the owned row g = 2 wg + gg through dh = i - 2 g, the slot row_slot[i] + g - g_lo: i in [4 wg, 4 wg + kh + 1]
          const int wgu = warp_uniform(wg);
          const int i_end = min(p.rows, 4 * wgu + p.kh + 2);
#pragma unroll 1
          for (int i = 4 * wgu; i < i_end; ++i) {
            const int g_lo = p.row_glo[i], g_hi = p.row_ghi[i];
            const uint32_t x_lo = ((slab + static_cast<uint32_t>(i) * kStemPitch) >> 4) | ((16u >> 4) << 16);
#pragma unroll
            for (int gg = 0; gg < 2; ++gg) {
              const int g = 2 * wgu + gg;
              if (g >= g_lo && g <= g_hi) {
                const uint32_t w_lo = ((wbase + static_cast<uint32_t>(p.row_slot[i] + g - g_lo) * kTapBytes) >> 4) | ((128u >> 4) << 16);
                stem_mma_t(acc + gg * (kStemTileT / 2), desc_from(w_hi, w_lo), desc_from(x_hi, x_lo));
              }
            }
          }
        } else {
#pragma unroll 1
          for (int i = 0; i < p.rows; ++i) {
            const int g_lo = p.row_glo[i], g_hi = p.row_ghi[i];
            if (g_lo > g_hi) continue;
            const uint32_t a_lo = ((slab + static_cast<uint32_t>(i) * kStemPitch) >> 4) | ((16u >> 4) << 16);
            const uint32_t b_lo = ((wbase + static_cast<uint32_t>(p.row_slot[i]) * kTapBytes) >> 4) | ((128u >> 4) << 16);
            stem_row_mma<BN, G>(acc, g_lo, g_hi, desc_from(x_hi, a_lo), desc_from(w_hi, b_lo));
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
      const int sb = lt % kStgBufs;
      mbar_wait(&stg_empty[sb], ((lt / kStgBufs) & 1) ^ 1);
      __half* stg = s_stg + sb * (kStgRows * kStgLd);
      const int n0 = w.ntile * BN;
      if constexpr (kT) {
        // fragment of row g = 2 wg + gg: channels m (d[4 j], d[4 j + 1]) and m + 8 (d[4 j + 2], d[4 j + 3]), positions 8 j + c0, +1.
        // stmatrix k = 2 q + h of step jp holds positions 16 jp + 8 q + [0, 8) x channels 16 (warp % 4) + 8 h + [0, 8); lane l
        // addresses its memory row l % 8, one position.  A 528-byte pitch puts those 8 rows x 16 B in 32 different banks.  Staging
        // rows 112..119 are not written: with Wo <= 112 the epilogue's col_ok is false there.
        const int lane = tid & 31, k = lane >> 3;
        const int m = n0 + 16 * (warp & 3) + (lane >> 2);
        const float sc0 = s_scale[m], sh0 = s_shift[m], sc1 = s_scale[m + 8], sh1 = s_shift[m + 8];
        const uint32_t st0 = smem_u32(stg + (8 * (k >> 1) + (lane & 7)) * kStgLd + 16 * (warp & 3) + 8 * (k & 1));
#pragma unroll
        for (int gg = 0; gg < 2; ++gg) {
#pragma unroll
          for (int jp = 0; jp < kStemTileT / 16; ++jp) {
            uint32_t r[4];
#pragma unroll
            for (int q = 0; q < 2; ++q) {
              const float* v = acc + gg * (kStemTileT / 2) + 4 * (2 * jp + q);
              float a0 = v[0] * sc0 + sh0, a1 = v[1] * sc0 + sh0;
              float b0 = v[2] * sc1 + sh1, b1 = v[3] * sc1 + sh1;
              if (p.relu) { a0 = fmaxf(a0, 0.f); a1 = fmaxf(a1, 0.f); b0 = fmaxf(b0, 0.f); b1 = fmaxf(b1, 0.f); }
              r[2 * q] = pack_half2(a0, a1);
              r[2 * q + 1] = pack_half2(b0, b1);
            }
            stmatrix_x4_trans(st0 + 2u * static_cast<uint32_t>(16 * jp * kStgLd + (2 * wg + gg) * BN), r);
          }
        }
      } else {
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
            *reinterpret_cast<uint32_t*>(stg + r0 * kStgLd + g * BN + c) = pack_half2(a0, a1);
            if (kStgRows == 128 || r0 + 8 < kStgRows)         // tile rows >= kStemTileW carry no output column
              *reinterpret_cast<uint32_t*>(stg + (r0 + 8) * kStgLd + g * BN + c) = pack_half2(b0, b1);
          }
        }
      }
      mbar_arrive(&stg_full[sb]);
    }
  } else {
    // ================================ epilogue ==========================================
    // thread = tile row (pixel) erow
    if constexpr (G == 4) setmaxnreg_dec<56>();
    const int ew = warp - kStemEpiWarp0;
    const int erow = tid - kStemEpiWarp0 * 32;
    const int lane = tid & 31;
    int lt = 0, xit = 0;
    for (int item = blockIdx.x; item < p.items_total; item += gridDim.x, ++lt) {
      const StemItem w = stem_item(p, item);
      const int g_valid = min(p.G, p.Ho - w.ho0);
      const int sb = lt % kStgBufs;
      const int n0 = w.ntile * BN;
      const int ncols_here = min(BN, p.ldy - n0);
      const int wo = p.pair ? (erow & 63) : w.w0 + erow;
      const int plane_out = p.pair ? 2 * w.plane_o + (erow >> 6) : w.plane_o;
      const bool col_ok = p.pair ? (wo < p.Wo && plane_out < p.planes_total) : ((erow < kStemTileW) && (wo < p.Wo));
      mbar_wait(&stg_full[sb], (lt / kStgBufs) & 1);
      // rows past a shorter staging tile have col_ok == false: they read (and then ignore) its last row
      const int srow_i = (kStgRows < 128 && erow >= kStgRows) ? kStgRows - 1 : erow;
      const __half* srow = s_stg + sb * (kStgRows * kStgLd) + srow_i * kStgLd;
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
