// b2_pgemm.cuh -- persistent, warp-specialised GEMM for the 1x1x1 convolutions and dense layers:
//
//     D[M][N] = act( scale[n] * (A[M][K] . B[N][K]^T  [+ A2[M][K2] . B2[N][K2]^T]) + shift[n] + residual[M][N] )
//                                                                                   (fp16 in/out, fp32 accumulate)
// The optional second operand pair accumulates into the same accumulators: it fuses the type-B shortcut projection of a
// bottleneck into its closing 1x1x1 convolution (BN scales folded into the two weight matrices), so the projected
// shortcut never goes through HBM.
//
// K runs from 64 to 2048 (plus the K2 of a fused projection).  The shallow-K layers are bound by HBM (every output element is
// written once and, for the block-closing conv3, a residual element is read once), the deep-K ones (conv1 of the late stages, the
// projection-fused conv3s) by the tensor core.  One CTA per SM loops over 128 x BN output tiles, n fastest, so the CTAs working on
// one M block share its A tile through L2; the non-persistent igemm_kernel pays the barrier set-up and a cold pipeline for every
// tile, and with K = 64 that prologue dominates.  Two consumer warpgroups each own 64 rows of the tile and keep its fp32
// accumulators in registers from the first K block to the last; they apply the epilogue to their fragments, stage fp16 in a
// 128B-swizzled box and TMA-store their 64 rows, while the producer streams the next tile's operands through the smem ring.
// The residual of a tile arrives by TMA in one of two buffers, which then also serve as that tile's output staging (each element
// is read and overwritten by the same thread): a buffer goes back to the producer once the bulk store that reads it is done.
//
//   warps 0-7   two consumer warpgroups: wgmma main loop, epilogue, TMA store of their 64 rows
//   warp 8      producer: the K blocks of tile i (A and B boxes, 128B-swizzled), then its residual tile
//   warps 9-12  generator instance only: A-operand transform (see PgemmParams::in_scale)
#pragma once

#include "b2_ptx.cuh"

namespace b2 {

constexpr int kPgConsumerThreads = 256;
constexpr int kPgProdWarp = kPgConsumerThreads / 32;
constexpr int kPgXformWarp0 = kPgProdWarp + 1;
constexpr int kPgThreads = (kPgProdWarp + 1) * 32;
constexpr int kPgXformWarps = 4;                     // generator instance only: A-operand transform warps (see PgemmParams::in_scale)
constexpr int kPgThreadsGan = (kPgXformWarp0 + kPgXformWarps) * 32;
constexpr int kPgMaxStages = 4;

struct PgemmParams {
  int M, Ncols, ldy;        // rows, logical columns, output pitch (columns [Ncols, ldy) are written as zero)
  int nkb;                  // K blocks of 64 of the first operand pair
  int nkb2;                 // K blocks of the second operand pair (0 = none)
  int tiles_n, tiles_total;
  const float* scale;
  const float* shift;
  int has_residual;
  int relu;
  int aff_ld, aff_rows;     // > 0: scale/shift are [M / aff_rows][aff_ld] (per-sample affine; aff_rows % 128 == 0)
  // Residual taken from a LOW-resolution tensor (nearest-2x upsampling on the fly; GBlock skip path): output row
  // m = (n, h, w) of an Hh x Wh image adds res_up[((n * Hh/2 + h/2) * Wh/2 + w/2) * res_ld + column].  The 128 output rows
  // of a tile are a segment of one image row (Wh >= 128) or whole pairs of image rows (Wh <= 64), so their sources are
  // res_rows = 64 (resp. 32) CONSECUTIVE rows of the low-res matrix: one TMA box per 64 columns, loaded like the plain
  // residual, and each fragment row r reads row src(r) of that box.  pgemm_kernel<BN, 1> only.
  const __half* res_up;
  int res_ld, Wh, Hh;
  int res_rows;             // rows of the low-res residual box: 64 (Wh >= 128) or 32
  FastDiv fd_Wh, fd_Hh;
  int res_pre;              // 1: y = act(scale * (acc + residual) + shift) instead of act(scale * acc + shift + residual)
  // Second output (pgemm_kernel<BN, 1>): y2 = relu(y * scale2[m / aff2_rows][n] + shift2[...]) -- the class-conditional
  // BatchNorm + ReLU of the NEXT block applied to this block's fp32 result, staged in a tile of its own and written through tmC2.
  int dual;
  const float* scale2;
  const float* shift2;
  int aff2_ld, aff2_rows;
  // Input-side per-sample affine + ReLU (pgemm_kernel<BN, 1>): the A operand becomes relu(a * in_scale[m / in_rows][k] + in_shift[...])
  // -- the class-conditional BatchNorm + ReLU that OPENS a GBlock, applied to the raw block input on its way to the tensor core
  // instead of in a stand-alone read + write pass over the tensor.  Four transform warps rewrite each A tile in place in shared
  // memory (one 128-byte row per thread, fp32 arithmetic) between the TMA landing and the MMA; the tile loop is HBM-bound, so
  // the ~280 instructions per K block per thread ride in issue slots that were idle.  First operand pair only; in_rows % 128 == 0.
  const float* in_scale;
  const float* in_shift;
  int in_ld, in_rows;
  const __half* mask;       // pgemm_kernel<BN, 0, 1> only: fp16 [M][ldm] ReLU-derivative mask of the output (see IgemmParams)
  int ldm;
};

template <int BN, int GAN>
struct PgemmSmem {
  static constexpr int kABytes = 128 * 128;
  static constexpr int kBBytes = BN * 128;
  static constexpr int kStage = kABytes + kBBytes;
  static constexpr int kTile = 128 * BN * 2;                 // fp16 128 x BN tile: BN / 64 boxes of [128 rows][128 B], 128B-swizzled
  static constexpr int kAffBytes = 2 * 4 * BN * 4;           // per consumer warpgroup: scale, shift, scale2, shift2 of the tile
  static constexpr int kFixed = 2 * kTile + (GAN ? kTile : 0) + 256 + kAffBytes + 1024;
  // operand ring: as deep as the budget allows, up to kPgMaxStages (BN = 128: 4 stages, 3 with the generator's second-output tile)
  static constexpr int kStages = (227 * 1024 - kFixed) / kStage < kPgMaxStages ? (227 * 1024 - kFixed) / kStage : kPgMaxStages;
  static constexpr int kResOff = kStages * kStage;           // 2 residual / output staging tiles
  static constexpr int kC2Off = kResOff + 2 * kTile;         // second-output staging tile (generator instance)
  static constexpr int kBarOff = kC2Off + (GAN ? kTile : 0);
  static constexpr int kAffOff = kBarOff + 256;
  static constexpr int kTotal = kAffOff + kAffBytes + 1024;
  static_assert(kStages >= 3 && kTotal <= 227 * 1024, "shared memory budget");
};

__device__ __forceinline__ void pg_bar(int id, int threads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory"); }

// Byte offset of the 4-byte column pair (row, 8 j + c) in a 128B-swizzled [rows][64 columns] box sequence (j < BN / 8, c even < 8):
// box j / 8, 16-byte chunk (j % 8) ^ (row % 8).  The fragment pattern (8 rows x 4 column pairs per warp) hits 32 distinct banks.
__device__ __forceinline__ uint32_t pg_sw_off(int row, int j, int c) {
  return static_cast<uint32_t>(j >> 3) * (128u * 128u) + static_cast<uint32_t>(row) * 128u +
         ((static_cast<uint32_t>(j & 7) ^ static_cast<uint32_t>(row & 7)) << 4) + static_cast<uint32_t>(c) * 2u;
}

template <int BN, int GAN, int MASK = 0>   // GAN = 1: instance with the generator extras (res_up gather, res_pre, dual output, A transform);
                                           // 0: the classic epilogue.  MASK = 1 (with GAN = 0): ReLU-derivative mask operand (fine-tuning backward)
__global__ void __launch_bounds__(GAN ? kPgThreadsGan : kPgThreads, 1)
pgemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
             const __grid_constant__ CUtensorMap tmA2, const __grid_constant__ CUtensorMap tmB2,
             const __grid_constant__ CUtensorMap tmC, const __grid_constant__ CUtensorMap tmR,
             const __grid_constant__ CUtensorMap tmC2, const PgemmParams p) {
  using S = PgemmSmem<BN, GAN>;
  constexpr int kSt = S::kStages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_align<1024>(smem_raw);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + S::kBarOff);   // [kSt]
  uint64_t* empty = full + kPgMaxStages;                             // [kSt]
  uint64_t* xf_full = empty + kPgMaxStages;                          // [kSt] A tile transformed (generator instance)
  uint64_t* res_full = xf_full + kPgMaxStages;                       // [2]
  uint64_t* res_empty = res_full + 2;                                // [2]
  const bool xform = GAN && p.in_scale != nullptr;

  const int tid = threadIdx.x, warp = tid >> 5;

  if (tid == 0) {
    for (int s = 0; s < kSt; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 2); mbar_init(&xf_full[s], kPgXformWarps * 32); }
    for (int i = 0; i < 2; ++i) { mbar_init(&res_full[i], 1); mbar_init(&res_empty[i], 2); }
    fence_mbar_init();
    tma_prefetch_desc(&tmA); tma_prefetch_desc(&tmB); tma_prefetch_desc(&tmC);
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();                       // everything above touched only weights / on-chip state

  if (warp == kPgProdWarp) {
    // ================================ producer ==========================================
    int it = 0, lt = 0;
    for (int tile = blockIdx.x; tile < p.tiles_total; tile += gridDim.x, ++lt) {
      const int m0 = (tile / p.tiles_n) * 128, n0 = (tile % p.tiles_n) * BN;
      for (int kb = 0; kb < p.nkb + p.nkb2; ++kb, ++it) {
        const int s = it % kSt;
        mbar_wait(&empty[s], ((it / kSt) & 1) ^ 1);
        if (elect_one()) {
          mbar_expect_tx(&full[s], S::kStage);
          uint8_t* dst = smem + s * S::kStage;
          if (kb < p.nkb) {
            tma_load_2d(dst, &tmA, &full[s], kb * 64, m0);
            tma_load_2d(dst + S::kABytes, &tmB, &full[s], kb * 64, n0);
          } else {
            tma_load_2d(dst, &tmA2, &full[s], (kb - p.nkb) * 64, m0);
            tma_load_2d(dst + S::kABytes, &tmB2, &full[s], (kb - p.nkb) * 64, n0);
          }
        }
        __syncwarp();
      }
      // The residual / staging buffer of tile i is free once the stores of tile i - 2 have read it.  Loaded after the K blocks,
      // which the consumers need first; without a residual the empty buffer is handed over all the same.
      const int rb = lt & 1;
      mbar_wait(&res_empty[rb], ((lt >> 1) & 1) ^ 1);
      if (p.has_residual) {
        int r0 = m0;                                       // first row of the residual box
        uint32_t rbytes = S::kTile;
        if (GAN && p.res_up) {
          const int t1 = fdiv(m0, p.fd_Wh), wq = m0 - t1 * p.Wh;
          const int nq = fdiv(t1, p.fd_Hh), hq = t1 - nq * p.Hh;
          r0 = (nq * (p.Hh >> 1) + (hq >> 1)) * (p.Wh >> 1) + (wq >> 1);
          rbytes = static_cast<uint32_t>(p.res_rows) * BN * 2;
        }
        if (elect_one()) {
          mbar_expect_tx(&res_full[rb], rbytes);
#pragma unroll
          for (int b = 0; b < BN / 64; ++b)
            tma_load_2d(smem + S::kResOff + rb * S::kTile + b * (128 * 128), &tmR, &res_full[rb], n0 + b * 64, r0);
        }
      } else if (elect_one()) {
        mbar_arrive(&res_full[rb]);
      }
      __syncwarp();
    }
  } else if (warp < kPgProdWarp) {
    // ================================ consumer warpgroups ===============================
    // Warpgroup wg owns tile rows [64 wg, 64 wg + 64).  Thread fragment: rows fr and fr + 8, column pairs 8 j + fc, j < BN / 8, at
    // acc[4 j .. 4 j + 1] (row fr) and acc[4 j + 2 .. 4 j + 3] (row fr + 8).  The MMAs of one K block form one commit group, one
    // group stays in flight, and a ring slot is released (one arrival per warpgroup) when the group that read it has retired.
    const int wg = warp >> 2, wt = tid & 127;
    const bool leader = wt == 0;                           // issues this warpgroup's bulk stores and its ring / buffer arrivals
    const int bar_wg = 1 + wg;                             // named barrier of the warpgroup's 128 threads
    const int fr = wg * 64 + (warp & 3) * 16 + ((tid & 31) >> 2);
    const int fc = 2 * (tid & 3);
    float* s_aff = reinterpret_cast<float*>(smem + S::kAffOff) + wg * 4 * BN;   // scale[BN], shift[BN], scale2[BN], shift2[BN]
    const uint32_t ring = smem_u32(smem);
    const uint32_t a_wg = static_cast<uint32_t>(wg) * (64u * 128u >> 4);        // this warpgroup's 64 A rows, in 16-byte units
    const int nkb = warp_uniform(p.nkb), nkb_all = warp_uniform(p.nkb + p.nkb2);
    float acc[BN / 2];
    int it = 0, lt = 0;
    for (int tile = blockIdx.x; tile < p.tiles_total; tile += gridDim.x, ++lt) {
      const int m0 = (tile / p.tiles_n) * 128, n0 = (tile % p.tiles_n) * BN;
      // the tile's affine, fetched before the main loop and stored after it
      float aff[4] = {0.f, 0.f, 0.f, 0.f};
      if (wt < BN && n0 + wt < p.Ncols) {
        // per-sample affine (class-conditional BN of the consumer): a 128-row tile never straddles two samples
        const size_t arow = p.aff_ld ? static_cast<size_t>(m0 / p.aff_rows) * p.aff_ld : 0;
        aff[0] = __ldg(&p.scale[arow + n0 + wt]);
        aff[1] = __ldg(&p.shift[arow + n0 + wt]);
        if (GAN && p.dual) {
          const size_t arow2 = static_cast<size_t>(m0 / p.aff2_rows) * p.aff2_ld;
          aff[2] = __ldg(&p.scale2[arow2 + n0 + wt]);
          aff[3] = __ldg(&p.shift2[arow2 + n0 + wt]);
        }
      }
#pragma unroll
      for (int k = 0; k < BN / 2; ++k) acc[k] = 0.f;
      reg_fence(acc);
      int prev_s = -1;
      for (int kb = 0; kb < nkb_all; ++kb, ++it) {
        const int s = it % kSt;
        if (xform && kb < nkb) mbar_wait(&xf_full[s], (it / kSt) & 1);     // operands landed AND the A tile was rewritten
        else mbar_wait(&full[s], (it / kSt) & 1);
        const uint64_t a = desc_from(kSw128DescHi, sw128_desc_lo(ring + s * S::kStage) + a_wg);
        const uint64_t b = desc_from(kSw128DescHi, sw128_desc_lo(ring + s * S::kStage + S::kABytes));
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_ss<BN>(acc, a + 2 * k, b + 2 * k);   // K step: +32 B on both start addresses
        wgmma_commit();
        wgmma_wait1();                                     // the previous K block's group has retired: release its slot
        if (leader && prev_s >= 0) mbar_arrive(&empty[prev_s]);
        prev_s = s;
      }
      wgmma_wait0();
      reg_fence(acc);
      if (leader) {
        mbar_arrive(&empty[prev_s]);                       // every tile has at least one K block
        // the stores of the previous tile had the whole main loop to read their staging tiles: hand that buffer back
        if (lt > 0) { tma_store_wait_read0(); mbar_arrive(&res_empty[(lt - 1) & 1]); }
      }
      if (wt < BN) { s_aff[wt] = aff[0]; s_aff[BN + wt] = aff[1]; s_aff[2 * BN + wt] = aff[2]; s_aff[3 * BN + wt] = aff[3]; }
      pg_bar(bar_wg, 128);                                 // (also: the second-output tile is free again)

      // ---- epilogue math on the fragments, in place (fp32) ----
      const int rb = lt & 1;
      mbar_wait(&res_full[rb], (lt >> 1) & 1);
      uint8_t* stage = smem + S::kResOff + rb * S::kTile;
      int rsrc[2] = {fr, fr + 8};                          // row of the residual box each fragment row adds
      if (GAN && p.res_up) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int r = fr + 8 * i;
          if (p.Wh >= 128) rsrc[i] = r >> 1;
          else { const int hr = fdiv(r, p.fd_Wh); rsrc[i] = (hr >> 1) * (p.Wh >> 1) + ((r - hr * p.Wh) >> 1); }
        }
      }
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int c = 8 * j + fc;
        const float2 sc = *reinterpret_cast<const float2*>(s_aff + c);
        const float2 sh = *reinterpret_cast<const float2*>(s_aff + BN + c);
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          float2 rf = make_float2(0.f, 0.f);
          if (p.has_residual) rf = unpack_half2(*reinterpret_cast<const uint32_t*>(stage + pg_sw_off(rsrc[i], j, fc)));
          float a0 = acc[4 * j + 2 * i], a1 = acc[4 * j + 2 * i + 1];
          if (GAN && p.res_pre) {
            a0 = (a0 + rf.x) * sc.x + sh.x;
            a1 = (a1 + rf.y) * sc.y + sh.y;
          } else {
            a0 = a0 * sc.x + sh.x + rf.x;
            a1 = a1 * sc.y + sh.y + rf.y;
          }
          if (p.relu) { a0 = fmaxf(a0, 0.f); a1 = fmaxf(a1, 0.f); }
          if constexpr (MASK) {
            const int mrow = m0 + fr + 8 * i, mcol = n0 + c;
            uint32_t mv = 0;
            if (mrow < p.M && mcol < p.ldm) mv = __ldg(reinterpret_cast<const unsigned int*>(p.mask + static_cast<size_t>(mrow) * p.ldm + mcol));
            const float2 mf = unpack_half2(mv);
            a0 = mf.x > 0.f ? a0 : 0.f;
            a1 = mf.y > 0.f ? a1 : 0.f;
          }
          acc[4 * j + 2 * i] = a0; acc[4 * j + 2 * i + 1] = a1;
        }
      }
      // upsampled residual: a box row feeds rows of both warpgroups, so every read precedes the first overwrite
      if (GAN && p.res_up) pg_bar(3, kPgConsumerThreads);

      // ---- fp16 into the staging tile, TMA store of this warpgroup's 64 rows ----
#pragma unroll
      for (int j = 0; j < BN / 8; ++j)
#pragma unroll
        for (int i = 0; i < 2; ++i)
          *reinterpret_cast<uint32_t*>(stage + pg_sw_off(fr + 8 * i, j, fc)) = pack_half2(acc[4 * j + 2 * i], acc[4 * j + 2 * i + 1]);
      fence_proxy_async();
      pg_bar(bar_wg, 128);
      if (leader && m0 + wg * 64 < p.M) {
#pragma unroll
        for (int b = 0; b < BN / 64; ++b)
          if (n0 + b * 64 < p.ldy) tma_store_2d(&tmC, stage + b * (128 * 128) + wg * (64 * 128), n0 + b * 64, m0 + wg * 64);
        tma_store_commit();
      }
      if (GAN && p.dual) {                                 // second output: next block's ccbn + ReLU on the fp32 value
        uint8_t* stage2 = smem + S::kC2Off;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int c = 8 * j + fc;
          const float2 sc2 = *reinterpret_cast<const float2*>(s_aff + 2 * BN + c);
          const float2 sh2 = *reinterpret_cast<const float2*>(s_aff + 3 * BN + c);
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            const float a0 = fmaxf(acc[4 * j + 2 * i] * sc2.x + sh2.x, 0.f);
            const float a1 = fmaxf(acc[4 * j + 2 * i + 1] * sc2.y + sh2.y, 0.f);
            *reinterpret_cast<uint32_t*>(stage2 + pg_sw_off(fr + 8 * i, j, fc)) = pack_half2(a0, a1);
          }
        }
        fence_proxy_async();
        pg_bar(bar_wg, 128);
        if (leader && m0 + wg * 64 < p.M) {
#pragma unroll
          for (int b = 0; b < BN / 64; ++b)
            if (n0 + b * 64 < p.ldy) tma_store_2d(&tmC2, stage2 + b * (128 * 128) + wg * (64 * 128), n0 + b * 64, m0 + wg * 64);
          tma_store_commit();
        }
      }
    }
    if (leader) tma_store_wait_read0();
  } else if (GAN) {
    // ================================ A-operand transform (generator instance) ==========
    if (xform) {
      // thread t owns logical 8-channel chunk j = t & 7 (its 8 scale + 8 shift values stay in registers for the K block) of the
      // rows (t >> 3) + 16 i, i = 0..7.  The eight threads of a quarter-warp cover one 128-byte row: conflict-free; all loads of a K
      // block are issued before the first use and all stores after the last (one row per thread with load -> store per chunk
      // serialised on shared-memory latency: 2x slower layers than the stand-alone pass it replaces).
      const int t = tid - kPgXformWarp0 * 32;
      const int j = t & 7, r0 = t >> 3;
      const uint32_t coff = (static_cast<uint32_t>(j) ^ static_cast<uint32_t>(r0 & 7)) << 4;     // (r0 + 16 i) & 7 == r0 & 7
      int it = 0;
      for (int tile = blockIdx.x; tile < p.tiles_total; tile += gridDim.x) {
        const int m0 = (tile / p.tiles_n) * 128;
        const size_t arow = static_cast<size_t>(m0 / p.in_rows) * p.in_ld;   // a 128-row tile never straddles two samples
        for (int kb = 0; kb < p.nkb + p.nkb2; ++kb, ++it) {
          if (kb >= p.nkb) continue;
          const int s = it % kSt;
          const float4* sc4 = reinterpret_cast<const float4*>(p.in_scale + arow + kb * 64 + j * 8);
          const float4* sh4 = reinterpret_cast<const float4*>(p.in_shift + arow + kb * 64 + j * 8);
          const float4 s0 = __ldg(sc4), s1 = __ldg(sc4 + 1), t0 = __ldg(sh4), t1 = __ldg(sh4 + 1);   // before the wait: independent of the tile
          mbar_wait(&full[s], (it / kSt) & 1);
          uint8_t* base = smem + s * S::kStage + r0 * 128 + coff;
          uint4 v[8];
#pragma unroll
          for (int i = 0; i < 8; ++i) v[i] = *reinterpret_cast<const uint4*>(base + i * (16 * 128));
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const float2 x0 = unpack_half2(v[i].x), x1 = unpack_half2(v[i].y), x2 = unpack_half2(v[i].z), x3 = unpack_half2(v[i].w);
            v[i].x = pack_half2(fmaxf(fmaf(x0.x, s0.x, t0.x), 0.f), fmaxf(fmaf(x0.y, s0.y, t0.y), 0.f));
            v[i].y = pack_half2(fmaxf(fmaf(x1.x, s0.z, t0.z), 0.f), fmaxf(fmaf(x1.y, s0.w, t0.w), 0.f));
            v[i].z = pack_half2(fmaxf(fmaf(x2.x, s1.x, t1.x), 0.f), fmaxf(fmaf(x2.y, s1.y, t1.y), 0.f));
            v[i].w = pack_half2(fmaxf(fmaf(x3.x, s1.z, t1.z), 0.f), fmaxf(fmaf(x3.y, s1.w, t1.w), 0.f));
          }
#pragma unroll
          for (int i = 0; i < 8; ++i) *reinterpret_cast<uint4*>(base + i * (16 * 128)) = v[i];
          fence_proxy_async();                        // generic-proxy writes -> visible to wgmma's shared-memory reads
          mbar_arrive(&xf_full[s]);
        }
      }
    }
  }
}

}  // namespace b2
