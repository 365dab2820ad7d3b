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
//
// Dual instance (pgemm_kernel<BN, 0, 4>, b2_gemm_dual_f16): a second fp16 output taken from the same fp32 accumulator,
//     d2 = relu(scale2[n] * acc + shift2[n]),
// next to d = act(scale[n] * acc + shift[n] + residual).  One application of a PolyNet poly-3 module closes with it: d is the
// running sum, d2 the next application's input, from one pass over the concatenated branches.
//
// Split-K instance (pgemm_kernel<BN, 0, 5>, b2_gemm_splitk_f16): work item t = s * tiles_mn + (output tile) accumulates the K blocks
// [s * nkb / S, (s + 1) * nkb / S) of that tile and stores its raw fp32 accumulators into slice s of a workspace [S][M][ldw] (no
// affine, no staging, no TMA store).  splitk_reduce_kernel then sums the S slices of each element in the order 0..S-1, applies the
// per-column affine and ReLU and writes fp16 or fp32.  The fully connected classifiers of VGG / AlexNet have M = batch rows, so
// their 128-row output tiles number fewer than the SMs while each walks a K of up to 25088; the splits put the idle SMs to work on
// the same weight stream.  No atomics: the result does not depend on the schedule.
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
  int dual;                 // pgemm_kernel<BN, 0, 4> too: d2 = relu(scale2[n] * acc + shift2[n]) of the accumulator (aff2_ld = 0)
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
  // pgemm_kernel<BN, 0, 2> only: per-sample affine at ANY rows per sample (aff_rows need not divide 128, so a tile may straddle
  // samples).  Each fragment row resolves its own sample n = m / aff_rows with this divider and reads row n of scale / shift.
  FastDiv fd_aff;
  // pgemm_kernel<BN, 0, 3> only: column-slice destinations.  The Ncols = ldy packed columns are whole 64-column store boxes;
  // destination d owns boxes [split_box[d], split_box[d + 1]) (split_box[d] = INT_MAX past the last one) and box b of it
  // lands at its column 64 (b - split_box[d]) through tensor map d (tmC, tmR, tmC2, tmA2: the residual, second-output and
  // second-operand maps this instance never reads).  Each map spans only its destination's columns, so TMA drops the
  // padding columns of a ragged last box and nothing outside the slice is written.
  int split_box[4];
  // pgemm_kernel<BN, 0, 5> only: K splits, output tiles per split (tiles_total = splits * tiles_mn), fp32 workspace [splits][M][ldw]
  int splits, tiles_mn, ldw;
  float* ws;
};

template <int BN, int GAN, int C2 = GAN>   // C2: a second-output staging tile (generator and dual instances)
struct PgemmSmem {
  static constexpr int kABytes = 128 * 128;
  static constexpr int kBBytes = BN * 128;
  static constexpr int kStage = kABytes + kBBytes;
  static constexpr int kTile = 128 * BN * 2;                 // fp16 128 x BN tile: BN / 64 boxes of [128 rows][128 B], 128B-swizzled
  static constexpr int kAffBytes = 2 * 4 * BN * 4;           // per consumer warpgroup: scale, shift, scale2, shift2 of the tile
  static constexpr int kFixed = 2 * kTile + (C2 ? kTile : 0) + 256 + kAffBytes + 1024;
  // operand ring: as deep as the budget allows, up to kPgMaxStages (BN = 128: 4 stages, 3 with the generator's second-output tile)
  static constexpr int kStages = (227 * 1024 - kFixed) / kStage < kPgMaxStages ? (227 * 1024 - kFixed) / kStage : kPgMaxStages;
  static constexpr int kResOff = kStages * kStage;           // 2 residual / output staging tiles
  static constexpr int kC2Off = kResOff + 2 * kTile;         // second-output staging tile (generator instance)
  static constexpr int kBarOff = kC2Off + (C2 ? kTile : 0);
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

template <int BN, int GAN, int EPI = 0>    // GAN = 1: instance with the generator extras (res_up gather, res_pre, dual output, A transform);
                                           // 0: the classic epilogue.  With GAN = 0, EPI = 1: ReLU-derivative mask operand (fine-tuning
                                           // backward); EPI = 2: per-sample affine resolved per fragment row (see PgemmParams::fd_aff);
                                           // EPI = 3: column-slice destinations; EPI = 4: second output from the accumulator (dual);
                                           // EPI = 5: split-K partial accumulators into the workspace (see PgemmParams::splits)
__global__ void __launch_bounds__(GAN ? kPgThreadsGan : kPgThreads, 1)
pgemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
             const __grid_constant__ CUtensorMap tmA2, const __grid_constant__ CUtensorMap tmB2,
             const __grid_constant__ CUtensorMap tmC, const __grid_constant__ CUtensorMap tmR,
             const __grid_constant__ CUtensorMap tmC2, const PgemmParams p) {
  using S = PgemmSmem<BN, GAN, GAN || EPI == 4>;
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
      const int tmn = EPI == 5 ? tile % p.tiles_mn : tile, sp = EPI == 5 ? tile / p.tiles_mn : 0;
      const int m0 = (tmn / p.tiles_n) * 128, n0 = (tmn % p.tiles_n) * BN;
      const int kb_lo = EPI == 5 ? sp * p.nkb / p.splits : 0, kb_hi = EPI == 5 ? (sp + 1) * p.nkb / p.splits : p.nkb + p.nkb2;
      for (int kb = kb_lo; kb < kb_hi; ++kb, ++it) {
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
      const int tmn = EPI == 5 ? tile % p.tiles_mn : tile, sp = EPI == 5 ? tile / p.tiles_mn : 0;
      const int m0 = (tmn / p.tiles_n) * 128, n0 = (tmn % p.tiles_n) * BN;
      const int kb_lo = EPI == 5 ? sp * nkb / p.splits : 0, kb_hi = EPI == 5 ? (sp + 1) * nkb / p.splits : nkb_all;
      // the tile's affine, fetched before the main loop and stored after it
      float aff[4] = {0.f, 0.f, 0.f, 0.f};
      if (EPI != 2 && EPI != 5 && wt < BN && n0 + wt < p.Ncols) {
        // per-sample affine (class-conditional BN of the consumer): a 128-row tile never straddles two samples
        const size_t arow = p.aff_ld ? static_cast<size_t>(m0 / p.aff_rows) * p.aff_ld : 0;
        aff[0] = __ldg(&p.scale[arow + n0 + wt]);
        aff[1] = __ldg(&p.shift[arow + n0 + wt]);
        if ((GAN || EPI == 4) && p.dual) {
          const size_t arow2 = static_cast<size_t>(m0 / p.aff2_rows) * p.aff2_ld;
          aff[2] = __ldg(&p.scale2[arow2 + n0 + wt]);
          aff[3] = __ldg(&p.shift2[arow2 + n0 + wt]);
        }
      }
#pragma unroll
      for (int k = 0; k < BN / 2; ++k) acc[k] = 0.f;
      reg_fence(acc);
      int prev_s = -1;
      for (int kb = kb_lo; kb < kb_hi; ++kb, ++it) {
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
      if constexpr (EPI == 5) {
        // raw accumulators of split sp; rows past M and columns past ldw (ragged last tiles) are dropped
        float* ws = p.ws + static_cast<size_t>(sp) * p.M * p.ldw;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int col = n0 + 8 * j + fc;
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            const int row = m0 + fr + 8 * i;
            if (row < p.M && col < p.ldw)
              *reinterpret_cast<float2*>(ws + static_cast<size_t>(row) * p.ldw + col) = make_float2(acc[4 * j + 2 * i], acc[4 * j + 2 * i + 1]);
          }
        }
        continue;
      }
      uint8_t* stage = smem + S::kResOff + rb * S::kTile;
      uint8_t* stage2 = smem + S::kC2Off;                  // second output (generator / dual instances): free since the bar above
      int rsrc[2] = {fr, fr + 8};                          // row of the residual box each fragment row adds
      const float* aff_rs[2] = {nullptr, nullptr};         // EPI = 2: scale / shift rows of the two fragment rows' samples
      const float* aff_rh[2] = {nullptr, nullptr};
      if constexpr (EPI == 2) {
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int m = min(m0 + fr + 8 * i, p.M - 1);    // rows past M (ragged last tile) are computed but never stored
          const size_t off = static_cast<size_t>(fdiv(m, p.fd_aff)) * p.aff_ld;
          aff_rs[i] = p.scale + off;
          aff_rh[i] = p.shift + off;
        }
      }
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
          if constexpr (EPI == 4) {
            // d2 from the accumulator before the first epilogue overwrites it (columns >= Ncols: zero affine, relu(0) = 0)
            const float2 sc2 = *reinterpret_cast<const float2*>(s_aff + 2 * BN + c);
            const float2 sh2 = *reinterpret_cast<const float2*>(s_aff + 3 * BN + c);
            *reinterpret_cast<uint32_t*>(stage2 + pg_sw_off(fr + 8 * i, j, fc)) =
                pack_half2(fmaxf(a0 * sc2.x + sh2.x, 0.f), fmaxf(a1 * sc2.y + sh2.y, 0.f));
          }
          if (GAN && p.res_pre) {
            a0 = (a0 + rf.x) * sc.x + sh.x;
            a1 = (a1 + rf.y) * sc.y + sh.y;
          } else {
            a0 = a0 * sc.x + sh.x + rf.x;
            a1 = a1 * sc.y + sh.y + rf.y;
          }
          if constexpr (EPI == 2) {
            // this fragment row's sample: columns >= Ncols get a zero affine (and a TMA zero-filled residual), so the pitch stays zero
            float2 rs = make_float2(0.f, 0.f), rh = make_float2(0.f, 0.f);
            if (n0 + c < p.Ncols) {
              rs = __ldg(reinterpret_cast<const float2*>(aff_rs[i] + n0 + c));
              rh = __ldg(reinterpret_cast<const float2*>(aff_rh[i] + n0 + c));
            }
            a0 = acc[4 * j + 2 * i] * rs.x + rh.x + rf.x;
            a1 = acc[4 * j + 2 * i + 1] * rs.y + rh.y + rf.y;
          }
          if (p.relu) { a0 = fmaxf(a0, 0.f); a1 = fmaxf(a1, 0.f); }
          if constexpr (EPI == 1) {
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
          if constexpr (EPI == 3) {
            const int box = (n0 >> 6) + b;
            int d = 0;
#pragma unroll
            for (int e = 1; e < 4; ++e) d = box >= p.split_box[e] ? e : d;
            const CUtensorMap* tm = d == 0 ? &tmC : d == 1 ? &tmR : d == 2 ? &tmC2 : &tmA2;
            if (n0 + b * 64 < p.ldy) tma_store_2d(tm, stage + b * (128 * 128) + wg * (64 * 128), (box - p.split_box[d]) * 64, m0 + wg * 64);
          } else {
            if (n0 + b * 64 < p.ldy) tma_store_2d(&tmC, stage + b * (128 * 128) + wg * (64 * 128), n0 + b * 64, m0 + wg * 64);
          }
        if constexpr (EPI == 4) {
          // d2 has d's pitch: its columns [Ncols, ldy) are written as zero too (zero affine, zero-filled B rows)
#pragma unroll
          for (int b = 0; b < BN / 64; ++b)
            if (n0 + b * 64 < p.ldy) tma_store_2d(&tmC2, stage2 + b * (128 * 128) + wg * (64 * 128), n0 + b * 64, m0 + wg * 64);
        }
        tma_store_commit();
      }
      if (GAN && p.dual) {                                 // second output: next block's ccbn + ReLU on the fp32 value
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

// The second pass of the split-K GEMM: d[m][n] = act(scale[n] * (ws[0][m][n] + ws[1][m][n] + ... + ws[S-1][m][n]) + shift[n]), the
// slices summed in that order in fp32, one fma with the affine, one rounding (fp16) or none (fp32).  Four columns per thread.
// fp16: columns [N, ldd) are written as zero; fp32: only columns [0, N) are written.
__global__ void __launch_bounds__(256)
splitk_reduce_kernel(const float* __restrict__ ws, int S, int M, int N, int ldw, const float* __restrict__ scale,
                     const float* __restrict__ shift, int relu, void* __restrict__ d, int ldd, int out_f32, int quads) {
  const long long idx = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= static_cast<long long>(M) * quads) return;
  const int m = static_cast<int>(idx / quads), c0 = static_cast<int>(idx % quads) * 4;
  const size_t slice = static_cast<size_t>(M) * ldw;
  float v[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int c = c0 + q;
    v[q] = 0.f;
    if (c < N) {
      const float* src = ws + static_cast<size_t>(m) * ldw + c;
      float sum = 0.f;
      for (int s = 0; s < S; ++s) sum += __ldg(src + s * slice);
      sum = fmaf(sum, __ldg(scale + c), __ldg(shift + c));
      v[q] = relu ? fmaxf(sum, 0.f) : sum;
    }
  }
  if (out_f32) {
    float* y = static_cast<float*>(d) + static_cast<size_t>(m) * ldd;
#pragma unroll
    for (int q = 0; q < 4; ++q)
      if (c0 + q < N) y[c0 + q] = v[q];
  } else {
    *reinterpret_cast<uint2*>(static_cast<__half*>(d) + static_cast<size_t>(m) * ldd + c0) = make_uint2(pack_half2(v[0], v[1]), pack_half2(v[2], v[3]));
  }
}

// ==================================================================================================================================
// Chained instance: a bottleneck's closing 1x1x1 GEMM and the NEXT block's conv1 in one pass over the block output
//
//     y  = relu( scale[n] * (A . B^T [+ A2 . B2^T]) + shift[n] [+ residual] )          [M][N],  N <= 256, N % 64 == 0, ldy == N
//     h1 = relu( scale1[n] * (y . W1^T) + shift1[n] )                                   [M][N1], ld1 <= 128
//
// A CTA owns a 128-row M block across all N columns.  The closing GEMM runs as N / BN passes of the pgemm_kernel<BN, 0> main
// loop and epilogue; each pass leaves its fp16 y columns in the 128B-swizzled [128 rows][64 columns] boxes of a full-width tile
// (which held the residual) and TMA-stores them.  Those boxes are exactly the K-major A operand layout a TMA load of y would
// produce, so the second GEMM reads them in place: K blocks of 64 columns in order, the W1 boxes streamed through the operand
// ring.  Its MMA width is the one the stand-alone conv1 launch picks (BN1 = 64 for ld1 <= 64, else 128), and both epilogues keep
// pgemm_kernel's arithmetic: the result is bit-identical to the two launches, without y's re-read from HBM.  h1 is staged in the
// first boxes of the same tile once the y stores have read them.
struct PgemmChainParams {
  int M, Ncols;             // rows, closing-GEMM columns (== output pitch)
  int nkb, nkb2;            // K blocks of the closing GEMM's two operand pairs (nkb2 = 0: none)
  int npass;                // closing-GEMM passes of BN columns
  int tiles_total;          // 128-row M blocks
  const float* scale;
  const float* shift;
  int has_residual, relu;
  int N1, ld1;              // chained GEMM: logical columns, output pitch (columns [N1, ld1) are written as zero)
  const float* scale1;
  const float* shift1;
};

template <int BN, int BN1>
struct PgemmChainSmem {
  static constexpr int kStages = 3;
  static constexpr int kABytes = 128 * 128;
  static constexpr int kStage = kABytes + 128 * 128;         // A box + B box of up to 128 rows (closing B, or a W1 K block)
  static constexpr int kFull = 128 * 256 * 2;                // full-width fp16 tile: residual, y staging, A of the chained GEMM, h1 staging
  static constexpr int kFullOff = kStages * kStage;          // 2 full-width tiles: the next tile's residual lands during this one
  static constexpr int kBarOff = kFullOff + 2 * kFull;
  static constexpr int kTotal = kBarOff + 256 + 1024;        // + barriers, + alignment slack
  // 3 x 32 KB ring + 2 x 64 KB tiles + 256 B barriers + 1 KB slack = 225.25 KB
  static_assert(kTotal <= 227 * 1024, "shared memory budget");
  static_assert(BN * 128 <= kStage - kABytes && BN1 * 128 <= kStage - kABytes, "B box exceeds the ring slot");
};

template <int BN, int BN1>
__global__ void __launch_bounds__(kPgThreads, 1)
pgemm_chain_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                   const __grid_constant__ CUtensorMap tmA2, const __grid_constant__ CUtensorMap tmB2,
                   const __grid_constant__ CUtensorMap tmC, const __grid_constant__ CUtensorMap tmR,
                   const __grid_constant__ CUtensorMap tmW1, const __grid_constant__ CUtensorMap tmH,
                   const PgemmChainParams p) {
  using S = PgemmChainSmem<BN, BN1>;
  constexpr int kSt = S::kStages;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_align<1024>(smem_raw);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + S::kBarOff);   // [kSt]
  uint64_t* empty = full + kSt;                                      // [kSt]
  uint64_t* res_full = empty + kSt;                                  // [2]
  uint64_t* res_empty = res_full + 2;                                // [2]
  const int tid = threadIdx.x, warp = tid >> 5;
  const int nkc = p.Ncols / 64;                                      // K blocks of the chained GEMM

  if (tid == 0) {
    for (int s = 0; s < kSt; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 2); }
    for (int i = 0; i < 2; ++i) { mbar_init(&res_full[i], 1); mbar_init(&res_empty[i], 2); }
    fence_mbar_init();
    tma_prefetch_desc(&tmA); tma_prefetch_desc(&tmB); tma_prefetch_desc(&tmC); tma_prefetch_desc(&tmW1);
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();

  if (warp == kPgProdWarp) {
    // ================================ producer ==========================================
    // per tile: the closing K blocks of each pass (the residual after the first pass's), then the W1 K blocks
    int it = 0, lt = 0;
    for (int tile = blockIdx.x; tile < p.tiles_total; tile += gridDim.x, ++lt) {
      const int m0 = tile * 128;
      for (int pass = 0; pass < p.npass; ++pass) {
        const int n0 = pass * BN;
        for (int kb = 0; kb < p.nkb + p.nkb2; ++kb, ++it) {
          const int s = it % kSt;
          mbar_wait(&empty[s], ((it / kSt) & 1) ^ 1);
          if (elect_one()) {
            mbar_expect_tx(&full[s], S::kABytes + BN * 128);
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
        if (pass == 0) {
          const int rb = lt & 1;
          mbar_wait(&res_empty[rb], ((lt >> 1) & 1) ^ 1);
          if (elect_one()) {
            if (p.has_residual) {
              mbar_expect_tx(&res_full[rb], static_cast<uint32_t>(nkc) * (128 * 128));
              for (int b = 0; b < nkc; ++b) tma_load_2d(smem + S::kFullOff + rb * S::kFull + b * (128 * 128), &tmR, &res_full[rb], b * 64, m0);
            } else {
              mbar_arrive(&res_full[rb]);
            }
          }
          __syncwarp();
        }
      }
      for (int kb = 0; kb < nkc; ++kb, ++it) {
        const int s = it % kSt;
        mbar_wait(&empty[s], ((it / kSt) & 1) ^ 1);
        if (elect_one()) {
          mbar_expect_tx(&full[s], BN1 * 128);
          tma_load_2d(smem + s * S::kStage + S::kABytes, &tmW1, &full[s], kb * 64, 0);
        }
        __syncwarp();
      }
    }
  } else {
    // ================================ consumer warpgroups ===============================
    // Fragment layout, ring protocol and epilogue as in pgemm_kernel; the affines are read from global memory (L1) instead of a
    // shared-memory copy, which the full-width tiles leave no room for.
    const int wg = warp >> 2, wt = tid & 127;
    const bool leader = wt == 0;
    const int bar_wg = 1 + wg;
    const int fr = wg * 64 + (warp & 3) * 16 + ((tid & 31) >> 2);
    const int fc = 2 * (tid & 3);
    const uint32_t ring = smem_u32(smem);
    const uint32_t a_wg = static_cast<uint32_t>(wg) * (64u * 128u >> 4);
    const int nkb_all = warp_uniform(p.nkb + p.nkb2), npass = warp_uniform(p.npass);
    float acc[(BN > BN1 ? BN : BN1) / 2];
    int it = 0, lt = 0;
    for (int tile = blockIdx.x; tile < p.tiles_total; tile += gridDim.x, ++lt) {
      const int m0 = tile * 128;
      const int rb = lt & 1;
      uint8_t* tile_s = smem + S::kFullOff + rb * S::kFull;
      for (int pass = 0; pass < npass; ++pass) {
        const int n0 = pass * BN;
#pragma unroll
        for (int k = 0; k < BN / 2; ++k) acc[k] = 0.f;
        reg_fence(acc);
        int prev_s = -1;
        for (int kb = 0; kb < nkb_all; ++kb, ++it) {
          const int s = it % kSt;
          mbar_wait(&full[s], (it / kSt) & 1);
          const uint64_t a = desc_from(kSw128DescHi, sw128_desc_lo(ring + s * S::kStage) + a_wg);
          const uint64_t b = desc_from(kSw128DescHi, sw128_desc_lo(ring + s * S::kStage + S::kABytes));
          wgmma_fence();
#pragma unroll
          for (int k = 0; k < 4; ++k) wgmma_ss<BN>(acc, a + 2 * k, b + 2 * k);
          wgmma_commit();
          wgmma_wait1();
          if (leader && prev_s >= 0) mbar_arrive(&empty[prev_s]);
          prev_s = s;
        }
        wgmma_wait0();
        reg_fence(acc);
        if (leader) {
          mbar_arrive(&empty[prev_s]);
          // the h1 stores of the previous tile had this main loop to read their staging boxes: hand that tile back
          if (pass == 0 && lt > 0) { tma_store_wait_read0(); mbar_arrive(&res_empty[(lt - 1) & 1]); }
        }
        if (pass == 0) mbar_wait(&res_full[rb], (lt >> 1) & 1);
        uint8_t* stage = tile_s + n0 * (128 * 2);          // boxes n0 / 64 .. of the full-width tile
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int c = n0 + 8 * j + fc;
          float2 sc = make_float2(0.f, 0.f), sh = make_float2(0.f, 0.f);
          if (c < p.Ncols) { sc = make_float2(__ldg(p.scale + c), __ldg(p.scale + c + 1)); sh = make_float2(__ldg(p.shift + c), __ldg(p.shift + c + 1)); }
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            float2 rf = make_float2(0.f, 0.f);
            if (p.has_residual) rf = unpack_half2(*reinterpret_cast<const uint32_t*>(stage + pg_sw_off(fr + 8 * i, j, fc)));
            float a0 = acc[4 * j + 2 * i], a1 = acc[4 * j + 2 * i + 1];
            a0 = a0 * sc.x + sh.x + rf.x;
            a1 = a1 * sc.y + sh.y + rf.y;
            if (p.relu) { a0 = fmaxf(a0, 0.f); a1 = fmaxf(a1, 0.f); }
            *reinterpret_cast<uint32_t*>(stage + pg_sw_off(fr + 8 * i, j, fc)) = pack_half2(a0, a1);
          }
        }
        fence_proxy_async();                               // y: generic-proxy writes -> the bulk store and the chained wgmma
        pg_bar(bar_wg, 128);
        if (leader && m0 + wg * 64 < p.M) {
#pragma unroll
          for (int b = 0; b < BN / 64; ++b)
            if (n0 + b * 64 < p.Ncols) tma_store_2d(&tmC, stage + b * (128 * 128) + wg * (64 * 128), n0 + b * 64, m0 + wg * 64);
          tma_store_commit();
        }
      }

      // ---- chained GEMM: this warpgroup's 64 rows of y (in the tile) times W1^T ----
#pragma unroll
      for (int k = 0; k < BN1 / 2; ++k) acc[k] = 0.f;
      reg_fence(acc);
      int prev_s = -1;
      const uint32_t ya = smem_u32(tile_s);
      for (int kb = 0; kb < nkc; ++kb, ++it) {
        const int s = it % kSt;
        mbar_wait(&full[s], (it / kSt) & 1);
        const uint64_t a = desc_from(kSw128DescHi, sw128_desc_lo(ya + kb * (128 * 128)) + a_wg);
        const uint64_t b = desc_from(kSw128DescHi, sw128_desc_lo(ring + s * S::kStage + S::kABytes));
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < 4; ++k) wgmma_ss<BN1>(acc, a + 2 * k, b + 2 * k);
        wgmma_commit();
        wgmma_wait1();
        if (leader && prev_s >= 0) mbar_arrive(&empty[prev_s]);
        prev_s = s;
      }
      wgmma_wait0();
      reg_fence(acc);
      if (leader) {
        mbar_arrive(&empty[prev_s]);
        tma_store_wait_read0();                            // the y stores have read the boxes h1 is staged in
      }
      pg_bar(bar_wg, 128);
#pragma unroll
      for (int j = 0; j < BN1 / 8; ++j) {
        const int c = 8 * j + fc;
        float2 sc = make_float2(0.f, 0.f), sh = make_float2(0.f, 0.f);
        if (c < p.N1) { sc.x = __ldg(p.scale1 + c); sh.x = __ldg(p.shift1 + c); }
        if (c + 1 < p.N1) { sc.y = __ldg(p.scale1 + c + 1); sh.y = __ldg(p.shift1 + c + 1); }
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const float2 rf = make_float2(0.f, 0.f);         // the stand-alone conv1 epilogue adds its (absent) residual as zero
          float a0 = acc[4 * j + 2 * i], a1 = acc[4 * j + 2 * i + 1];
          a0 = fmaxf(a0 * sc.x + sh.x + rf.x, 0.f);
          a1 = fmaxf(a1 * sc.y + sh.y + rf.y, 0.f);
          *reinterpret_cast<uint32_t*>(tile_s + pg_sw_off(fr + 8 * i, j, fc)) = pack_half2(a0, a1);
        }
      }
      fence_proxy_async();
      pg_bar(bar_wg, 128);
      if (leader && m0 + wg * 64 < p.M) {
#pragma unroll
        for (int b = 0; b < BN1 / 64; ++b)
          if (b * 64 < p.ld1) tma_store_2d(&tmH, tile_s + b * (128 * 128) + wg * (64 * 128), b * 64, m0 + wg * 64);
        tma_store_commit();
      }
    }
    if (leader) tma_store_wait_read0();
  }
}

}  // namespace b2
