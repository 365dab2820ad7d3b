// b2_pgemm.cuh -- persistent, warp-specialised GEMM for the 1x1x1 convolutions and dense layers:
//
//     D[M][N] = act( scale[n] * (A[M][K] . B[N][K]^T  [+ A2[M][K2] . B2[N][K2]^T]) + shift[n] + residual[M][N] )
//                                                                                   (fp16 in/out, fp32 accumulate)
// The optional second operand pair accumulates into the same accumulator tile: it fuses the type-B shortcut projection of a
// bottleneck into its closing 1x1x1 convolution (BN scales folded into the two weight matrices), so the projected
// shortcut never goes through HBM.
//
// These layers are HBM-bound (K is 64..2048 while every output element is written once and, for the block-closing
// conv3, a residual element is read once), so the kernel is organised around keeping the memory system busy rather
// than the tensor core: one CTA per SM loops over output tiles, and the three stages of a tile -- TMA loads of A/B
// (and of the residual tile), the wgmma MMAs, and the epilogue (accumulators -> registers -> BN/residual/ReLU -> smem ->
// TMA store) -- belong to different warps and overlap across consecutive tiles through double-buffered accumulator
// tiles in shared memory, a double-buffered residual tile and an smem operand ring.  The non-persistent igemm_kernel
// pays the barrier set-up and a cold pipeline for every tile; with K = 64 that prologue dominates.
// Only the 64-wide instance fits: two 128 x 128 fp32 accumulator tiles beside the ring and the staging tiles of a
// 128-wide tile would exceed 227 KB.
//
//   warps 8-11  MMA warpgroup: accumulates tile i into accumulator buffer i & 1
//   warp 12     producer: residual tile of tile i, then its K blocks (A and B boxes, 128B-swizzled)
//   warps 0-7   epilogue of tile i (thread = accumulator row x one half of the columns), TMA store from a staging tile
#pragma once

#include "b2_ptx.cuh"

namespace b2 {

constexpr int kPgEpiWarps = 8;                       // two warps per 32 accumulator rows, each takes half of the columns
constexpr int kPgMmaWarp0 = kPgEpiWarps;
constexpr int kPgProdWarp = kPgMmaWarp0 + 4;
constexpr int kPgXformWarp0 = kPgProdWarp + 1;
constexpr int kPgThreads = (kPgProdWarp + 1) * 32;
constexpr int kPgXformWarps = 4;                     // generator instance only: A-operand transform warps (see PgemmParams::in_scale)
constexpr int kPgThreadsGan = (kPgXformWarp0 + kPgXformWarps) * 32;
constexpr int kPgStages = 3;

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
  // res_rows = 64 (resp. 32) CONSECUTIVE rows of the low-res matrix: one TMA box per 64 columns, loaded a tile ahead like
  // the plain residual, and the epilogue thread of row r reads row src(r) of that box.  pgemm_kernel<BN, 1> only.
  const __half* res_up;
  int res_ld, Wh, Hh;
  int res_rows;             // rows of the low-res residual box: 64 (Wh >= 128) or 32
  FastDiv fd_Wh, fd_Hh;
  int res_pre;              // 1: y = act(scale * (acc + residual) + shift) instead of act(scale * acc + shift + residual)
  // Second output (pgemm_kernel<BN, 1>): y2 = relu(y * scale2[m / aff2_rows][n] + shift2[...]) -- the class-conditional
  // BatchNorm + ReLU of the NEXT block applied to this block's fp32 result, written through tmC2 in a second epilogue pass
  // over the same accumulator (the HBM-bound tile loop has the issue slots to spare; no extra shared memory).
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

template <int BN>
struct PgemmSmem {
  static constexpr int kABytes = 128 * 128;
  static constexpr int kBBytes = BN * 128;
  static constexpr int kStage = kABytes + kBBytes;
  static constexpr int kTile = 128 * BN * 2;                 // one C / residual staging tile
  static constexpr int kRing = kPgStages * kStage;
  static constexpr int kResOff = kRing;                      // 2 residual tiles
  static constexpr int kCOff = kResOff + 2 * kTile;          // 1 C tile
  static constexpr int kC2Off = kCOff + kTile;               // second C tile (second output; 64-wide instance only: the
                                                             // 128-wide one has no room and falls back to re-using C)
  static constexpr int kBarOff = kC2Off + (BN == 64 ? kTile : 0);
  static constexpr int kAffOff = kBarOff + 256;              // scale[BN], shift[BN] (+ scale2[BN], shift2[BN]) of the current tile
  static constexpr int kAccOff = kAffOff + 4 * BN * 4;       // two accumulator tiles of BN columns
  static constexpr int kTotal = kAccOff + acc_bytes(2 * BN) + 1024;
  static_assert(kTotal <= 227 * 1024, "shared memory budget");
};

template <int BN, int GAN, int MASK = 0>   // GAN = 1: instance with the generator extras (res_up gather, res_pre, A transform); 0: the classic
                                           // epilogue.  MASK = 1 (with GAN = 0): ReLU-derivative mask operand (fine-tuning backward)
__global__ void __launch_bounds__(GAN ? kPgThreadsGan : kPgThreads, 1)
pgemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
             const __grid_constant__ CUtensorMap tmA2, const __grid_constant__ CUtensorMap tmB2,
             const __grid_constant__ CUtensorMap tmC, const __grid_constant__ CUtensorMap tmR,
             const __grid_constant__ CUtensorMap tmC2, const PgemmParams p) {
  using S = PgemmSmem<BN>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_align<1024>(smem_raw);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + S::kBarOff);   // [3]
  uint64_t* empty = full + kPgStages;                                // [3]
  uint64_t* acc_full = empty + kPgStages;                            // [2]
  uint64_t* acc_empty = acc_full + 2;                                // [2]
  uint64_t* res_full = acc_empty + 2;                                // [2]
  uint64_t* res_empty = res_full + 2;                                // [2]
  const AccTile at{reinterpret_cast<float*>(smem + S::kAccOff), acc_ld(2 * BN)};
  uint64_t* xf_full = reinterpret_cast<uint64_t*>(smem + S::kBarOff + 128);   // [3] A tile transformed (generator instance)
  const bool xform = GAN && p.in_scale != nullptr;

  const int tid = threadIdx.x, warp = tid >> 5;

  if (tid == kPgEpiWarps * 32) {
    for (int s = 0; s < kPgStages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 1); mbar_init(&xf_full[s], kPgXformWarps * 32); }
    for (int i = 0; i < 2; ++i) {
      mbar_init(&acc_full[i], 1); mbar_init(&acc_empty[i], kPgEpiWarps * 32);
      mbar_init(&res_full[i], 1); mbar_init(&res_empty[i], kPgEpiWarps * 32);
    }
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
      const int rb = lt & 1;
      if (p.has_residual) {
        mbar_wait(&res_empty[rb], ((lt >> 1) & 1) ^ 1);
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
        __syncwarp();
      }
      for (int kb = 0; kb < p.nkb + p.nkb2; ++kb, ++it) {
        const int s = it % kPgStages;
        mbar_wait(&empty[s], ((it / kPgStages) & 1) ^ 1);
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
    }
  } else if (warp >= kPgMmaWarp0 && warp < kPgMmaWarp0 + 4) {
    // ================================ MMA warpgroup =====================================
    const uint32_t ring = smem_u32(smem);
    int it = 0, lt = 0;
    for (int tile = blockIdx.x; tile < p.tiles_total; tile += gridDim.x, ++lt) {
      const int ab = lt & 1;
      mbar_wait(&acc_empty[ab], ((lt >> 1) & 1) ^ 1);        // epilogue has drained this accumulator
      const int nkb_all = p.nkb + p.nkb2;
      for (int kb = 0; kb < nkb_all; ++kb, ++it) {
        const int s = it % kPgStages;
        if (xform && kb < p.nkb) mbar_wait(&xf_full[s], (it / kPgStages) & 1);     // operands landed AND the A tile was rewritten
        else mbar_wait(&full[s], (it / kPgStages) & 1);
        const uint32_t a_lo = sw128_desc_lo(ring + s * S::kStage);
        const uint32_t b_lo = sw128_desc_lo(ring + s * S::kStage + S::kABytes);
        wg_mma(at, ab * BN, BN, wg_sw128(desc_from(kSw128DescHi, a_lo), desc_from(kSw128DescHi, b_lo)), 4, kb != 0);
        wg_sync();
        wg_arrive(&empty[s]);
        if (kb == nkb_all - 1) wg_arrive(&acc_full[ab]);
      }
    }
  } else if (GAN && warp >= kPgXformWarp0) {
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
          const int s = it % kPgStages;
          const float4* sc4 = reinterpret_cast<const float4*>(p.in_scale + arow + kb * 64 + j * 8);
          const float4* sh4 = reinterpret_cast<const float4*>(p.in_shift + arow + kb * 64 + j * 8);
          const float4 s0 = __ldg(sc4), s1 = __ldg(sc4 + 1), t0 = __ldg(sh4), t1 = __ldg(sh4 + 1);   // before the wait: independent of the tile
          mbar_wait(&full[s], (it / kPgStages) & 1);
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
  } else {
    // ================================ epilogue ==========================================
    float* s_scale = reinterpret_cast<float*>(smem + S::kAffOff);
    float* s_shift = s_scale + BN;
    float* s_scale2 = s_shift + BN;
    float* s_shift2 = s_scale2 + BN;
    const int r = (warp & 3) * 32 + (tid & 31);        // accumulator row
    const int half = warp >> 2;                        // which half of the tile's columns this warp handles
    const uint32_t swz = static_cast<uint32_t>(r & 7);
    uint8_t* c_stage0 = smem + S::kCOff;
    uint8_t* c_stage1 = smem + (BN == 64 ? S::kC2Off : S::kCOff);
    int lt = 0;
    for (int tile = blockIdx.x; tile < p.tiles_total; tile += gridDim.x, ++lt) {
      const int m0 = (tile / p.tiles_n) * 128, n0 = (tile % p.tiles_n) * BN;
      const int ab = lt & 1;
      mbar_wait(&acc_full[ab], (lt >> 1) & 1);
      const uint8_t* r_stage = smem + S::kResOff + ab * S::kTile;
      int rsrc = r;                                        // row of the residual box this thread's output row adds
      if (GAN && p.res_up) {
        if (p.Wh >= 128) rsrc = r >> 1;
        else { const int hr = fdiv(r, p.fd_Wh); rsrc = (hr >> 1) * (p.Wh >> 1) + ((r - hr * p.Wh) >> 1); }
      }
      const uint32_t rswz = static_cast<uint32_t>(rsrc & 7);
      if (p.has_residual) mbar_wait(&res_full[ab], (lt >> 1) & 1);
      const int npass = (GAN && p.dual) ? 2 : 1;
#pragma unroll 1
      for (int pass = 0; pass < npass; ++pass) {
        // the previous TMA store must have finished reading the staging tile before we overwrite it (the second pass of
        // the 64-wide instance has its own tile: nothing to wait for)
        // Without a residual the two residual tiles are free: the C staging tile alternates between them and its own slot, and
        // only the store of two tiles ago has to have drained -- the TMA store of tile i then overlaps the epilogue math of
        // tile i + 1 (write-dominated layers, e.g. the 64 -> 256 expansions, were serialised on that drain).
        const bool alt = !p.has_residual && !(GAN && p.dual);
        uint8_t* c_stage = pass == 0 ? ((alt && (lt & 1)) ? smem + S::kResOff : c_stage0) : c_stage1;
        if (pass == 0 || BN != 64) {
          if (tid == 0) { if (alt) tma_store_wait_read1(); else tma_store_wait_read0(); }
          asm volatile("bar.sync 1, 256;" ::: "memory");   // (also: everyone is done with the previous tile's affine)
        }
        if (pass == 0 && tid < BN) {
          const int c = n0 + tid;
          // per-sample affine (class-conditional BN of the consumer): a 128-row tile never straddles two samples
          const size_t arow = p.aff_ld ? static_cast<size_t>(m0 / p.aff_rows) * p.aff_ld : 0;
          s_scale[tid] = (c < p.Ncols) ? __ldg(&p.scale[arow + c]) : 0.f;
          s_shift[tid] = (c < p.Ncols) ? __ldg(&p.shift[arow + c]) : 0.f;
          if (GAN && p.dual) {
            const size_t arow2 = static_cast<size_t>(m0 / p.aff2_rows) * p.aff2_ld;
            s_scale2[tid] = (c < p.Ncols) ? __ldg(&p.scale2[arow2 + c]) : 0.f;
            s_shift2[tid] = (c < p.Ncols) ? __ldg(&p.shift2[arow2 + c]) : 0.f;
          }
        }
        if (pass == 0) asm volatile("bar.sync 1, 256;" ::: "memory");
#pragma unroll 1
        for (int j = half * (BN / 64); j < (half + 1) * (BN / 64); ++j) {
          uint32_t v[32];
          acc_ld32(at, r, ab * BN + j * 32, v);
          const int box = j >> 1, chunk0 = (j & 1) * 4;
          uint8_t* crow = c_stage + box * (128 * 128) + r * 128;
          const uint8_t* rrow = r_stage + box * (128 * 128) + rsrc * 128;
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const uint32_t coff = (static_cast<uint32_t>(chunk0 + q) ^ swz) << 4;
            uint4 rv = make_uint4(0, 0, 0, 0);
            if (p.has_residual) rv = *reinterpret_cast<const uint4*>(rrow + ((static_cast<uint32_t>(chunk0 + q) ^ rswz) << 4));
            const uint32_t rr[4] = {rv.x, rv.y, rv.z, rv.w};
            uint4 mv = make_uint4(0, 0, 0, 0);
            if constexpr (MASK) {
              const int mrow = m0 + r, mcol = n0 + j * 32 + q * 8;
              if (mrow < p.M && mcol < p.ldm) mv = __ldg(reinterpret_cast<const uint4*>(p.mask + static_cast<size_t>(mrow) * p.ldm + mcol));
            }
            const uint32_t mm[4] = {mv.x, mv.y, mv.z, mv.w};
            uint32_t out[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              const int ci = j * 32 + q * 8 + e * 2;
              const float2 rf = unpack_half2(rr[e]);
              float a0 = __uint_as_float(v[q * 8 + e * 2]), a1 = __uint_as_float(v[q * 8 + e * 2 + 1]);
              if (GAN && p.res_pre) {
                a0 = (a0 + rf.x) * s_scale[ci] + s_shift[ci];
                a1 = (a1 + rf.y) * s_scale[ci + 1] + s_shift[ci + 1];
              } else {
                a0 = a0 * s_scale[ci] + s_shift[ci] + rf.x;
                a1 = a1 * s_scale[ci + 1] + s_shift[ci + 1] + rf.y;
              }
              if (p.relu) { a0 = fmaxf(a0, 0.f); a1 = fmaxf(a1, 0.f); }
              if constexpr (MASK) {
                const float2 mf = unpack_half2(mm[e]);
                a0 = mf.x > 0.f ? a0 : 0.f;
                a1 = mf.y > 0.f ? a1 : 0.f;
              }
              if (GAN && pass == 1) {                          // second output: next block's ccbn + ReLU on the fp32 value
                a0 = fmaxf(a0 * s_scale2[ci] + s_shift2[ci], 0.f);
                a1 = fmaxf(a1 * s_scale2[ci + 1] + s_shift2[ci + 1], 0.f);
              }
              out[e] = pack_half2(a0, a1);
            }
            *reinterpret_cast<uint4*>(crow + coff) = make_uint4(out[0], out[1], out[2], out[3]);
          }
        }
        if (pass == npass - 1) {
          // accumulator and residual buffers are free for tile lt + 2
          mbar_arrive(&acc_empty[ab]);
          if (p.has_residual) mbar_arrive(&res_empty[ab]);
        }
        fence_proxy_async();
        asm volatile("bar.sync 1, 256;" ::: "memory");
        if (tid == 0) {
#pragma unroll
          for (int b = 0; b < BN / 64; ++b)
            if (n0 + b * 64 < p.ldy) tma_store_2d(pass == 0 ? &tmC : &tmC2, c_stage + b * (128 * 128), n0 + b * 64, m0);
          tma_store_commit();
        }
      }
    }
    if (tid == 0) tma_store_wait_read0();
  }
}

}  // namespace b2
