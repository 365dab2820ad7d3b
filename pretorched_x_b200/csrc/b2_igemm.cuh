// b2_igemm.cuh -- implicit-GEMM convolution / GEMM on wgmma with a fused BN/residual/ReLU epilogue.
//
//   D[M][N] = act( scale * (A_im2col[M][Ktot] . W[N][Ktot]^T) + shift + residual )
//
// One CTA computes one 128 x BN output tile.  9 warps:
//   warps 0-3  A producers in gather mode (cp.async im2col, one output row per thread), then
//              the epilogue (thread = accumulator row)
//   warps 4-7  MMA warpgroup (wgmma)
//   warp  8    TMA producer (weights always; activations too in AMODE_TMA)
// K is consumed in blocks of 64 fp16 (one 128-byte swizzle row) through a STAGES-deep smem ring
// guarded by full/empty mbarriers; accumulators live in a shared-memory AccTile (BN fp32 columns x 128 rows).
//
// smem tiles use the canonical K-major SWIZZLE_128B layout: row r at r*128 B, 16-byte chunk j of a
// row stored at chunk (j ^ (r & 7)).  TMA produces that layout natively; the gather producers
// reproduce it by hand.
#pragma once

#include "b2_ptx.cuh"

namespace b2 {

constexpr int kBM = 128;     // output rows (pixels) per CTA
constexpr int kBK = 64;      // K elements per pipeline stage
constexpr int kStages = 3;   // smem ring depth
constexpr int kThreads = 288;
constexpr int kIgMmaWarp0 = 4;
constexpr int kIgTmaWarp = 8;

enum : int { AMODE_TMA = 0, AMODE_GATHER = 1 };
enum : int { EPI_TMA_F16 = 0, EPI_DIRECT_F16 = 1, EPI_DIRECT_F32 = 2 };

struct IgemmParams {
  // A operand (gather modes)
  const __half* x;
  int N, T, H, W, C;       // input dims, C = channel pitch (elements)
  int To, Ho, Wo;
  int kt, kh, kw, st, sh, sw, pt, ph, pw;
  int cchunks;             // ceil(C / 64): K blocks per filter tap      (AMODE_GATHER)
  // problem
  int M_total;             // rows of D
  int Ncols;               // logical columns of D (Cout)
  int nkb;                 // number of 64-wide K blocks
  // epilogue
  const float* scale;
  const float* shift;
  const __half* residual;  // nullable
  int ldr;
  void* y;
  int ldy;
  int relu;
  int per_row;             // scale/shift indexed by row (swap-AB GEMMs)
  int accumulate;          // EPI_DIRECT_F32: y += result
  int amode;
  int epi;
  int aff_ld, aff_rows;    // per-sample affine (persistent GEMM only): scale/shift row (m / aff_rows), pitch aff_ld; 0 = off
  int res_up, res_pre;     // persistent GEMM only: residual is the low-res tensor of an (up_H x up_W) image / added before the scale
  int up_H, up_W;
  void* y2;                // persistent GEMM only: second output relu(y * scale2[m / aff2_rows] + shift2[...]) (same pitch as y)
  const float* scale2;
  const float* shift2;
  int aff2_ld, aff2_rows;
  const float* in_scale;   // persistent GEMM (generator instance) only: per-sample affine + ReLU on the A operand, see PgemmParams
  const float* in_shift;
  int in_ld, in_rows;
  const __half* mask;      // MASK instances only: fp16 [M][ldm]; the output is zeroed where mask <= 0 (ReLU derivative)
  int ldm;
};

// Eight mask entries of output row m, columns [c, c + 8) (zeros past the mask's rows / pitch), and the masked pair select.
__device__ __forceinline__ uint4 load_mask8(const IgemmParams& p, int m, int c) {
  if (m >= p.M_total || c >= p.ldm) return make_uint4(0, 0, 0, 0);
  return __ldg(reinterpret_cast<const uint4*>(p.mask + static_cast<size_t>(m) * p.ldm + c));
}
__device__ __forceinline__ void apply_mask2(uint32_t mk, float& a0, float& a1) {
  const float2 mf = unpack_half2(mk);
  a0 = mf.x > 0.f ? a0 : 0.f;
  a1 = mf.y > 0.f ? a1 : 0.f;
}

template <int BN>
struct IgemmSmem {
  static constexpr int kABytes = kBM * kBK * 2;          // 16 KB
  static constexpr int kBBytes = BN * kBK * 2;           // 8 / 16 KB
  static constexpr int kStageBytes = kABytes + kBBytes;
  static constexpr int kRingBytes = kStages * kStageBytes;
  // epilogue staging aliases the ring: C tile then residual tile, each BN/64 boxes of 128x64 fp16
  static constexpr int kCTileBytes = kBM * BN * 2;
  static_assert(2 * kCTileBytes <= kRingBytes, "epilogue staging must fit in the ring");
  static constexpr int kBarOffset = kRingBytes;          // barriers + scale/shift after the ring
  static constexpr int kAccOffset = kRingBytes + 256 + 2 * BN * 4 + 2 * kBM * 4;
  static constexpr int kTotalBytes = kAccOffset + acc_bytes(BN) + 1024 /*align slack*/;
};

template <int BN, int MASK = 0>   // MASK = 1: ReLU-derivative mask operand in the fp16 epilogue (fine-tuning backward)
__global__ void __launch_bounds__(kThreads, 1)
igemm_kernel(const __grid_constant__ CUtensorMap tmA,   // activations as [M][C] matrix (AMODE_TMA only)
             const __grid_constant__ CUtensorMap tmB,   // weights [N][Ktot]
             const __grid_constant__ CUtensorMap tmC,   // output  [M][ldy]   (EPI_TMA_F16 only)
             const __grid_constant__ CUtensorMap tmR,   // residual [M][ldr]  (EPI_TMA_F16 + residual)
             const IgemmParams p) {
  using S = IgemmSmem<BN>;
  extern __shared__ uint8_t smem_raw[];
  // SWIZZLE_128B tiles need 1024-byte alignment
  uint8_t* smem = smem_align<1024>(smem_raw);

  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + S::kBarOffset);
  uint64_t* empty_bar = full_bar + kStages;
  uint64_t* acc_full_bar = empty_bar + kStages;
  uint64_t* res_bar = acc_full_bar + 1;
  const AccTile acc{reinterpret_cast<float*>(smem + S::kAccOffset), acc_ld(BN)};
  float* s_scale = reinterpret_cast<float*>(smem + S::kBarOffset + 256);
  float* s_shift = s_scale + (BN > kBM ? BN : kBM);  // per-column needs BN entries, per-row kBM

  const int tid = threadIdx.x;
  const int warp = tid >> 5;
  const int n0 = blockIdx.x * BN;
  const int m0 = blockIdx.y * kBM;
  const bool gather = (p.amode != AMODE_TMA);

  // ---- one-time setup -------------------------------------------------------------------
  if (tid == 128) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full_bar[s], gather ? (128 + 1) : 1);
      mbar_init(&empty_bar[s], 1);
    }
    mbar_init(acc_full_bar, 1);
    mbar_init(res_bar, 1);
    fence_mbar_init();
    tma_prefetch_desc(&tmB);
    if (!gather) tma_prefetch_desc(&tmA);
  }
  // folded-BN affine for this tile
  if (p.per_row) {
    if (tid < kBM) {
      int r = m0 + tid;
      s_scale[tid] = (r < p.M_total) ? __ldg(&p.scale[r]) : 0.f;
      s_shift[tid] = (r < p.M_total) ? __ldg(&p.shift[r]) : 0.f;
    }
  } else {
    for (int i = tid; i < BN; i += kThreads) {
      int c = n0 + i;
      s_scale[i] = (c < p.Ncols) ? __ldg(&p.scale[c]) : 0.f;
      s_shift[i] = (c < p.Ncols) ? __ldg(&p.shift[c]) : 0.f;
    }
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();                       // everything above touched only weights / on-chip state

  // ---- warp roles -----------------------------------------------------------------------
  if (warp < 4) {
    // ================= A gather producers (one output row per thread) ====================
    if (gather) {
      const int r = tid;
      const int m = m0 + r;
      const bool row_ok = m < p.M_total;
      int n = 0, to = 0, ho = 0, wo = 0;
      if (row_ok) {
        int q = m;
        wo = q % p.Wo; q /= p.Wo;
        ho = q % p.Ho; q /= p.Ho;
        to = q % p.To; n = q / p.To;
      }
      const int ti0 = to * p.st - p.pt;
      const int hi0 = ho * p.sh - p.ph;
      const uint32_t row_off = static_cast<uint32_t>(r) * 128u;
      const uint32_t swz = static_cast<uint32_t>(r & 7);

      {
        const int wi0 = wo * p.sw - p.pw;
        int dt = 0, dh = 0, dw = 0, cc = 0;
        for (int kb = 0; kb < p.nkb; ++kb) {
          const int s = kb % kStages;
          const uint32_t par = (kb / kStages) & 1;
          mbar_wait(&empty_bar[s], par ^ 1);
          const int ti = ti0 + dt, hi = hi0 + dh, wi = wi0 + dw;
          const bool ok = row_ok && (unsigned)ti < (unsigned)p.T && (unsigned)hi < (unsigned)p.H &&
                          (unsigned)wi < (unsigned)p.W;
          const int c0 = cc * kBK;
          const __half* src = p.x;
          if (ok) src = p.x + ((((size_t)n * p.T + ti) * p.H + hi) * p.W + wi) * (size_t)p.C + c0;
          const uint32_t dst = smem_u32(smem + s * S::kStageBytes) + row_off;
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const bool okj = ok && (c0 + j * 8 < p.C);
            cp_async_16_ca(dst + ((static_cast<uint32_t>(j) ^ swz) << 4), okj ? (src + j * 8) : p.x,
                           okj ? 16u : 0u);
          }
          cp_async_mbar_arrive_noinc(&full_bar[s]);
          // advance (cc fastest, then kw, kh, kt)
          if (++cc == p.cchunks) {
            cc = 0;
            if (++dw == p.kw) {
              dw = 0;
              if (++dh == p.kh) { dh = 0; ++dt; }
            }
          }
        }
      }
    }

    // ================================ epilogue ==========================================
    mbar_wait(acc_full_bar, 0);
    const int r = tid;                      // accumulator row
    const int m = m0 + r;
    const uint32_t swz = static_cast<uint32_t>(r & 7);
    uint8_t* c_stage = smem;                          // BN/64 boxes of [128][64] fp16, 128B swizzle
    uint8_t* r_stage = smem + S::kCTileBytes;

    if (p.epi == EPI_TMA_F16) {
      if (p.residual != nullptr) {
        if (tid == 0) {
          mbar_expect_tx(res_bar, S::kCTileBytes);
#pragma unroll
          for (int b = 0; b < BN / 64; ++b) tma_load_2d(r_stage + b * (kBM * 128), &tmR, res_bar, n0 + b * 64, m0);
        }
        mbar_wait(res_bar, 0);
      }
#pragma unroll 1
      for (int j = 0; j < BN / 32; ++j) {
        uint32_t v[32];
        acc_ld32(acc, r, j * 32, v);
        const int box = j >> 1;
        const int chunk0 = (j & 1) * 4;
        uint8_t* crow = c_stage + box * (kBM * 128) + r * 128;
        const uint8_t* rrow = r_stage + box * (kBM * 128) + r * 128;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const uint32_t coff = ((static_cast<uint32_t>(chunk0 + q)) ^ swz) << 4;
          uint4 rv = make_uint4(0, 0, 0, 0);
          if (p.residual != nullptr) rv = *reinterpret_cast<const uint4*>(rrow + coff);
          const uint32_t rr[4] = {rv.x, rv.y, rv.z, rv.w};
          uint4 mv = make_uint4(0, 0, 0, 0);
          if constexpr (MASK) mv = load_mask8(p, m, n0 + j * 32 + q * 8);
          const uint32_t mm[4] = {mv.x, mv.y, mv.z, mv.w};
          uint32_t out[4];
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int i = q * 8 + e * 2;
            const int ci = j * 32 + i;
            float sc0, sc1, sh0, sh1;
            if (p.per_row) {   // swap-AB GEMMs: affine follows the row; columns past Ncols stay zero
              sc0 = (n0 + ci < p.Ncols) ? s_scale[r] : 0.f;     sh0 = (n0 + ci < p.Ncols) ? s_shift[r] : 0.f;
              sc1 = (n0 + ci + 1 < p.Ncols) ? s_scale[r] : 0.f; sh1 = (n0 + ci + 1 < p.Ncols) ? s_shift[r] : 0.f;
            }
            else { sc0 = s_scale[ci]; sc1 = s_scale[ci + 1]; sh0 = s_shift[ci]; sh1 = s_shift[ci + 1]; }
            float a0 = __uint_as_float(v[i]) * sc0 + sh0;
            float a1 = __uint_as_float(v[i + 1]) * sc1 + sh1;
            const float2 rf = unpack_half2(rr[e]);
            a0 += rf.x; a1 += rf.y;
            if (p.relu) { a0 = fmaxf(a0, 0.f); a1 = fmaxf(a1, 0.f); }
            if constexpr (MASK) apply_mask2(mm[e], a0, a1);
            out[e] = pack_half2(a0, a1);
          }
          *reinterpret_cast<uint4*>(crow + coff) = make_uint4(out[0], out[1], out[2], out[3]);
        }
      }
      fence_proxy_async();                      // st.shared -> visible to the TMA store engine
      asm volatile("bar.sync 1, 128;" ::: "memory");
      if (tid == 0) {
#pragma unroll
        for (int b = 0; b < BN / 64; ++b) {
          if (n0 + b * 64 < p.ldy) tma_store_2d(&tmC, c_stage + b * (kBM * 128), n0 + b * 64, m0);
        }
        tma_store_commit();
        tma_store_wait_read0();
      }
    } else {
      // direct-store epilogue (fp16 or fp32), used for small / oddly shaped outputs (heads, MLPs)
      const bool row_ok = m < p.M_total;
#pragma unroll 1
      for (int j = 0; j < BN / 32; ++j) {
        uint32_t v[32];
        acc_ld32(acc, r, j * 32, v);
        if (row_ok) {
#pragma unroll 4
          for (int i = 0; i < 32; ++i) {
            const int ci = j * 32 + i;
            const int c = n0 + ci;
            if (c >= p.ldy) break;
            float a = 0.f;
            if (c < p.Ncols) {
              const float sc = p.per_row ? s_scale[r] : s_scale[ci];
              const float sh = p.per_row ? s_shift[r] : s_shift[ci];
              a = __uint_as_float(v[i]) * sc + sh;
              if (p.residual != nullptr) a += __half2float(p.residual[(size_t)m * p.ldr + c]);
              if (p.relu) a = fmaxf(a, 0.f);
            }
            if (p.epi == EPI_DIRECT_F32) {
              float* yo = reinterpret_cast<float*>(p.y) + (size_t)m * p.ldy + c;
              if (c < p.Ncols) *yo = p.accumulate ? (*yo + a) : a;
            } else {
              reinterpret_cast<__half*>(p.y)[(size_t)m * p.ldy + c] = __float2half_rn(a);
            }
          }
        }
      }
    }
  } else if (warp == kIgTmaWarp) {
    // ================================ TMA producer ======================================
    // (whole warp with warp-uniform operands; one elected lane issues -- see elect_one())
    const uint32_t tx = S::kBBytes + (gather ? 0 : S::kABytes);
    for (int kb = 0; kb < p.nkb; ++kb) {
      const int s = kb % kStages;
      const uint32_t par = (kb / kStages) & 1;
      mbar_wait(&empty_bar[s], par ^ 1);
      int kcol = kb * kBK;
      if (p.amode == AMODE_GATHER) {          // weight columns are [tap][C]: block (tap, cc) starts at tap*C + cc*64
        const int tap = kb / p.cchunks;
        kcol = tap * p.C + (kb - tap * p.cchunks) * kBK;
      }
      if (elect_one()) {
        mbar_expect_tx(&full_bar[s], tx);
        uint8_t* a_dst = smem + s * S::kStageBytes;
        tma_load_2d(a_dst + S::kABytes, &tmB, &full_bar[s], kcol, n0);
        if (!gather) tma_load_2d(a_dst, &tmA, &full_bar[s], kb * kBK, m0);
      }
      __syncwarp();
    }
  } else {
    // ================================ MMA warpgroup =====================================
    const uint32_t ring = smem_u32(smem);
    for (int kb = 0; kb < p.nkb; ++kb) {
      const int s = kb % kStages;
      const uint32_t par = (kb / kStages) & 1;
      mbar_wait(&full_bar[s], par);
      if (gather) fence_proxy_async();
      const uint32_t a_lo = sw128_desc_lo(ring + s * S::kStageBytes);
      const uint32_t b_lo = sw128_desc_lo(ring + s * S::kStageBytes + S::kABytes);
      wg_mma(acc, 0, BN, wg_sw128(desc_from(kSw128DescHi, a_lo), desc_from(kSw128DescHi, b_lo)), 4, kb != 0);
      wg_sync();
      wg_arrive(&empty_bar[s]);                          // frees the smem slot
      if (kb == p.nkb - 1) wg_arrive(acc_full_bar);     // accumulator complete -> epilogue
    }
  }
}

}  // namespace b2
