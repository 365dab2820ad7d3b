// b2_attention.cu -- fused QK^T -> softmax -> .V kernel for the non-local block
// (reference: nonlocalnet.py:143-166, `_embedded_gaussian`: f = theta^T phi (unscaled), softmax over
// keys, y = f . g).  The Npos x Npos matrix never leaves the SM.  Softmax modes with d <= 256 run the
// single-pass kernel below (register accumulators, lazy rescaling); the two-pass kernel takes d = 512,
// the dot-product and concatenation modes, and is the exact cross-check of the single-pass one.
//
// Two-pass kernel: logits are produced by wgmma into a shared-memory accumulator tile, each of 128 softmax
// threads owns one query row, probabilities go back to shared memory as the fp16 A operand of the second
// MMA, and the output accumulates beside the logits.
//
// Two passes over the keys (exact softmax, no accumulator rescaling):
//   pass 1: S = Q K^T per 64-key block -> running row max m and row sum l (fp32 registers)
//   pass 2: S again -> P = exp(S - m) / l (fp16, smem) -> O += P . V   (O: DVT fp32 columns)
//
// CTA = (128 query rows, sample b, 64-wide slice of the value channels).  9 warps: 0-3 softmax + output
// epilogue, 4-7 MMA warpgroup, 8 TMA producer.  Q, K and P are K-major 128B-swizzled tiles; V stays in its
// natural [positions][dv] layout and enters the second MMA as an MN-major B operand ([64 keys x 128 B],
// SBO = 1 KB between 8-key groups), so theta, phi and g come out of ONE projection GEMM and no transposed copy
// of g is ever made.  The accumulator tile (2 x 64 logit columns + 64 output columns, 98 KB) leaves room for a
// 2-slot operand ring in 227 KB of shared memory, which is what limits the value slice to 64 channels.
#include "b2_host.h"
#include "b2_ptx.cuh"

#include <math.h>
#include <string.h>

namespace b2 {

constexpr int kAttThreads = 288;
constexpr int kAttTmaWarp = 8;
constexpr int kAttBM = 128;        // queries per CTA
constexpr int kAttBKV = 64;        // keys per block
constexpr int kAttSlots = 2;       // smem ring slots
constexpr int kAttSlotBytes = 32768;

struct AttParams {
  int Nq;         // query positions per sample
  int Nk;         // key / value positions per sample (== Nq unless phi and g were sub-sampled)
  int nkb;        // d / 64
  int nkv;        // ceil(Nk / 64)
  int mode;       // 0: softmax over keys (embedded gaussian / gaussian); 1: f / Nk without softmax (dot product);
                  // 2: relu(f) / Nk (concatenation mode: the caller encodes f_ij = a_i + b_j as a rank-2 product, see engine.run_nonlocal)
  float scale;    // mode 1: 1 / Nk
  __half* o;
  int ldo;
};

template <int DVT>
struct AttSmem {
  static constexpr int kRing = kAttSlots * kAttSlotBytes;        // 64 KB
  static constexpr int kPBytes = kAttBM * kAttBKV * 2;           // 16 KB
  static constexpr int kPOff = kRing;
  static constexpr int kBarOff = kRing + 2 * kPBytes;
  static constexpr int kAccCols = 2 * kAttBKV + DVT;             // S[2] then O
  static constexpr int kAccOff = kBarOff + 256;
  static constexpr int kTotal = kAccOff + acc_bytes(kAccCols) + 1024;
  static_assert(DVT * 128 <= kAttSlotBytes, "V tile must fit a ring slot");
  static_assert(kTotal <= 227 * 1024, "shared memory budget");
};

template <int DVT>
__global__ void __launch_bounds__(kAttThreads, 1)
nonlocal_attention_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                          const __grid_constant__ CUtensorMap tmV, const AttParams p) {
  using S = AttSmem<DVT>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_align<1024>(smem_raw);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + S::kBarOff);   // [4]
  uint64_t* empty_bar = full_bar + kAttSlots;                            // [4]
  uint64_t* s_full = empty_bar + kAttSlots;                              // [2]
  uint64_t* s_empty = s_full + 2;                                        // [2]
  uint64_t* p_full = s_empty + 2;                                        // [2]
  uint64_t* p_empty = p_full + 2;                                        // [2]
  uint64_t* o_full = p_empty + 2;                                        // [1]
  const AccTile at{reinterpret_cast<float*>(smem + S::kAccOff), acc_ld(S::kAccCols)};

  const int tid = threadIdx.x, warp = tid >> 5;
  const int q0 = blockIdx.x * kAttBM;            // first query row of this CTA within the sample
  const int b = blockIdx.y;
  const int dv0 = blockIdx.z * DVT;
  const int q_base = b * p.Nq;                   // first global query row of the sample
  const int k_base = b * p.Nk;                   // first global key / value row of the sample
  const bool two_pass = (p.mode == 0);

  if (tid == 128) {
    for (int s = 0; s < kAttSlots; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 1); }
    for (int i = 0; i < 2; ++i) {
      mbar_init(&s_full[i], 1); mbar_init(&s_empty[i], 128);
      mbar_init(&p_full[i], 128); mbar_init(&p_empty[i], 1);
    }
    mbar_init(o_full, 1);
    fence_mbar_init();
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();                       // everything above touched only weights / on-chip state
  constexpr int kColS = 0;                       // 2 x 64 columns
  constexpr int kColO = 2 * kAttBKV;             // DVT columns

  if (warp < 4) {
    // =========================== softmax + epilogue =====================================
    const int r = tid;
    const float L2E = 1.4426950408889634f;
    float m_run = -INFINITY, l_run = 0.f;
    uint32_t v[32];
    int g = 0;
    // ---- pass 1: row max and row sum (softmax modes only) ----
    for (int kvb = 0; two_pass && kvb < p.nkv; ++kvb, ++g) {
      const int buf = g & 1;
      mbar_wait(&s_full[buf], (g >> 1) & 1);
      const int nvalid = p.Nk - kvb * kAttBKV;      // keys >= nvalid belong to the next sample / OOB
      float sv[64];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        acc_ld32(at, r, kColS + buf * 64 + h * 32, v);
#pragma unroll
        for (int i = 0; i < 32; ++i) sv[h * 32 + i] = (h * 32 + i < nvalid) ? __uint_as_float(v[i]) : -INFINITY;
      }
      mbar_arrive(&s_empty[buf]);
      float mx = m_run;
#pragma unroll
      for (int i = 0; i < 64; ++i) mx = fmaxf(mx, sv[i]);
      float sum = 0.f;
      const float mb = mx * L2E;
#pragma unroll
      for (int i = 0; i < 64; ++i) sum += exp2f(sv[i] * L2E - mb);
      l_run = l_run * exp2f((m_run - mx) * L2E) + sum;
      m_run = mx;
    }
    const float inv_l = two_pass ? 1.f / l_run : 0.f;
    const float mb = m_run * L2E;
    // ---- pass 2: probabilities -> smem (A operand of P.V) ----
    const uint32_t swz = static_cast<uint32_t>(r & 7);
    for (int j = 0; j < p.nkv; ++j, ++g) {
      const int buf = g & 1;
      const int pb = j & 1;
      mbar_wait(&s_full[buf], (g >> 1) & 1);
      const int nvalid = p.Nk - j * kAttBKV;
      mbar_wait(&p_empty[pb], ((j >> 1) & 1) ^ 1);
      uint8_t* prow = smem + S::kPOff + pb * S::kPBytes + r * 128;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        acc_ld32(at, r, kColS + buf * 64 + h * 32, v);
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          uint32_t o4[4];
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int i = c * 8 + e * 2;
            const int key = h * 32 + i;
            float p0, p1;
            if (two_pass) {
              p0 = (key < nvalid) ? exp2f(__uint_as_float(v[i]) * L2E - mb) * inv_l : 0.f;
              p1 = (key + 1 < nvalid) ? exp2f(__uint_as_float(v[i + 1]) * L2E - mb) * inv_l : 0.f;
            } else {                                   // dot-product mode: f / N (nonlocalnet.py:203-204)
              p0 = (key < nvalid) ? __uint_as_float(v[i]) * p.scale : 0.f;
              p1 = (key + 1 < nvalid) ? __uint_as_float(v[i + 1]) * p.scale : 0.f;
              if (p.mode == 2) { p0 = fmaxf(p0, 0.f); p1 = fmaxf(p1, 0.f); }   // concatenation mode: ReLU(.) / N (nonlocalnet.py:231-237)
            }
            o4[e] = pack_half2(p0, p1);
          }
          const uint32_t chunk = static_cast<uint32_t>(h * 4 + c);
          *reinterpret_cast<uint4*>(prow + ((chunk ^ swz) << 4)) = make_uint4(o4[0], o4[1], o4[2], o4[3]);
        }
      }
      mbar_arrive(&s_empty[buf]);
      fence_proxy_async();
      mbar_arrive(&p_full[pb]);
    }
    // ---- epilogue: O -> fp16 global ----
    mbar_wait(o_full, 0);
    const bool row_ok = (q0 + r) < p.Nq;
    __half* orow = p.o + (size_t)(q_base + q0 + r) * p.ldo + dv0;
#pragma unroll 1
    for (int jc = 0; jc < DVT / 32; ++jc) {
      acc_ld32(at, r, kColO + jc * 32, v);
      if (row_ok) {
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          uint32_t o4[4];
#pragma unroll
          for (int e = 0; e < 4; ++e)
            o4[e] = pack_half2(__uint_as_float(v[c * 8 + e * 2]), __uint_as_float(v[c * 8 + e * 2 + 1]));
          *reinterpret_cast<uint4*>(orow + jc * 32 + c * 8) = make_uint4(o4[0], o4[1], o4[2], o4[3]);
        }
      }
    }
  } else if (warp == kAttTmaWarp) {
    // =========================== TMA producer ===========================================
    // whole warp, warp-uniform operands; one elected lane issues (see elect_one() in b2_ptx.cuh)
    int it = 0;
    auto load_qk = [&](int kvb) {
      for (int kb = 0; kb < p.nkb; ++kb, ++it) {
        const int s = it % kAttSlots;
        mbar_wait(&empty_bar[s], ((it / kAttSlots) & 1) ^ 1);
        if (elect_one()) {
          mbar_expect_tx(&full_bar[s], kAttBM * 128 + kAttBKV * 128);
          uint8_t* dst = smem + s * kAttSlotBytes;
          tma_load_2d(dst, &tmQ, &full_bar[s], kb * 64, q_base + q0);
          tma_load_2d(dst + kAttBM * 128, &tmK, &full_bar[s], kb * 64, k_base + kvb * kAttBKV);
        }
        __syncwarp();
      }
    };
    for (int kvb = 0; two_pass && kvb < p.nkv; ++kvb) load_qk(kvb);   // pass 1
    load_qk(0);                                                   // pass 2 prologue
    for (int j = 0; j < p.nkv; ++j) {
      if (j + 1 < p.nkv) load_qk(j + 1);
      const int s = it % kAttSlots;
      mbar_wait(&empty_bar[s], ((it / kAttSlots) & 1) ^ 1);
      if (elect_one()) {
        mbar_expect_tx(&full_bar[s], DVT * 128);
#pragma unroll
        for (int blk = 0; blk < DVT / 64; ++blk)      // [64 dv x 64 keys] boxes, 8 KB apart
          tma_load_2d(smem + s * kAttSlotBytes + blk * 8192, &tmV, &full_bar[s], dv0 + blk * 64, k_base + j * kAttBKV);
      }
      __syncwarp();
      ++it;
    }
  } else {
    // =========================== MMA warpgroup ==========================================
    constexpr uint32_t v_hi = kSw128DescHi;                                        // SBO 1024, 128B swizzle
    const uint32_t ring = smem_u32(smem);
    int it = 0;
    int g = 0;
    auto issue_qk = [&]() {       // S[g&1] = Q . K_block^T
      const int buf = g & 1;
      mbar_wait(&s_empty[buf], ((g >> 1) & 1) ^ 1);
      for (int kb = 0; kb < p.nkb; ++kb, ++it) {
        const int s = it % kAttSlots;
        mbar_wait(&full_bar[s], (it / kAttSlots) & 1);
        const uint32_t a_lo = sw128_desc_lo(ring + s * kAttSlotBytes);
        const uint32_t b_lo = sw128_desc_lo(ring + s * kAttSlotBytes + kAttBM * 128);
        wg_mma(at, kColS + buf * 64, kAttBKV, wg_sw128(desc_from(kSw128DescHi, a_lo), desc_from(kSw128DescHi, b_lo)), 4, kb != 0);
        wg_sync();
        wg_arrive(&empty_bar[s]);
        if (kb == p.nkb - 1) wg_arrive(&s_full[buf]);
      }
      ++g;
    };
    for (int kvb = 0; two_pass && kvb < p.nkv; ++kvb) issue_qk();     // pass 1
    issue_qk();                                                   // pass 2 prologue: S for block 0
    for (int j = 0; j < p.nkv; ++j) {
      if (j + 1 < p.nkv) issue_qk();                              // overlap softmax(j) with QK(j+1)
      const int pb = j & 1;
      mbar_wait(&p_full[pb], (j >> 1) & 1);
      const int s = it % kAttSlots;
      mbar_wait(&full_bar[s], (it / kAttSlots) & 1);
      const uint32_t a_lo = sw128_desc_lo(ring + S::kPOff + pb * S::kPBytes);
      // V tile (MN-major B): LBO = 8192 B (next 64-wide dv block); stepping K by 16 keys = 16 rows x 128 B = +2048 B
      const uint32_t b_lo = (((ring + s * kAttSlotBytes) & 0x3FFFFu) >> 4) | ((8192u >> 4) << 16);
      const WgOperands ops{desc_from(kSw128DescHi, a_lo), desc_from(v_hi, b_lo), 2u, 512u, 128u, 512u, 0u};
      wg_mma<1>(at, kColO, DVT, ops, 4, j != 0);
      wg_sync();
      wg_arrive(&empty_bar[s]);
      wg_arrive(&p_empty[pb]);
      if (j == p.nkv - 1) wg_arrive(o_full);
      ++it;
    }
  }
}

// ------------------------------------------------------------------------------------------
// Single-pass variant (softmax modes, d <= 256): Q stays resident in shared memory, keys come in blocks of 128, and
// the running maximum is applied lazily: P = exp(S - m_used) with a *stale* maximum that is only advanced -- and the
// output accumulator rescaled -- when a block's maximum exceeds it by more than 2^8 (P <= 256 stays far inside fp16, O
// accumulates in fp32, the final O / l is exact in the same sense as the two-pass kernel).  Half the tensor work of
// the two-pass kernel and a quarter of its L2 traffic.
//
// CTA = (128 query rows, sample b, DVT-wide slice of the value channels), 9 warps: two consumer warpgroups of 64 query
// rows each and a TMA producer warp.  A consumer warpgroup keeps its logits S (64 x 128 fp32) and its output O (64 x DVT
// fp32) in registers: S = Q K^T is one m64n128 wgmma per K step (Q and K from shared memory), the softmax works on the
// accumulator fragment (a row lives in the four threads of a quad: max and sum by two shuffles), and P goes back to the
// tensor core from registers as the A operand of O += P . V -- the accumulator fragment of 16 columns is exactly the A
// fragment of one K step -- with V consumed in its natural layout as an MN-major B operand.
// ------------------------------------------------------------------------------------------
constexpr int kOnBKV = 128;          // keys per block
constexpr int kOnSlots = 4;          // 32 KB ring slots: K [128 keys x 128 d] (two 64-wide chunks) or V [64 keys x DVT]
constexpr float kOnLazyLog2 = 8.0f;  // rescale only when the block maximum exceeds the stale one by > 2^8
constexpr int kOnThreads = 288;      // warps 0-7: two consumer warpgroups, warp 8: TMA producer
constexpr int kOnProdWarp = 8;

template <int DVT>
struct OnSmem {
  static constexpr int kQBytes = 4 * kAttBM * 128;               // up to four 64-wide d chunks: 64 KB
  static constexpr int kRingOff = kQBytes;
  static constexpr int kBarOff = kRingOff + kOnSlots * kAttSlotBytes;
  static constexpr int kTotal = kBarOff + 256 + 1024;
  static_assert(DVT == 64 || DVT == 128, "O of a 64-row warpgroup slice: DVT / 2 registers per thread");
  static_assert(kTotal <= 227 * 1024, "shared memory budget");
};

template <int DVT>
__global__ void __launch_bounds__(kOnThreads, 1)
nonlocal_attention_online_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                                 const __grid_constant__ CUtensorMap tmV, const AttParams p) {
  using S = OnSmem<DVT>;
  constexpr int NB = DVT / 64;                   // 64-column blocks of O
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_align<1024>(smem_raw);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + S::kBarOff);   // [kOnSlots]
  uint64_t* empty_bar = full_bar + kOnSlots;                             // [kOnSlots] one arrival per consumer warp
  uint64_t* q_full = empty_bar + kOnSlots;                               // [1]

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int q0 = blockIdx.x * kAttBM;
  const int b = blockIdx.y;
  const int dv0 = blockIdx.z * DVT;
  const int q_base = b * p.Nq, k_base = b * p.Nk;
  const int nblk = (p.Nk + kOnBKV - 1) / kOnBKV;
  const int kslots = (p.nkb + 1) / 2;            // ring slots per key block (two d chunks per slot)

  if (tid == 0) {
    for (int s = 0; s < kOnSlots; ++s) { mbar_init(&full_bar[s], 1); mbar_init(&empty_bar[s], 8); }
    mbar_init(q_full, 1);
    fence_mbar_init();
    tma_prefetch_desc(&tmQ); tma_prefetch_desc(&tmK); tma_prefetch_desc(&tmV);
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();

  if (warp == kOnProdWarp) {
    // =========================== TMA producer ===========================================
    // ring order = consumption order: K(0), V(0), K(1), V(1), ...
    if (elect_one()) {
      mbar_expect_tx(q_full, static_cast<uint32_t>(p.nkb * kAttBM * 128));
      for (int kb = 0; kb < p.nkb; ++kb) tma_load_2d(smem + kb * (kAttBM * 128), &tmQ, q_full, kb * 64, q_base + q0);
    }
    __syncwarp();
    int it = 0;
    for (int j = 0; j < nblk; ++j) {
      for (int ks = 0; ks < kslots; ++ks, ++it) {
        const int s = it % kOnSlots;
        const int nch = min(2, p.nkb - ks * 2);
        mbar_wait(&empty_bar[s], ((it / kOnSlots) & 1) ^ 1);
        if (elect_one()) {
          mbar_expect_tx(&full_bar[s], static_cast<uint32_t>(nch * kOnBKV * 128));
          for (int c = 0; c < nch; ++c)
            tma_load_2d(smem + S::kRingOff + s * kAttSlotBytes + c * (kOnBKV * 128), &tmK, &full_bar[s], (ks * 2 + c) * 64,
                        k_base + j * kOnBKV);
        }
        __syncwarp();
      }
      for (int h = 0; h < 2; ++h, ++it) {           // V rows of the two 64-key halves
        const int s = it % kOnSlots;
        mbar_wait(&empty_bar[s], ((it / kOnSlots) & 1) ^ 1);
        if (elect_one()) {
          mbar_expect_tx(&full_bar[s], DVT * 128);
#pragma unroll
          for (int blk = 0; blk < NB; ++blk)
            tma_load_2d(smem + S::kRingOff + s * kAttSlotBytes + blk * 8192, &tmV, &full_bar[s], dv0 + blk * 64,
                        k_base + j * kOnBKV + h * 64);
        }
        __syncwarp();
      }
    }
  } else if (warp < kOnProdWarp) {
    // =========================== consumer warpgroups =====================================
    // thread t of warpgroup wg holds rows wg*64 + 16*(t/32) + (t%32)/4 (+ 8) and column pairs 8 i + 2 (t % 4)
    const int wg = warp >> 2;
    const int qc = lane & 3;
    const uint32_t base = smem_u32(smem), ring = base + S::kRingOff;
    const float L2E = 1.4426950408889634f;
    float o[NB][32];
#pragma unroll
    for (int nb = 0; nb < NB; ++nb)
#pragma unroll
      for (int i = 0; i < 32; ++i) o[nb][i] = 0.f;
    float m_used[2] = {-INFINITY, -INFINITY}, l_part[2] = {0.f, 0.f};
    auto release = [&](int s) {                    // this warp is done reading slot s
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[s]);
    };
    mbar_wait(q_full, 0);
    int it = 0;
    for (int j = 0; j < nblk; ++j) {
      // ---- S = Q . K_j^T (64 x 128 per warpgroup) ----
      float sacc[64];
#pragma unroll
      for (int i = 0; i < 64; ++i) sacc[i] = 0.f;
      for (int ks = 0; ks < kslots; ++ks) mbar_wait(&full_bar[(it + ks) % kOnSlots], ((it + ks) / kOnSlots) & 1);
      wgmma_fence();
      for (int ks = 0; ks < kslots; ++ks) {
        const int s = (it + ks) % kOnSlots;
        const int nch = min(2, p.nkb - ks * 2);
        for (int c = 0; c < nch; ++c) {
          const int kb = ks * 2 + c;
          const uint32_t a_lo = sw128_desc_lo(base + kb * (kAttBM * 128) + wg * (64 * 128));
          const uint32_t b_lo = sw128_desc_lo(ring + s * kAttSlotBytes + c * (kOnBKV * 128));
#pragma unroll
          for (int k = 0; k < 4; ++k)
            wgmma_n128_ss(sacc, desc_from(kSw128DescHi, a_lo + 2 * k), desc_from(kSw128DescHi, b_lo + 2 * k));
        }
      }
      wgmma_commit();
      wgmma_wait0();
      for (int ks = 0; ks < kslots; ++ks) release((it + ks) % kOnSlots);
      it += kslots;

      // ---- lazy-max softmax on the fragment ----
      const int nvalid = p.Nk - j * kOnBKV;      // keys >= nvalid belong to the next sample / are out of range
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int i = 0; i < 16; ++i)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const bool ok = 8 * i + 2 * qc + e < nvalid;
#pragma unroll
          for (int r = 0; r < 2; ++r) {
            float& v = sacc[4 * i + 2 * r + e];
            v = ok ? v : -INFINITY;
            mx[r] = fmaxf(mx[r], v);
          }
        }
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
        const float mb = mx[r] * L2E;
        if (mb > m_used[r] + kOnLazyLog2) {     // always true for the first block (m_used = -inf); uniform over the quad
          const float f = exp2f(m_used[r] - mb);
          m_used[r] = mb;
          l_part[r] *= f;
#pragma unroll
          for (int nb = 0; nb < NB; ++nb)
#pragma unroll
            for (int i = 0; i < 8; ++i) { o[nb][4 * i + 2 * r] *= f; o[nb][4 * i + 2 * r + 1] *= f; }
        }
      }
      uint32_t pa[8][4];                          // P as the A fragments of the eight 16-key steps
#pragma unroll
      for (int kk = 0; kk < 8; ++kk)
#pragma unroll
        for (int g = 0; g < 4; ++g) {
          const int r = g & 1;
          const float p0 = exp2f(fmaf(sacc[8 * kk + 2 * g], L2E, -m_used[r]));
          const float p1 = exp2f(fmaf(sacc[8 * kk + 2 * g + 1], L2E, -m_used[r]));
          l_part[r] += p0 + p1;
          pa[kk][g] = pack_half2(p0, p1);
        }

      // ---- O += P . V_j (two 64-key halves, one ring slot each) ----
#pragma unroll
      for (int h = 0; h < 2; ++h, ++it) {
        const int s = it % kOnSlots;
        mbar_wait(&full_bar[s], (it / kOnSlots) & 1);
        wgmma_fence();
        // V tile (MN-major B): LBO = 8192 B (next 64-wide dv block); 16 keys = 16 rows x 128 B = +2048 B
        const uint32_t b_lo = (((ring + s * kAttSlotBytes) & 0x3FFFFu) >> 4) | ((8192u >> 4) << 16);
#pragma unroll
        for (int k4 = 0; k4 < 4; ++k4)
#pragma unroll
          for (int nb = 0; nb < NB; ++nb)
            wgmma_n64_rs<1>(o[nb], pa[h * 4 + k4], desc_from(kSw128DescHi, b_lo + k4 * 128 + nb * 512));
        wgmma_commit();
        wgmma_wait0();
        release(s);
      }
    }
    // ---- epilogue: O / l -> fp16 global ----
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      float l = l_part[r];
      l += __shfl_xor_sync(0xffffffffu, l, 1);
      l += __shfl_xor_sync(0xffffffffu, l, 2);
      const float inv_l = 1.f / l;
      const int row = q0 + wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * r;
      if (row < p.Nq) {
        __half* orow = p.o + (size_t)(q_base + row) * p.ldo + dv0;
#pragma unroll
        for (int nb = 0; nb < NB; ++nb)
#pragma unroll
          for (int i = 0; i < 8; ++i)
            *reinterpret_cast<uint32_t*>(orow + nb * 64 + 8 * i + 2 * qc) =
                pack_half2(o[nb][4 * i + 2 * r] * inv_l, o[nb][4 * i + 2 * r + 1] * inv_l);
      }
    }
  }
}

template <int DVT>
static int launch_attention(const void* q, int ldq, const void* k, int ldk, const void* v, int ldv, void* o, int ldo,
                            int B, int Nq, int Nk, int d, int dv, int mode, cudaStream_t stream) {
  using S = AttSmem<DVT>;
  B2_OPT_IN_SMEM(nonlocal_attention_kernel<DVT>, S::kTotal);
  CUtensorMap tmQ, tmK, tmV;
  int rc;
  const uint64_t qrows = (uint64_t)B * Nq, krows = (uint64_t)B * Nk;
  if ((rc = make_tmap_2d_f16(&tmQ, q, (uint64_t)d, qrows, (uint64_t)ldq, 64, kAttBM, true)) != B2_OK) return rc;
  if ((rc = make_tmap_2d_f16(&tmK, k, (uint64_t)d, krows, (uint64_t)ldk, 64, kAttBKV, true)) != B2_OK) return rc;
  if ((rc = make_tmap_2d_f16(&tmV, v, (uint64_t)dv, krows, (uint64_t)ldv, 64, kAttBKV, true)) != B2_OK) return rc;
  AttParams p;
  p.Nq = Nq; p.Nk = Nk; p.nkb = d / 64; p.nkv = (Nk + kAttBKV - 1) / kAttBKV;
  p.mode = mode; p.scale = 1.0f / (float)Nk;
  p.o = reinterpret_cast<__half*>(o); p.ldo = ldo;
  dim3 grid((Nq + kAttBM - 1) / kAttBM, B, dv / DVT);
  B2_CHECK_CUDA(launch_pdl(nonlocal_attention_kernel<DVT>, grid, dim3(kAttThreads), S::kTotal, stream, tmQ, tmK, tmV, p));
  B2_CHECK_LAUNCH("nonlocal_attention_kernel");
  return B2_OK;
}

template <int DVT>
static int launch_attention_online(const void* q, int ldq, const void* k, int ldk, const void* v, int ldv, void* o, int ldo,
                                   int B, int Nq, int Nk, int d, int dv, cudaStream_t stream) {
  using S = OnSmem<DVT>;
  B2_OPT_IN_SMEM(nonlocal_attention_online_kernel<DVT>, S::kTotal);
  CUtensorMap tmQ, tmK, tmV;
  int rc;
  const uint64_t qrows = (uint64_t)B * Nq, krows = (uint64_t)B * Nk;
  if ((rc = make_tmap_2d_f16(&tmQ, q, (uint64_t)d, qrows, (uint64_t)ldq, 64, kAttBM, true)) != B2_OK) return rc;
  if ((rc = make_tmap_2d_f16(&tmK, k, (uint64_t)d, krows, (uint64_t)ldk, 64, kOnBKV, true)) != B2_OK) return rc;
  if ((rc = make_tmap_2d_f16(&tmV, v, (uint64_t)dv, krows, (uint64_t)ldv, 64, 64, true)) != B2_OK) return rc;
  AttParams p;
  p.Nq = Nq; p.Nk = Nk; p.nkb = d / 64; p.nkv = (Nk + kOnBKV - 1) / kOnBKV;
  p.mode = 0; p.scale = 0.f;
  p.o = reinterpret_cast<__half*>(o); p.ldo = ldo;
  dim3 grid((Nq + kAttBM - 1) / kAttBM, B, dv / DVT);
  B2_CHECK_CUDA(launch_pdl(nonlocal_attention_online_kernel<DVT>, grid, dim3(kOnThreads), S::kTotal, stream, tmQ, tmK, tmV, p));
  B2_CHECK_LAUNCH("nonlocal_attention_online_kernel");
  return B2_OK;
}

}  // namespace b2

using namespace b2;

static int g_att_algo = 0;   // debug: 1 = always the two-pass kernel
extern "C" int b2_debug_set_attention_algo(int algo) { g_att_algo = algo; return B2_OK; }

extern "C" int b2_nonlocal_attention(const void* q, int ldq, const void* k, int ldk, const void* v, int ldv, void* o,
                                     int ldo, int B, int Nq, int Nk, int d, int dv, int mode, void* stream) {
  B2_CHECK_ARG(q && k && v && o, "null pointer");
  B2_CHECK_ARG(B > 0 && Nq > 0 && Nk > 0 && d > 0 && dv > 0, "non-positive dimension");
  B2_CHECK_ARG(mode >= 0 && mode <= 2, "unknown attention mode %d", mode);
  B2_CHECK_ARG(ldq % 8 == 0 && ldk % 8 == 0 && ldv % 8 == 0 && ldo % 8 == 0, "pitches must be multiples of 8");
  B2_CHECK_ARG(ldq >= d && ldk >= d && ldo >= dv && ldv >= dv, "pitch smaller than extent");
  if (d % 64 != 0 || dv % 64 != 0)
    return set_error(B2_ERR_UNSUPPORTED, "non-local attention needs d and dv multiples of 64 (got %d, %d)", d, dv);
  int rc;
  if ((rc = require_sm90()) != B2_OK) return rc;
  cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (mode == 0 && d <= 256 && g_att_algo != 1) {              // single-pass kernel (Q resident, lazy rescaling)
    if (dv % 128 == 0) return launch_attention_online<128>(q, ldq, k, ldk, v, ldv, o, ldo, B, Nq, Nk, d, dv, st);
    return launch_attention_online<64>(q, ldq, k, ldk, v, ldv, o, ldo, B, Nq, Nk, d, dv, st);
  }
  return launch_attention<64>(q, ldq, k, ldk, v, ldv, o, ldo, B, Nq, Nk, d, dv, mode, st);
}
