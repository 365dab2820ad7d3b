// b2_densem.cuh -- dense-M implicit GEMM with split-K across a thread-block cluster, for the SMALL-M regime.
//
// The slab kernel (b2_slabconv.cuh) tiles one (n, t) plane at a time: a 7x7 plane fills 49 of the 128 rows of an MMA tile and a
// 4x4 plane 16 of them, and a layer with M = N*T*H*W of a few thousand positions yields far fewer work items than the 132 SMs --
// the late stages of every video net here (resnet3d50 layer3/4, all of R(2+1)D-34 beyond layer2, everything at 2 clips per GPU).
// Those layers are bound by streaming their WEIGHTS (2.6 - 10.6 MB per launch) through few SMs.  This kernel:
//   * packs output positions densely: tile row r is output pixel m0 + r whatever plane it lies in (im2col gather by cp.async,
//     one row per producer thread, zero fill for padding taps; the activation tensor of such a layer is L2-resident);
//   * splits the K loop (taps x 64-channel blocks) over the S CTAs of a thread-block CLUSTER (S <= 8): every CTA streams 1/S of
//     the weights, so tiles x S >= #SMs work units exist even for a 4-tile layer;
//   * reduces the S partial accumulators through distributed shared memory, reduce-scatter style: CTA r owns the column slice
//     [r*bn/S, (r+1)*bn/S) of the tile; every peer writes its partial of that slice into r's shared memory
//     (st.shared::cluster), one cluster barrier later r adds them to its own partial, applies BN / residual / ReLU and
//     stores the slice.  No global workspace, no second pass, no atomics; the epilogue work is spread over all S CTAs.
// Operands as everywhere else: fp16, K-major SWIZZLE_128B tiles, fp32 accumulation in a shared-memory AccTile, one MMA warpgroup.
#pragma once

#include "b2_igemm.cuh"

namespace b2 {

constexpr int kDmThreads = 288;    // warps 0-3: A gather producers, then epilogue; warps 4-7: MMA warpgroup; warp 8: TMA producer
constexpr int kDmTmaWarp = 8;
constexpr int kDmMaxStages = 6;

struct DensemParams {
  IgemmParams g;           // geometry / epilogue description shared with the gather kernel (epi is ignored: direct stores)
  int bn;                  // N per tile (multiple of 32, <= 128); bn / ksplit is a multiple of 32
  int bbytes;              // weight stage bytes: bn * 128
  int stage_bytes;         // 16 KB (A) + bbytes, multiple of 1024
  int acc_off;             // byte offset of the AccTile (bn columns) behind the ring and the barriers
  int ksplit;              // cluster size along K (gridDim.z)
  int kb_per;              // K blocks per CTA (the last CTA may get fewer)
  int nstages;             // operand ring depth (as many as fit: the loop is latency-bound, bytes in flight are what count)
};

__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {      // every thread of every CTA of the cluster
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ uint32_t map_to_cta(uint32_t smem_addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(smem_addr), "r"(rank));
  return r;
}
__device__ __forceinline__ void st_cluster_v4(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.shared::cluster.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}

__global__ void __launch_bounds__(kDmThreads, 1)
densem_kernel(const __grid_constant__ CUtensorMap tmA,   // activations as [M][C] (AMODE_TMA: 1x1x1 stride-1 layers)
              const __grid_constant__ CUtensorMap tmB,   // weights [Ncols][Ktot], box (64, bn)
              const DensemParams dp) {
  const IgemmParams& p = dp.g;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_align<1024>(smem_raw);
  const int kDmStages = dp.nstages;
  const int ring_bytes = kDmStages * dp.stage_bytes;
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + ring_bytes);
  uint64_t* empty_bar = full_bar + kDmMaxStages;
  uint64_t* acc_full_bar = empty_bar + kDmMaxStages;
  const AccTile at{reinterpret_cast<float*>(smem + dp.acc_off), acc_ld(dp.bn)};

  const int tid = threadIdx.x, warp = tid >> 5;
  const int bn = dp.bn;
  const int n0 = blockIdx.x * bn;
  const int m0 = blockIdx.y * kBM;
  const uint32_t rank = dp.ksplit > 1 ? cluster_ctarank() : 0u;          // == blockIdx.z: cluster dims are (1, 1, ksplit)
  const int kb0 = static_cast<int>(rank) * dp.kb_per;
  const int kb1 = min(p.nkb, kb0 + dp.kb_per);
  const int nkb_here = max(0, kb1 - kb0);
  const bool gather = (p.amode != AMODE_TMA);

  if (tid == 128) {
    for (int s = 0; s < kDmStages; ++s) { mbar_init(&full_bar[s], gather ? (128 + 1) : 1); mbar_init(&empty_bar[s], 1); }
    mbar_init(acc_full_bar, 1);
    fence_mbar_init();
    tma_prefetch_desc(&tmB);
    if (!gather) tma_prefetch_desc(&tmA);
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();

  if (warp < 4) {
    // ================= A gather producers (one output row per thread) ====================
    if (gather && nkb_here > 0) {
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
      const int ti0 = to * p.st - p.pt, hi0 = ho * p.sh - p.ph, wi0 = wo * p.sw - p.pw;
      const uint32_t row_off = static_cast<uint32_t>(r) * 128u;
      const uint32_t swz = static_cast<uint32_t>(r & 7);
      // K block kb = (tap, cc) with cc fastest; tap = (dt * kh + dh) * kw + dw
      int tap = kb0 / p.cchunks;
      int cc = kb0 - tap * p.cchunks;
      int dw = tap % p.kw; int t2 = tap / p.kw;
      int dh = t2 % p.kh; int dt = t2 / p.kh;
      for (int i = 0; i < nkb_here; ++i) {
        const int s = i % kDmStages;
        mbar_wait(&empty_bar[s], ((i / kDmStages) & 1) ^ 1);
        const int ti = ti0 + dt, hi = hi0 + dh, wi = wi0 + dw;
        const bool ok = row_ok && (unsigned)ti < (unsigned)p.T && (unsigned)hi < (unsigned)p.H && (unsigned)wi < (unsigned)p.W;
        const int c0 = cc * kBK;
        const __half* src = p.x;
        if (ok) src = p.x + ((((size_t)n * p.T + ti) * p.H + hi) * p.W + wi) * (size_t)p.C + c0;
        const uint32_t dst = smem_u32(smem + s * dp.stage_bytes) + row_off;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const bool okj = ok && (c0 + j * 8 < p.C);
          cp_async_16_cg(dst + ((static_cast<uint32_t>(j) ^ swz) << 4), okj ? (src + j * 8) : p.x, okj ? 16u : 0u);
        }
        cp_async_mbar_arrive_noinc(&full_bar[s]);
        if (++cc == p.cchunks) {
          cc = 0;
          if (++dw == p.kw) { dw = 0; if (++dh == p.kh) { dh = 0; ++dt; } }
        }
      }
    }
  } else if (warp == kDmTmaWarp) {
    // ================================ TMA producer ======================================
    const uint32_t tx = static_cast<uint32_t>(dp.bbytes) + (gather ? 0u : static_cast<uint32_t>(kBM * kBK * 2));
    for (int i = 0; i < nkb_here; ++i) {
      const int kb = kb0 + i;
      const int s = i % kDmStages;
      mbar_wait(&empty_bar[s], ((i / kDmStages) & 1) ^ 1);
      int kcol = kb * kBK;
      if (gather) {                     // weight columns are [tap][C]: block (tap, cc) starts at tap*C + cc*64
        const int tap = kb / p.cchunks;
        kcol = tap * p.C + (kb - tap * p.cchunks) * kBK;
      }
      if (elect_one()) {
        mbar_expect_tx(&full_bar[s], tx);
        uint8_t* a_dst = smem + s * dp.stage_bytes;
        tma_load_2d(a_dst + kBM * kBK * 2, &tmB, &full_bar[s], kcol, n0);
        if (!gather) tma_load_2d(a_dst, &tmA, &full_bar[s], kb * kBK, m0);
      }
      __syncwarp();
    }
  } else {
    // ================================ MMA warpgroup =====================================
    const uint32_t ring = smem_u32(smem);
    for (int i = 0; i < nkb_here; ++i) {
      const int s = i % kDmStages;
      mbar_wait(&full_bar[s], (i / kDmStages) & 1);
      if (gather) fence_proxy_async();
      const uint32_t a_lo = sw128_desc_lo(ring + s * dp.stage_bytes);
      const uint32_t b_lo = sw128_desc_lo(ring + s * dp.stage_bytes + kBM * kBK * 2);
      wg_mma(at, 0, bn, wg_sw128(desc_from(kSw128DescHi, a_lo), desc_from(kSw128DescHi, b_lo)), 4, i != 0);
      wg_sync();
      wg_arrive(&empty_bar[s]);
      if (i == nkb_here - 1) wg_arrive(acc_full_bar);
    }
    if (nkb_here == 0) wg_arrive(acc_full_bar);      // (cannot happen: the host gives every CTA >= 1 block)
  }

  // ---- everyone: this CTA's partial accumulator is complete (its operand ring is no longer read) ----
  mbar_wait(acc_full_bar, 0);
  const int S = dp.ksplit;
  const int slice = bn / S;                         // columns this CTA finalises (multiple of 32)
  float* stage = reinterpret_cast<float*>(smem);    // [S - 1][128][slice] fp32 partials from the peers, aliasing the ring
  if (S > 1) {
    cluster_sync_all();                             // B0: every CTA of the cluster is done with its ring -> safe to overwrite
    if (warp < 4) {
      for (int peer = 0; peer < S; ++peer) {
        if (peer == static_cast<int>(rank)) continue;
        const int slot = static_cast<int>(rank) < peer ? static_cast<int>(rank) : static_cast<int>(rank) - 1;   // my slot in the peer's staging area
        // staging layout [slot][16-byte column group][row]: the 32 lanes of a warp (consecutive rows) write 512 contiguous bytes
        const uint32_t remote = map_to_cta(smem_u32(stage + static_cast<size_t>(slot) * kBM * slice) + static_cast<uint32_t>(tid) * 16u,
                                           static_cast<uint32_t>(peer));
        for (int c = 0; c < slice; c += 32) {
          uint32_t v[32];
          acc_ld32(at, tid, peer * slice + c, v);
#pragma unroll
          for (int q = 0; q < 8; ++q)
            st_cluster_v4(remote + static_cast<uint32_t>(c / 4 + q) * (kBM * 16u), v[q * 4], v[q * 4 + 1], v[q * 4 + 2], v[q * 4 + 3]);
        }
      }
    }
    cluster_sync_all();                             // B1: all partials have landed
  }

  if (warp < 4) {
    // ================================ epilogue: my column slice =========================
    const int r = tid;
    const int m = m0 + r;
    const bool row_ok = m < p.M_total;
    const int col0 = static_cast<int>(rank) * slice;              // first tile column of my slice
    for (int c = 0; c < slice; c += 32) {
      uint32_t v[32];
      acc_ld32(at, r, col0 + c, v);
      float acc[32];
#pragma unroll
      for (int i = 0; i < 32; ++i) acc[i] = __uint_as_float(v[i]);
      for (int sl = 0; sl < S - 1; ++sl) {
        const float4* src = reinterpret_cast<const float4*>(stage + static_cast<size_t>(sl) * kBM * slice) + (c / 4) * kBM + r;
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          const float4 t = src[q * kBM];
          acc[q * 4] += t.x; acc[q * 4 + 1] += t.y; acc[q * 4 + 2] += t.z; acc[q * 4 + 3] += t.w;
        }
      }
      if (!row_ok) continue;
      const int cg0 = n0 + col0 + c;                              // global output column of acc[0]
      if (p.epi == EPI_DIRECT_F32) {
        float* yo = reinterpret_cast<float*>(p.y) + (size_t)m * p.ldy;
        for (int i = 0; i < 32; ++i) {
          const int cg = cg0 + i;
          if (cg >= p.Ncols) break;
          float a = acc[i] * __ldg(&p.scale[p.per_row ? m : cg]) + __ldg(&p.shift[p.per_row ? m : cg]);
          if (p.residual != nullptr) a += __half2float(p.residual[(size_t)m * p.ldr + cg]);
          if (p.relu) a = fmaxf(a, 0.f);
          yo[cg] = p.accumulate ? (yo[cg] + a) : a;
        }
      } else {
        __half* yrow = reinterpret_cast<__half*>(p.y) + (size_t)m * p.ldy;
        const __half* rrow = p.residual ? p.residual + (size_t)m * p.ldr : nullptr;
#pragma unroll
        for (int c8 = 0; c8 < 4; ++c8) {
          const int cg = cg0 + c8 * 8;
          if (cg >= p.ldy) break;                                   // columns [Ncols, ldy) are written as zero
          uint32_t rr[4] = {0u, 0u, 0u, 0u};
          if (rrow != nullptr && cg < p.ldr) {
            const uint4 rv = __ldg(reinterpret_cast<const uint4*>(rrow + cg));
            rr[0] = rv.x; rr[1] = rv.y; rr[2] = rv.z; rr[3] = rv.w;
          }
          uint32_t o[4];
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int i = c8 * 8 + e * 2;
            const int ca = cg + e * 2;
            float a0 = 0.f, a1 = 0.f;
            const float2 rf = unpack_half2(rr[e]);
            if (ca < p.Ncols) {
              a0 = acc[i] * __ldg(&p.scale[ca]) + __ldg(&p.shift[ca]) + rf.x;
              if (p.relu) a0 = fmaxf(a0, 0.f);
            }
            if (ca + 1 < p.Ncols) {
              a1 = acc[i + 1] * __ldg(&p.scale[ca + 1]) + __ldg(&p.shift[ca + 1]) + rf.y;
              if (p.relu) a1 = fmaxf(a1, 0.f);
            }
            o[e] = pack_half2(a0, a1);
          }
          *reinterpret_cast<uint4*>(yrow + cg) = make_uint4(o[0], o[1], o[2], o[3]);
        }
      }
    }
  }

}

}  // namespace b2
