// b2_slab_t128.cuh -- the slab convolution (b2_slabconv.cuh) for 128-wide and 64-wide output tiles as the transposed product.
//
// The slab kernel's 128-wide N tile runs one 128-position M tile per work item (kSlabAccCols = 192 leaves room for no second), so
// each 16 KB weight stage (one tap x one 64-channel chunk x 128 outputs) serves 128 positions and is fetched from L2 again for the
// next item: layers 2-3 of the 3-D ResNets stream ~5 bytes of filter per MAC column from L2.  Here (BN = 128) each consumer warpgroup
// owns 64 of the tile's 128 output channels -- its half of the weight stage (8 KB, 1024-aligned) is the m64 A operand -- and the B
// operand is a whole work item of NP padded positions taken straight from the slab rows (K-major SWIZZLE_128B, taps are row shifts
// of the start address as in the slab kernel): one m64 n(NP) k16 per K step.  An item is `rows` whole output rows of one (n, t)
// plane (SlabParams::qitem = rows * PW positions, NP = qitem rounded up to a compiled width), so a weight stage serves up to 256
// positions, and per tensor cycle the MMAs read 2 x (2 KB + NP x 32 B) / NP bytes of shared memory (80 at NP = 256) instead of 96.
// Every compiled column is issued: the positions past qitem fall on rows of the slab that the host sized for NP positions from
// every item start, and their columns are dropped by the epilogue.
//
// BN = 64 (at most 64 output channels): the two warpgroups cannot split channels, so they split positions.  An item is 2 NP
// consecutive padded positions of one plane (qitem = 2 NP, as the slab kernel's items are MT * 128 of them); warpgroup wg owns
// positions [wg NP, wg NP + NP), takes the whole 8 KB weight stage as its A operand and the slab rows from its own first position as
// B.  The slab kernel's 64-wide tile (slabconv_kernel<64, 2>) does the same with NP = 128, but stores its fp32 fragments into an
// accumulator tile that caps the item at 256 positions; with the fp16 staging tile below an item is 336 positions (NP = 168), so
// each weight stage serves 1.3x the positions.  Every compiled column is issued here too: the slab is sized for 2 NP positions
// from every item start, also where the second warpgroup's half lies partly or wholly past the plane.
//
// The NP / 2 fp32 accumulators per consumer thread (84 - 128) need more than the 168 registers twelve warps get: setmaxnreg moves
// the producer / epilogue warpgroup down to 56 and the consumers up to 224.  An fp32 accumulator tile would not fit next to the
// slab and weight rings, so the consumers apply the folded-BN affine and the ReLU to their fragments themselves (the same fp32
// expression and single rounding as the slab kernel's epilogue) and store fp16 with stmatrix .trans into a [position][channel]
// staging tile; the three epilogue warps copy its valid rows to y.  Every output element keeps the slab kernel's accumulation order
// (temporal tap, channel chunk, phase, in-plane tap, K step), so the outputs are bitwise those of the slab kernel.
//
// Scope (slab_t_geometry in b2_conv_api.cu): 3x3 or 3x3x3 filters with in-plane padding 0 ("valid") or 1 ("same") and temporal
// padding "same" -- slab_geometry's tap table, whose row offsets are centred on the window -- spatial stride 1 or 2 (the phase
// sub-images of the slab producer, unchanged), C % 64 == 0, K % 128 == 0 (BN = 128) or K <= 64 (BN = 64), rows that fit one TMA
// box; no residual, per-sample affine or upsampling.
#pragma once

#include "b2_slabconv.cuh"

namespace b2 {

// weight stage: BN output channels x one 64-channel chunk of one tap.  Staging tile row: one position's BN fp16 channels.
template <int BN> constexpr int kSlabTWBytes = BN * 128;
template <int BN> constexpr int kSlabTRowBytes = BN * 2;
// staging tile: NP positions of 256 B (BN = 128) or 2 NP positions of 128 B (BN = 64)
template <int NP> constexpr int kSlabTStageBytes = NP * 256;

// Work item = (N tile, position group of a plane, plane) in the slab kernel's order; SlabParams::MT = 1, so slab_item's q0 is the
// group's index times 128
template <int BN>
__device__ __forceinline__ SlabItem slab_t_item(const SlabParams& p, int item) {
  SlabItem w = slab_item(p, item, BN);
  w.q0 = (w.q0 >> 7) * p.qitem;
  const int lo = w.q0 - p.reach;
  w.r_lo = (lo >= 0) ? fdiv(lo, p.fd_PW) : -fdiv(-lo + p.PW - 1, p.fd_PW);
  return w;
}

// Staging tile: row v (position) holds BN / 8 chunks of 8 channels, chunk c at (c ^ (v & 7)) * 16, so that the 8 rows of one
// stmatrix matrix (one chunk, 8 consecutive positions) fall in 8 different bank groups
template <int BN, int NP>
__device__ __forceinline__ void slab_t_consumer(const SlabParams& p, uint32_t slab0, uint32_t w0s, uint32_t stage,
                                                const float* s_scale, const float* s_shift, uint64_t* slab_full,
                                                uint64_t* slab_empty, uint64_t* w_full, uint64_t* w_empty, uint64_t* acc_full,
                                                uint64_t* acc_empty) {
  static_assert(BN == 128 || BN == 64, "output tile width");
  static_assert(NP % 8 == 0, "staging rows of one warpgroup start on a swizzle period");
  constexpr int kRow = kSlabTRowBytes<BN>;
  float acc[NP / 2];
  const int wg = warp_uniform(threadIdx.x >> 7);
  const int lane = threadIdx.x & 31, wq = (threadIdx.x >> 5) & 3;
  const bool lead = lane == 0;                               // one arrival per consumer warp on the ring barriers
  // BN = 128: this warpgroup's 64 weight rows (output channels) for all positions; BN = 64: all weight rows for its NP positions
  const uint32_t a_wg = BN == 128 ? static_cast<uint32_t>(wg) * (kSlabTWBytes<BN> / 2) : 0u;
  const int v_wg = BN == 128 ? 0 : wg * NP;                  // item position of fragment column 0
  const int ch_wg = BN == 128 ? wg * 64 : 0;                 // output channel of fragment row 0 (chunk ch_wg / 8)
  // stmatrix address of this lane: matrix m = lane / 8 is (fragment rows + 8 (m & 1), columns + 8 (m >> 1)); its chunk and the
  // position offset inside a pair of 8-column blocks
  const int m = lane >> 3;
  const uint32_t chunk = static_cast<uint32_t>((BN == 128 ? wg * 8 : 0) + wq * 2 + (m & 1));
  const uint32_t st_lane = stage + static_cast<uint32_t>((v_wg + (m >> 1) * 8 + (lane & 7)) * kRow) + ((chunk ^ (lane & 7)) << 4);
  const uint32_t st_lane2 = stage + static_cast<uint32_t>((v_wg + (lane & 7)) * kRow) + ((chunk ^ (lane & 7)) << 4);   // x2 form
  const __half2 zero2 = __floats2half2_rn(0.f, 0.f);
  int wit = 0, sg = 0, lt = 0;
  for (int item = blockIdx.x; item < p.items_total; item += gridDim.x, ++lt) {
    const SlabItem w = slab_t_item<BN>(p, item);
#pragma unroll
    for (int k = 0; k < NP / 2; ++k) acc[k] = 0.f;
    reg_fence(acc);
    int prev_ws = -1, prev_s = -1;                           // ring slots read by the group in flight
    for (int si = 0; si < w.n_slabs; ++si, ++sg) {
      const int sub = si % p.n_sub;
      const int ntaps = p.sub_ntaps[sub];
      const int s = sg % kSlabSStages;
      mbar_wait(&slab_full[s], (sg / kSlabSStages) & 1);
      const uint32_t slab_addr = slab0 + s * p.slab_bytes;
      for (int ti = 0; ti < ntaps; ++ti, ++wit) {
        const int ws = wit % kSlabWStages;
        mbar_wait(&w_full[ws], (wit / kSlabWStages) & 1);
        const int pix0 = w.q0 + v_wg + p.sub_off[sub][ti] - w.r_lo * p.PW;    // slab pixel of fragment column 0 under this tap
        const uint64_t a = desc_from(kSw128DescHi, sw128_desc_lo(w0s + ws * kSlabTWBytes<BN> + a_wg));
        const uint64_t b = desc_from(kSw128DescHi, sw128_desc_lo(slab_addr + static_cast<uint32_t>(pix0) * 128u));
        wgmma_fence();
        slab_mma<NP>(acc, a, b, 4);                          // C % 64 == 0: every K step holds channels
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
    if (lead) {
      mbar_arrive(&w_empty[prev_ws]);
      mbar_arrive(&slab_empty[prev_s]);
    }
    // fragment rows are output channels ch and ch + 8, columns are positions: affine, round, ReLU per element as the slab epilogue
    const int ch = w.n0 + ch_wg + wq * 16 + (lane >> 2);
    const float sc0 = s_scale[ch], sh0 = s_shift[ch], sc1 = s_scale[ch + 8], sh1 = s_shift[ch + 8];
    const bool relu = p.relu != 0;
    auto pk = [&](float v0, float v1, float sc, float sh) -> uint32_t {
      __half2 hv = __floats2half2_rn(fmaf(v0, sc, sh), fmaf(v1, sc, sh));
      if (relu) hv = __hmax2(hv, zero2);
      return *reinterpret_cast<uint32_t*>(&hv);
    };
    mbar_wait(acc_empty, (lt & 1) ^ 1);
#pragma unroll
    for (int j = 0; j + 1 < NP / 8; j += 2) {
      const uint32_t r[4] = {pk(acc[4 * j], acc[4 * j + 1], sc0, sh0), pk(acc[4 * j + 2], acc[4 * j + 3], sc1, sh1),
                             pk(acc[4 * j + 4], acc[4 * j + 5], sc0, sh0), pk(acc[4 * j + 6], acc[4 * j + 7], sc1, sh1)};
      stmatrix_x4_trans(st_lane + static_cast<uint32_t>(j * 8 * kRow), r);
    }
    if constexpr ((NP / 8) % 2 == 1) {
      constexpr int j = NP / 8 - 1;
      stmatrix_x2_trans(st_lane2 + static_cast<uint32_t>(j * 8 * kRow), pk(acc[4 * j], acc[4 * j + 1], sc0, sh0),
                        pk(acc[4 * j + 2], acc[4 * j + 3], sc1, sh1));
    }
    mbar_arrive(acc_full);
  }
}

// Epilogue warps: each group of BN / 8 threads copies one position row (BN / 8 chunks of 8 channels) of the staging tile to y per
// pass, skipping the positions past the item, past the plane and on halo columns
template <int BN>
__device__ __forceinline__ void slab_t_epilogue(const SlabParams& p, const uint8_t* stage, uint64_t* acc_full, uint64_t* acc_empty) {
  constexpr int kChunks = BN / 8;
  const int et = threadIdx.x - kSlabEpiWarp0 * 32;
  const int slot = et >> (BN == 128 ? 4 : 3), c16 = et & (kChunks - 1);
  constexpr int kSlots = kSlabEpiWarps * 32 / kChunks;
  int lt = 0;
  for (int item = blockIdx.x; item < p.items_total; item += gridDim.x, ++lt) {
    const SlabItem w = slab_t_item<BN>(p, item);
    const bool col_ok = c16 * 8 < p.ldy - w.n0;           // chunks of this N tile that exist in y (incl. zero padding)
    mbar_wait(acc_full, lt & 1);
#pragma unroll 1
    for (int v = slot; v < p.qitem; v += kSlots) {
      const int q = w.q0 + v;
      const int h = fdiv(q, p.fd_PW), wo = q - h * p.PW - p.halo_l;
      if (col_ok && q < p.P && wo >= 0 && wo < p.Wo) {
        const uint4 val = *reinterpret_cast<const uint4*>(stage + v * kSlabTRowBytes<BN> + ((c16 ^ (v & 7)) << 4));
        *reinterpret_cast<uint4*>(p.y + ((static_cast<size_t>(w.plane_o) * p.Ho + h) * p.Wo + wo) * p.ldy + w.n0 + c16 * 8) = val;
      }
    }
    mbar_arrive(acc_empty);
  }
}

// Shared memory: two slab stages, four weight stages, the staging tile, barriers, folded-BN scale / shift
template <int BN, int NP>
__global__ void __launch_bounds__(kSlabThreads, 1)
slab_t_kernel(const __grid_constant__ CUtensorMap tmX,   // input as (C, W, H, N*T), box (64, PW, R, 1)
              const __grid_constant__ CUtensorMap tmB,   // weights [Ncols][taps*C], box (64, BN)
              const SlabParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_align<1024>(smem_raw);
  uint8_t* slab_base = smem;
  uint8_t* w_base = smem + kSlabSStages * p.slab_bytes;
  uint8_t* stage = w_base + kSlabWStages * kSlabTWBytes<BN>;
  uint8_t* tail = stage + kSlabTStageBytes<NP>;
  uint64_t* slab_full = reinterpret_cast<uint64_t*>(tail);
  uint64_t* slab_empty = slab_full + kSlabSStages;
  uint64_t* w_full = slab_empty + kSlabSStages;
  uint64_t* w_empty = w_full + kSlabWStages;
  uint64_t* acc_full = w_empty + kSlabWStages;
  uint64_t* acc_empty = acc_full + 1;
  float* s_scale = reinterpret_cast<float*>(tail + 256);     // barriers occupy the first 128 bytes
  float* s_shift = s_scale + p.naff;

  const int tid = threadIdx.x, warp = tid >> 5;
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
    s_scale[i] = i < p.Ncols ? __ldg(&p.scale[i]) : 0.f;
    s_shift[i] = i < p.Ncols ? __ldg(&p.shift[i]) : 0.f;
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();                       // everything above touched only weights / on-chip state

  if (warp >= kSlabEpiWarp0) {
    setmaxnreg_dec<56>();
    if (warp == kSlabTmaWarp)
      slab_producer<0>(p, &tmX, &tmB, slab_base, w_base, kSlabTWBytes<BN>, BN, slab_full, slab_empty, w_full, w_empty,
                       [&](int it) { return slab_t_item<BN>(p, it); });
    else
      slab_t_epilogue<BN>(p, stage, acc_full, acc_empty);
  } else {
    setmaxnreg_inc<224>();
    slab_t_consumer<BN, NP>(p, smem_u32(slab_base), smem_u32(w_base), smem_u32(stage), s_scale, s_shift, slab_full, slab_empty,
                            w_full, w_empty, acc_full, acc_empty);
  }
}

}  // namespace b2
