// b2_slab_t128.cuh -- the slab convolution (b2_slabconv.cuh) for 128-wide output tiles as the transposed product.
//
// The slab kernel's 128-wide N tile runs one 128-position M tile per work item (kSlabAccCols = 192 leaves room for no second), so
// each 16 KB weight stage (one tap x one 64-channel chunk x 128 outputs) serves 128 positions and is fetched from L2 again for the
// next item: layers 2-3 of the 3-D ResNets stream ~5 bytes of filter per MAC column from L2.  Here each consumer warpgroup owns 64
// of the tile's 128 output channels -- its half of the weight stage (8 KB, 1024-aligned) is the m64 A operand -- and the B operand
// is a whole work item of NP padded positions taken straight from the slab rows (K-major SWIZZLE_128B, taps are row shifts of the
// start address as in the slab kernel): one m64 n(NP) k16 per K step.  An item is `rows` whole output rows of one (n, t) plane
// (SlabParams::qitem = rows * PW positions, NP = qitem rounded up to a compiled width), so a weight stage serves up to 256
// positions, and per tensor cycle the MMAs read 2 x (2 KB + NP x 32 B) / NP bytes of shared memory (80 at NP = 256) instead of 96.
// Every compiled column is issued: the positions past qitem fall on rows of the slab that the host sized for NP positions from
// every item start, and their columns are dropped by the epilogue.
//
// The NP / 2 fp32 accumulators per consumer thread (108 - 128) need more than the 168 registers twelve warps get: setmaxnreg moves
// the producer / epilogue warpgroup down to 56 and the consumers up to 224.  An fp32 accumulator tile of NP x 128 would not fit next
// to the slab and weight rings, so the consumers apply the folded-BN affine and the ReLU to their fragments themselves (the same
// fp32 expression and single rounding as the slab kernel's epilogue) and store fp16 with stmatrix .trans into a [position][channel]
// staging tile; the three epilogue warps copy its valid rows to y.  Every output element keeps the slab kernel's accumulation order
// (temporal tap, channel chunk, phase, in-plane tap, K step), so the outputs are bitwise those of the slab kernel.
//
// Scope (slab_t128_geometry in b2_conv_api.cu): 3x3 or 3x3x3 filters with in-plane padding 0 ("valid") or 1 ("same") and temporal
// padding "same" -- slab_geometry's tap table, whose row offsets are centred on the window -- spatial stride 1 or 2 (the phase
// sub-images of the slab producer, unchanged), C % 64 == 0, K % 128 == 0, rows that fit one TMA box; no residual, per-sample affine
// or upsampling.
#pragma once

#include "b2_slabconv.cuh"

namespace b2 {

constexpr int kT128WBytes = 128 * 128;   // weight stage: 128 output channels x one 64-channel chunk of one tap
constexpr int kT128RowBytes = 128 * 2;   // staging tile row: one position's 128 fp16 channels

// Work item = (N tile, row group of a plane, plane) in the slab kernel's order; SlabParams::MT = 1, so slab_item's q0 is the row
// group's index times 128
__device__ __forceinline__ SlabItem slab_t128_item(const SlabParams& p, int item) {
  SlabItem w = slab_item(p, item, 128);
  w.q0 = (w.q0 >> 7) * p.qitem;
  const int lo = w.q0 - p.reach;
  w.r_lo = (lo >= 0) ? fdiv(lo, p.fd_PW) : -fdiv(-lo + p.PW - 1, p.fd_PW);
  return w;
}

// Staging tile: row v (position) holds 16 chunks of 8 channels, chunk c at (c ^ (v & 7)) * 16, so that the 8 rows of one stmatrix
// matrix (one chunk, 8 consecutive positions) fall in 8 different bank groups
template <int NP>
__device__ __forceinline__ void slab_t128_consumer(const SlabParams& p, uint32_t slab0, uint32_t w0s, uint32_t stage,
                                                   const float* s_scale, const float* s_shift, uint64_t* slab_full,
                                                   uint64_t* slab_empty, uint64_t* w_full, uint64_t* w_empty, uint64_t* acc_full,
                                                   uint64_t* acc_empty) {
  float acc[NP / 2];
  const int wg = warp_uniform(threadIdx.x >> 7);
  const int lane = threadIdx.x & 31, wq = (threadIdx.x >> 5) & 3;
  const bool lead = lane == 0;                               // one arrival per consumer warp on the ring barriers
  const uint32_t a_wg = static_cast<uint32_t>(wg) * (kT128WBytes / 2);   // this warpgroup's 64 weight rows
  // stmatrix address of this lane: matrix m = lane / 8 is (fragment rows + 8 (m & 1), columns + 8 (m >> 1)); its chunk and the
  // position offset inside a pair of 8-column blocks
  const int m = lane >> 3;
  const uint32_t chunk = static_cast<uint32_t>(wg * 8 + wq * 2 + (m & 1));
  const uint32_t st_lane = stage + static_cast<uint32_t>(((m >> 1) * 8 + (lane & 7)) * kT128RowBytes) + ((chunk ^ (lane & 7)) << 4);
  const uint32_t st_lane2 = stage + static_cast<uint32_t>((lane & 7) * kT128RowBytes) + ((chunk ^ (lane & 7)) << 4);   // x2 form
  const __half2 zero2 = __floats2half2_rn(0.f, 0.f);
  int wit = 0, sg = 0, lt = 0;
  for (int item = blockIdx.x; item < p.items_total; item += gridDim.x, ++lt) {
    const SlabItem w = slab_t128_item(p, item);
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
        const int pix0 = w.q0 + p.sub_off[sub][ti] - w.r_lo * p.PW;    // slab pixel of position q0 under this tap
        const uint64_t a = desc_from(kSw128DescHi, sw128_desc_lo(w0s + ws * kT128WBytes + a_wg));
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
    const int ch = w.n0 + wg * 64 + wq * 16 + (lane >> 2);
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
      stmatrix_x4_trans(st_lane + static_cast<uint32_t>(j * 8 * kT128RowBytes), r);
    }
    if constexpr ((NP / 8) % 2 == 1) {
      constexpr int j = NP / 8 - 1;
      stmatrix_x2_trans(st_lane2 + static_cast<uint32_t>(j * 8 * kT128RowBytes), pk(acc[4 * j], acc[4 * j + 1], sc0, sh0),
                        pk(acc[4 * j + 2], acc[4 * j + 3], sc1, sh1));
    }
    mbar_arrive(acc_full);
  }
}

// Epilogue warps: each half-warp copies one position row (16 chunks of 8 channels) of the staging tile to y per pass, skipping the
// positions past the item's rows, past the plane and on halo columns
__device__ __forceinline__ void slab_t128_epilogue(const SlabParams& p, const uint8_t* stage, uint64_t* acc_full, uint64_t* acc_empty) {
  const int et = threadIdx.x - kSlabEpiWarp0 * 32;
  const int slot = et >> 4, c16 = et & 15;
  constexpr int kSlots = kSlabEpiWarps * 2;
  int lt = 0;
  for (int item = blockIdx.x; item < p.items_total; item += gridDim.x, ++lt) {
    const SlabItem w = slab_t128_item(p, item);
    const bool col_ok = c16 * 8 < p.ldy - w.n0;           // chunks of this N tile that exist in y (incl. zero padding)
    mbar_wait(acc_full, lt & 1);
#pragma unroll 1
    for (int v = slot; v < p.qitem; v += kSlots) {
      const int q = w.q0 + v;
      const int h = fdiv(q, p.fd_PW), wo = q - h * p.PW - p.halo_l;
      if (col_ok && q < p.P && wo >= 0 && wo < p.Wo) {
        const uint4 val = *reinterpret_cast<const uint4*>(stage + v * kT128RowBytes + ((c16 ^ (v & 7)) << 4));
        *reinterpret_cast<uint4*>(p.y + ((static_cast<size_t>(w.plane_o) * p.Ho + h) * p.Wo + wo) * p.ldy + w.n0 + c16 * 8) = val;
      }
    }
    mbar_arrive(acc_empty);
  }
}

// Shared memory: two slab stages, four 16 KB weight stages, the NP x 256 B staging tile, barriers, folded-BN scale / shift
template <int NP>
__global__ void __launch_bounds__(kSlabThreads, 1)
slab_t128_kernel(const __grid_constant__ CUtensorMap tmX,   // input as (C, W, H, N*T), box (64, PW, R, 1)
                 const __grid_constant__ CUtensorMap tmB,   // weights [Ncols][taps*C], box (64, 128)
                 const SlabParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_align<1024>(smem_raw);
  uint8_t* slab_base = smem;
  uint8_t* w_base = smem + kSlabSStages * p.slab_bytes;
  uint8_t* stage = w_base + kSlabWStages * kT128WBytes;
  uint8_t* tail = stage + NP * kT128RowBytes;
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
      slab_producer<0>(p, &tmX, &tmB, slab_base, w_base, kT128WBytes, 128, slab_full, slab_empty, w_full, w_empty,
                       [&](int it) { return slab_t128_item(p, it); });
    else
      slab_t128_epilogue(p, stage, acc_full, acc_empty);
  } else {
    setmaxnreg_inc<224>();
    slab_t128_consumer<NP>(p, smem_u32(slab_base), smem_u32(w_base), smem_u32(stage), s_scale, s_shift, slab_full, slab_empty,
                           w_full, w_empty, acc_full, acc_empty);
  }
}

}  // namespace b2
