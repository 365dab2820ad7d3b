// b2_groupconv.cuh -- grouped 3x3x3 / (1,3,3) "same" convolution with C == K (ResNeXt-3D conv2, resnext3D.py:76-121) at its
// grouped cost: the group-aware MMA step of the slab kernel (b2_slabconv.cuh, slabconv_kernel<64, 0, G>) and the filter packing.
//
// With cg = C / groups in {4, 8, 16, 32} channels per group and C % 64 == 0, a 64-channel slice of the output holds 64 / cg whole
// groups and reads only the same 64 input channels, so the convolution is C / 64 independent 64 -> 64 convolutions.  A work item
// of the slab kernel is (position tiles, slice): the slice index takes the place of the N tile, it is also the channel
// coordinate of the slab's TMA box (one channel chunk per item instead of C / 64), and the slab, its taps, the accumulator
// fragment (64 x 64 per warpgroup and M tile) and the epilogue are the dense 64-channel convolution's.
//
// Inside a slice the filter is block diagonal in blocks of G = 16 channels (G = 32 for cg = 32).  Where the dense kernel issues
// per tap four m64n64k16 MMAs -- K step j into all 64 output channels -- the grouped kernel issues
//   G = 16: four m64n16k16, K step j into accumulator columns [16 j, 16 j + 16)   (fragment registers [8 j, 8 j + 8))
//   G = 32: four m64n32k16, K steps 2 h and 2 h + 1 into columns [32 h, 32 h + 32) (fragment registers [16 h, 16 h + 16))
// Executed over algorithmic multiply-accumulates: 4x (cg = 4), 2x (cg = 8), 1x (cg = 16, 32); the block-diagonal dense filter costs
// C / cg = 32x.  Accumulation is fp32 in a fixed order (temporal tap, input phase, in-plane tap, K step ascending), no atomics.
//
// Packed filter: fp16 [C / 64 slices][taps][G rows][64], C * G * taps elements.  Row r of a (slice, tap) tile holds, in its 16-element
// segment j, the filter row that K step j multiplies: output channel 16 j + r (G = 16) or 32 (j / 2) + r (G = 32) of the slice
// against input channels [16 j, 16 j + 16) of the slice, zero where the two channels are in different groups (cg < 16 only).  One
// TMA box of G 128-byte rows (SWIZZLE_128B) is a tap's weight stage; the B operand of K step j is that tile with its descriptor
// start advanced by 32 j bytes -- the dense kernel's K-step walk, over G rows instead of 64.
#pragma once

#include "b2_ptx.cuh"

namespace b2 {

// diagonal block width of the packed filter for cg channels per group
__host__ __device__ constexpr int group_block(int cg) { return cg == 32 ? 32 : 16; }

// the four K steps of one tap for one 64-row accumulator fragment d (32 registers); a: slab rows, b: the tap's weight stage
template <int G>
__device__ __forceinline__ void group_mma(float* d, uint64_t a, uint64_t b) {
  static_assert(G == 16 || G == 32, "diagonal blocks are 16 or 32 channels wide");
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    if constexpr (G == 16) wgmma_n16<0>(*reinterpret_cast<float(*)[8]>(d + 8 * k), a + 2 * k, b + 2 * k);
    else wgmma_n32<0>(*reinterpret_cast<float(*)[16]>(d + 16 * (k >> 1)), a + 2 * k, b + 2 * k);
  }
}

// fp32 [K][cg][taps] (nn.Conv3d.weight of a grouped convolution) -> the packed filter above; one thread per packed element
__global__ void pack_grouped_weight_kernel(const float* __restrict__ w, __half* __restrict__ out, int cg, int taps, int G,
                                           long long total) {
  const long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int kk = (int)(i & 15), j = (int)((i >> 4) & 3);
  const long long row = i >> 6;                       // (slice, tap, r)
  const int r = (int)(row % G);
  const long long st = row / G;
  const int tap = (int)(st % taps), slice = (int)(st / taps);
  const int o = slice * 64 + (G == 16 ? 16 * j + r : 32 * (j >> 1) + r);
  const int ci = slice * 64 + 16 * j + kk;
  float v = 0.f;
  if (o / cg == ci / cg) v = w[((long long)o * cg + ci % cg) * taps + tap];
  out[i] = __float2half_rn(v);
}

}  // namespace b2
