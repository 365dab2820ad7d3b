// b2_probe.cu -- single-CTA experiments that pin down the wgmma shared-memory descriptor semantics the
// convolution kernels rely on.  Not part of the product path; exercised by tools/probe_umma.py.
//
//   mode 0: K-major SWIZZLE_128B A operand whose start address is shifted by `shift` rows (128 B each)
//           from a 1024-byte aligned tile, with descriptor base_offset = `base_off`.  Expected result:
//           D[r][n] = sum_k A[shift + r][k] * B[n][k]   (A is 256 x 64, loaded by TMA as two boxes).
//   mode 2: MN-major SWIZZLE_128B B operand.  B is given as V[K = 64][N = 128] row-major (N contiguous), loaded
//           by TMA as two [64 n x 64 k-rows] boxes 8 KB apart; descriptor: LBO = 8192 (next 64-wide N block),
//           SBO = 1024 (next 8 K rows), K step of 16 = +2048 B; B transposed (MN-major) in the instruction.
//           Expected: D[r][n] = sum_k A[r][k] * V[k][n]  with N = 128.
//   mode 1: K-major SWIZZLE_NONE A operand built as an overlapping (Toeplitz) view of a linear buffer:
//           row r starts at byte 16*r, K = 32 elements: LBO = 16 B, SBO = 128 B.
//           Expected: D[r][n] = sum_{k<32} buf[8*r + k] * B[n][k].
//   mode 3: the mode 0 question for the B operand (the slab kernel's 64-wide tile reads its slab as B): K-major SWIZZLE_128B
//           B of N = `base_off` (64, 128 or 192) rows whose start address is shifted by `shift` rows from a 1024-byte aligned
//           tile; A is the 64 x 64 K-major tile given as `b`, the 256 x 64 tile given as `a` holds the B rows.  Expected:
//           D[m][n] = sum_k b[m][k] * a[shift + n][k], written to out as [64][N].
//   mode 4: the mode 1 Toeplitz view as the B operand at N = 112 (the transposed stem reads a slab row so): A is the 64 x 32
//           no-swizzle K-major tile of mode 1's B (LBO = 128 B, SBO = 512 B), B row n starts at byte 16*n of the linear buffer
//           (LBO = 16 B, SBO = 128 B).  Expected: D[m][n] = sum_{k<32} b[m][k] * buf[8*n + k], written to out as [64][112].
#include "b2_host.h"
#include "b2_ptx.cuh"

#include <string.h>

namespace b2 {

// modes 3 and 4: accumulator fragments of an m64nN tile written straight to out[64][N]
template <int N>
__device__ void probe_store_frag(const float (&d)[N / 2], float* __restrict__ out) {
  const int t = threadIdx.x & 127;
  const int r = (t >> 5) * 16 + ((t & 31) >> 2), c = 2 * (t & 3);
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
    out[r * N + 8 * j + c] = d[4 * j];
    out[r * N + 8 * j + c + 1] = d[4 * j + 1];
    out[(r + 8) * N + 8 * j + c] = d[4 * j + 2];
    out[(r + 8) * N + 8 * j + c + 1] = d[4 * j + 3];
  }
}

// mode 3: one m64nNk16 chain with the accumulators in registers
template <int N>
__device__ void probe_shifted_b(uint32_t a_addr, uint32_t b_addr, float* __restrict__ out) {
  float d[N / 2];
#pragma unroll
  for (int i = 0; i < N / 2; ++i) d[i] = 0.f;
  reg_fence(d);
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < 4; ++k)
    wgmma_ss<N>(d, make_desc_sw128_kmajor(a_addr) + 2 * k, make_desc_sw128_kmajor(b_addr) + 2 * k);
  wgmma_commit();
  wgmma_wait0();
  reg_fence(d);
  probe_store_frag<N>(d, out);
}

// mode 4: two K steps of 16 (A +256 B, B +32 B), as the transposed stem issues them
__device__ void probe_toeplitz_b(uint32_t a_addr, uint32_t b_addr, float* __restrict__ out) {
  float d[56];
#pragma unroll
  for (int i = 0; i < 56; ++i) d[i] = 0.f;
  reg_fence(d);
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < 2; ++k)
    wgmma_ss<112>(d, make_desc_noswz_kmajor(a_addr, 128, 512) + 16 * k, make_desc_noswz_kmajor(b_addr, 16, 128) + 2 * k);
  wgmma_commit();
  wgmma_wait0();
  reg_fence(d);
  probe_store_frag<112>(d, out);
}

__global__ void __launch_bounds__(128, 1)
mma_probe_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                 const __half* __restrict__ lin_a, const __half* __restrict__ lin_b, float* __restrict__ out,
                 int mode, int shift, int base_off) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_align<1024>(smem_raw);
  uint8_t* sA = smem;                 // 256 rows x 128 B = 32 KB
  uint8_t* sB = smem + 32768;         // 64 rows x 128 B  = 8 KB (mode 0) / no-swizzle B (mode 1)
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem + 32768 + 8192);
  const AccTile at{reinterpret_cast<float*>(smem + 32768 + 8192 + 64), acc_ld(128)};
  const int tid = threadIdx.x;

  if (tid == 0) { mbar_init(bar, 1); fence_mbar_init(); }
  __syncthreads();

  const int ncol = (mode == 2) ? 128 : 64;
  if (mode == 3) {
    if (tid == 0) {
      mbar_expect_tx(bar, 32768 + 8192);
      tma_load_2d(sA, &tmA, bar, 0, 0);
      tma_load_2d(sA + 16384, &tmA, bar, 0, 128);
      tma_load_2d(sB, &tmB, bar, 0, 0);
    }
    mbar_wait(bar, 0);
    const uint32_t b_addr = smem_u32(sA) + shift * 128;
    if (base_off == 64) probe_shifted_b<64>(smem_u32(sB), b_addr, out);
    else if (base_off == 128) probe_shifted_b<128>(smem_u32(sB), b_addr, out);
    else probe_shifted_b<192>(smem_u32(sB), b_addr, out);
    return;
  }
  if (mode == 0) {
    if (tid == 0) {
      mbar_expect_tx(bar, 32768 + 8192);
      tma_load_2d(sA, &tmA, bar, 0, 0);
      tma_load_2d(sA + 16384, &tmA, bar, 0, 128);
      tma_load_2d(sB, &tmB, bar, 0, 0);
    }
    mbar_wait(bar, 0);
    const uint64_t ad = make_desc_sw128_kmajor(smem_u32(sA) + shift * 128) | (static_cast<uint64_t>(base_off & 7) << 49);
    wg_mma(at, 0, 64, wg_sw128(ad, make_desc_sw128_kmajor(smem_u32(sB))), 4, false);
  } else if (mode == 2) {
    if (tid == 0) {
      mbar_expect_tx(bar, 16384 + 16384);
      tma_load_2d(sA, &tmA, bar, 0, 0);                 // A: 128 x 64 K-major
      tma_load_2d(sA + 16384, &tmB, bar, 0, 0);         // V block n in [0,64):   64 k-rows x 128 B
      tma_load_2d(sA + 16384 + 8192, &tmB, bar, 64, 0); // V block n in [64,128)
    }
    mbar_wait(bar, 0);
    uint64_t bd = 0;
    bd |= static_cast<uint64_t>(((smem_u32(sA + 16384)) & 0x3FFFF) >> 4);
    bd |= static_cast<uint64_t>(8192 >> 4) << 16;   // LBO: next 64-wide N block
    bd |= static_cast<uint64_t>(1024 >> 4) << 32;   // SBO: next 8 K rows
    bd |= static_cast<uint64_t>(1) << 62;           // SWIZZLE_128B
    const WgOperands ops{make_desc_sw128_kmajor(smem_u32(sA)), bd, 2u, 512u, 128u, 512u, 0u};
    wg_mma<1>(at, 0, 128, ops, 4, false);
  } else {
    // linear buffers copied with plain stores: A buffer 4 KB (2048 halfs), B = 64 rows x 32 k in the
    // canonical no-swizzle K-major layout: chunk (n, j) at (n/8)*SBO_B + j*LBO_B + (n%8)*16, LBO_B = 128,
    // SBO_B = 512 (4 K-chunks of 16 B per 8-row group).
    for (int i = tid; i < 2048; i += 128) reinterpret_cast<__half*>(sA)[i] = lin_a[i];
    for (int i = tid; i < 64 * 32; i += 128) {
      const int n = i / 32, k = i % 32;
      const int off = (n / 8) * 512 + (k / 8) * 128 + (n % 8) * 16 + (k % 8) * 2;
      *reinterpret_cast<__half*>(sB + off) = lin_b[i];
    }
    fence_proxy_async();
    __syncthreads();
    if (mode == 4) {
      probe_toeplitz_b(smem_u32(sB), smem_u32(sA), out);
      return;
    }
    // K = 32 -> two K=16 steps; A advances two 16-byte chunks (32 B), B two 128-byte chunk columns (256 B)
    const WgOperands ops{make_desc_noswz_kmajor(smem_u32(sA), /*LBO*/ 16, /*SBO*/ 128),
                         make_desc_noswz_kmajor(smem_u32(sB), /*LBO*/ 128, /*SBO*/ 512), 2u, 64u, 16u, 256u, 64u};
    wg_mma(at, 0, 64, ops, 2, false);
  }
  __syncthreads();
  uint32_t v[32];
  for (int j = 0; j < ncol / 32; ++j) {
    acc_ld32(at, tid, j * 32, v);
    for (int i = 0; i < 32; ++i) out[tid * ncol + j * 32 + i] = __uint_as_float(v[i]);
  }
}

}  // namespace b2

using namespace b2;

// a: mode 0 / 3 -> fp16 [256][64]; mode 1 / 4 -> fp16 [2048] linear.  b: mode 0 / 3 -> fp16 [64][64]; mode 1 / 4 -> fp16 [64][32].
// out: mode 3 -> fp32 [64][base_off], mode 4 -> [64][112], otherwise [128][64] ([128][128] for mode 2).
extern "C" int b2_debug_umma_probe(const void* a, const void* b, float* out, int mode, int shift, int base_off,
                                   void* stream) {
  B2_CHECK_ARG(a && b && out, "null pointer");
  B2_CHECK_ARG(mode != 3 || ((base_off == 64 || base_off == 128 || base_off == 192) && shift >= 0 && shift + base_off <= 256),
               "mode 3 takes N = 64, 128 or 192 rows of B inside the 256-row tile");
  int rc;
  if ((rc = require_sm90()) != B2_OK) return rc;
  const int smem_bytes = 32768 + 8192 + 64 + acc_bytes(128) + 1024;
  B2_OPT_IN_SMEM(mma_probe_kernel, smem_bytes);
  CUtensorMap tmA, tmB;
  memset(&tmA, 0, sizeof(tmA)); memset(&tmB, 0, sizeof(tmB));
  if (mode == 0 || mode == 3) {
    if ((rc = make_tmap_2d_f16(&tmA, a, 64, 256, 64, 64, 128, true)) != B2_OK) return rc;
    if ((rc = make_tmap_2d_f16(&tmB, b, 64, 64, 64, 64, 64, true)) != B2_OK) return rc;
  } else if (mode == 2) {
    if ((rc = make_tmap_2d_f16(&tmA, a, 64, 128, 64, 64, 128, true)) != B2_OK) return rc;
    if ((rc = make_tmap_2d_f16(&tmB, b, 128, 64, 128, 64, 64, true)) != B2_OK) return rc;   // V[64][128]
  }
  mma_probe_kernel<<<1, 128, smem_bytes, reinterpret_cast<cudaStream_t>(stream)>>>(
      tmA, tmB, reinterpret_cast<const __half*>(a), reinterpret_cast<const __half*>(b), out, mode, shift, base_off);
  B2_CHECK_LAUNCH("mma_probe_kernel");
  return B2_OK;
}
