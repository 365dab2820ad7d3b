// b2_ptx.cuh -- thin inline-PTX wrappers for the sm_90a features the hot path uses:
// mbarrier, TMA (cp.async.bulk.tensor), cp.async, wgmma and the shared-memory matrix descriptors it consumes.
//
// Everything here is device-side and header-only.  No CUTLASS/CuTe is used; the bit layouts
// follow the PTX ISA "matrix descriptor" table of the warpgroup-level MMA.
#pragma once

#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace b2 {

// ------------------------------------------------------------------------------------------
// address helpers
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// Aligns the dynamic shared-memory base with pointer arithmetic on the __shared__ array itself.  Going through
// uintptr_t makes the compiler lose the address space: every later access becomes a generic LD/ST.
// Programmatic dependent launch: the tensor-core kernels are launched with programmatic stream serialization, so a
// CTA of launch i+1 starts (barrier init, tensor-map prefetch, BN-affine staging) on every SM that
// launch i has vacated and only then waits for launch i to finish; without the attribute both are no-ops.
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

template <int ALIGN>
__device__ __forceinline__ uint8_t* smem_align(uint8_t* smem_raw) {
  return smem_raw + ((ALIGN - (smem_u32(smem_raw) & (ALIGN - 1))) & (ALIGN - 1));
}

// ------------------------------------------------------------------------------------------
// mbarrier
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ uint32_t mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok;
}
// Blocking wait with a watchdog: a pipeline bug traps (surfacing as a CUDA error in the caller)
// instead of hanging the GPU.  try_wait suspends in hardware, so the loop count is small in
// the normal case.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
#ifndef B2_NO_WATCHDOG
  uint32_t spins = 0;
#endif
  while (!mbar_try_wait(bar, parity)) {
#ifndef B2_NO_WATCHDOG
    if (++spins > (1u << 24)) __trap();
#endif
  }
}

// generic-proxy writes (st.shared / cp.async) -> async-proxy readers (TMA store, wgmma)
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ------------------------------------------------------------------------------------------
// TMA (tiled mode).  Coordinates are innermost-first, in elements.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0,
                                            int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0,
                                            int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1),
      "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0,
                                            int c1, int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1),
      "r"(c2), "r"(c3)
      : "memory");
}
__device__ __forceinline__ void tma_load_5d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0,
                                            int c1, int c2, int c3, int c4) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.tile.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1),
      "r"(c2), "r"(c3), "r"(c4)
      : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, const void* smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.tile.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// all but the most recent bulk store group have finished READING shared memory (double-buffered staging tiles)
__device__ __forceinline__ void tma_store_wait_read1() { asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_read0() {
  asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}

// ------------------------------------------------------------------------------------------
// cp.async (LDGSTS): 16-byte gather with zero fill (src_bytes == 0 writes 16 zero bytes)
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void cp_async_16_ca(uint32_t smem_dst, const void* gsrc, uint32_t src_bytes) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 16, %2;" ::"r"(smem_dst), "l"(gsrc), "r"(src_bytes)
               : "memory");
}
__device__ __forceinline__ void cp_async_16_cg(uint32_t smem_dst, const void* gsrc, uint32_t src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_dst), "l"(gsrc), "r"(src_bytes)
               : "memory");
}
// arrive on `bar` once every cp.async this thread issued so far has landed (counts against the
// barrier's expected arrival count: .noinc)
__device__ __forceinline__ void cp_async_mbar_arrive_noinc(uint64_t* bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}

// ------------------------------------------------------------------------------------------
// Warpgroup MMA (wgmma) into an accumulator tile in shared memory
// ------------------------------------------------------------------------------------------
// Hopper has no tensor memory: the fp32 accumulators of a 128-row MMA tile live in shared memory as [128 rows][ld]
// ("AccTile", ld = columns + 4 so that neither the fragment stores nor the row-per-thread reads of the epilogue
// conflict).  One warpgroup (4 warps, 128 threads) issues the MMAs: wg_mma() loads a 64 x <=64 piece of the tile
// into registers, accumulates one K block with wgmma (both operands from shared memory, K-major or, for B, MN-major
// descriptors), waits for it and stores the piece back.  An epilogue thread owns tile row r and reads / writes
// 32 consecutive columns at a time (acc_ld32 / acc_st32 / acc_zero32).
struct AccTile {
  float* p;   // row 0, column 0
  int ld;     // row pitch in floats
};
__host__ __device__ constexpr int acc_ld(int cols) { return cols + 4; }
__host__ __device__ constexpr int acc_bytes(int cols) { return 128 * acc_ld(cols) * 4; }

__device__ __forceinline__ void acc_ld32(const AccTile& t, int row, int col, uint32_t (&v)[32]) {
  const float4* s = reinterpret_cast<const float4*>(t.p + static_cast<size_t>(row) * t.ld + col);
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const float4 f = s[q];
    v[4 * q] = __float_as_uint(f.x); v[4 * q + 1] = __float_as_uint(f.y);
    v[4 * q + 2] = __float_as_uint(f.z); v[4 * q + 3] = __float_as_uint(f.w);
  }
}
__device__ __forceinline__ void acc_st32(const AccTile& t, int row, int col, const uint32_t (&v)[32]) {
  float4* s = reinterpret_cast<float4*>(t.p + static_cast<size_t>(row) * t.ld + col);
#pragma unroll
  for (int q = 0; q < 8; ++q)
    s[q] = make_float4(__uint_as_float(v[4 * q]), __uint_as_float(v[4 * q + 1]), __uint_as_float(v[4 * q + 2]),
                       __uint_as_float(v[4 * q + 3]));
}
__device__ __forceinline__ void acc_zero32(const AccTile& t, int row, int col) {
  float4* s = reinterpret_cast<float4*>(t.p + static_cast<size_t>(row) * t.ld + col);
#pragma unroll
  for (int q = 0; q < 8; ++q) s[q] = make_float4(0.f, 0.f, 0.f, 0.f);
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait1() { asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory"); }
// Register accumulators that wgmma reads and writes asynchronously: keeps the compiler from moving ordinary reads or writes of
// them across a wgmma.fence / wait_group.
template <int N>
__device__ __forceinline__ void reg_fence(float (&d)[N]) {
#pragma unroll
  for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

template <int TB>
__device__ __forceinline__ void wgmma_n64(float (&d)[32], uint64_t a, uint64_t b) {
  asm volatile(
      "{\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, 1, 1, 1, 0, %34;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(a), "l"(b), "n"(TB));
}
template <int TB>
__device__ __forceinline__ void wgmma_n32(float (&d)[16], uint64_t a, uint64_t b) {
  asm volatile(
      "{\n"
      "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, 1, 1, 1, 0, %18;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(a), "l"(b), "n"(TB));
}
template <int TB>
__device__ __forceinline__ void wgmma_n16(float (&d)[8], uint64_t a, uint64_t b) {
  asm volatile(
      "{\n"
      "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, 1, 1, 1, 0, %10;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
      : "l"(a), "l"(b), "n"(TB));
}

// D[64 x 128] += A[64 x 16] . B[128 x 16]^T, both operands K-major in shared memory (descriptors), D in registers
__device__ __forceinline__ void wgmma_n128_ss(float (&d)[64], uint64_t a, uint64_t b) {
  asm volatile(
      "{\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, 1, 1, 1, 0, 0;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a), "l"(b));
}
// Same shape with BOTH operands MN-major (transposed) in shared memory: A is a [16 K rows][64 M] tile, B a [16 K rows][128 N]
// tile, each row holding consecutive M / N elements (the natural [positions][channels] layout of an activation)
__device__ __forceinline__ void wgmma_n128_ss_mn(float (&d)[64], uint64_t a, uint64_t b) {
  asm volatile(
      "{\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, 1, 1, 1, 1, 1;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a), "l"(b));
}
// D[64 x N] += A[64 x 16] . B[N x 16]^T, both operands K-major in shared memory, D = d[0, N / 2) in registers: one instruction for
// each N tile of the slab kernels.  N = 144 ... 192 are runtime tiles for the channel counts of the (2+1)D factorisation.
template <int N>
__device__ __forceinline__ void wgmma_ss(float* d, uint64_t a, uint64_t b);
template <>
__device__ __forceinline__ void wgmma_ss<16>(float* d, uint64_t a, uint64_t b) { wgmma_n16<0>(*reinterpret_cast<float(*)[8]>(d), a, b); }
template <>
__device__ __forceinline__ void wgmma_ss<64>(float* d, uint64_t a, uint64_t b) { wgmma_n64<0>(*reinterpret_cast<float(*)[32]>(d), a, b); }
template <>
__device__ __forceinline__ void wgmma_ss<128>(float* d, uint64_t a, uint64_t b) { wgmma_n128_ss(*reinterpret_cast<float(*)[64]>(d), a, b); }
template <>
__device__ __forceinline__ void wgmma_ss<144>(float* d, uint64_t a, uint64_t b) {
  asm volatile(
      "{\n"
      "wgmma.mma_async.sync.aligned.m64n144k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71}, %72, %73, 1, 1, 1, 0, 0;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71])
      : "l"(a), "l"(b));
}
template <>
__device__ __forceinline__ void wgmma_ss<160>(float* d, uint64_t a, uint64_t b) {
  asm volatile(
      "{\n"
      "wgmma.mma_async.sync.aligned.m64n160k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79}, %80, %81, 1, 1, 1, 0, 0;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79])
      : "l"(a), "l"(b));
}
template <>
__device__ __forceinline__ void wgmma_ss<176>(float* d, uint64_t a, uint64_t b) {
  asm volatile(
      "{\n"
      "wgmma.mma_async.sync.aligned.m64n176k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87}, %88, %89, 1, 1, 1, 0, 0;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87])
      : "l"(a), "l"(b));
}
template <>
__device__ __forceinline__ void wgmma_ss<192>(float* d, uint64_t a, uint64_t b) {
  asm volatile(
      "{\n"
      "wgmma.mma_async.sync.aligned.m64n192k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95}, %96, %97, 1, 1, 1, 0, 0;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95])
      : "l"(a), "l"(b));
}
// D[64 x 64] += A[64 x 16] . B, A from registers (four fp16x2 per thread in the accumulator-fragment layout of its
// columns), B a shared-memory descriptor (TB = 1: MN-major)
template <int TB>
__device__ __forceinline__ void wgmma_n64_rs(float (&d)[32], const uint32_t (&a)[4], uint64_t b) {
  asm volatile(
      "{\n"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, 1, 1, 1, %37;\n"
      "}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "n"(TB));
}

// Operand walk of wg_mma: descriptor of rows / columns 0 at K step 0 and the descriptor increments (16-byte units)
// per 16-element K step, per 64 rows of A, per 64 and per 16 columns of B.
struct WgOperands {
  uint64_t a, b;
  uint32_t a_k, a_m64, b_k, b_n64, b_n16;
};
// K-major SWIZZLE_128B tiles (rows 128 B apart): K step +32 B, 16 rows +2 KB
__device__ __forceinline__ WgOperands wg_sw128(uint64_t a, uint64_t b) {
  return WgOperands{a, b, 2u, 512u, 2u, 512u, 128u};
}

// Fragment <-> tile: thread t of the warpgroup holds rows 16 (t / 32) + (t % 32) / 4 (+ 8) of a 64-row piece and
// column pairs 8 j + 2 (t % 4).
template <int W>
__device__ __forceinline__ void frag_io(const AccTile& t, int row0, int col0, float (&d)[W / 2], bool load, bool zero) {
  const int wt = threadIdx.x & 127;
  const int row = row0 + (wt >> 5) * 16 + ((wt & 31) >> 2);
  float* p0 = t.p + static_cast<size_t>(row) * t.ld + col0 + 2 * (wt & 3);
  float* p1 = p0 + 8 * t.ld;
#pragma unroll
  for (int j = 0; j < W / 8; ++j) {
    if (load) {
      float2 u = zero ? make_float2(0.f, 0.f) : *reinterpret_cast<const float2*>(p0 + 8 * j);
      float2 w = zero ? make_float2(0.f, 0.f) : *reinterpret_cast<const float2*>(p1 + 8 * j);
      d[4 * j] = u.x; d[4 * j + 1] = u.y; d[4 * j + 2] = w.x; d[4 * j + 3] = w.y;
    } else {
      *reinterpret_cast<float2*>(p0 + 8 * j) = make_float2(d[4 * j], d[4 * j + 1]);
      *reinterpret_cast<float2*>(p1 + 8 * j) = make_float2(d[4 * j + 2], d[4 * j + 3]);
    }
  }
}

template <int W, int TB>
__device__ __forceinline__ void wg_mma_piece(const AccTile& t, int row0, int col0, uint64_t a, uint64_t b, uint32_t a_k,
                                             uint32_t b_k, int ksteps, bool accumulate) {
  float d[W / 2];
  frag_io<W>(t, row0, col0, d, true, !accumulate);
  wgmma_fence();
  for (int k = 0; k < ksteps; ++k) {
    if constexpr (W == 64) wgmma_n64<TB>(d, a + k * a_k, b + k * b_k);
    else if constexpr (W == 32) wgmma_n32<TB>(d, a + k * a_k, b + k * b_k);
    else wgmma_n16<TB>(d, a + k * a_k, b + k * b_k);
  }
  wgmma_commit();
  wgmma_wait0();
  frag_io<W>(t, row0, col0, d, false, false);
}

// D[128 rows][col0, col0 + n) (+)= A[128][16 ksteps] . B[n][16 ksteps]^T.  Called by all 128 threads of the MMA
// warpgroup with warp-uniform arguments; n is a multiple of 16 (of 64 for an MN-major B, TB = 1).  Synchronous: the
// operands have been read and the tile updated when every thread has returned.
template <int TB = 0>
__device__ __forceinline__ void wg_mma(const AccTile& t, int col0, int n, const WgOperands& o, int ksteps, bool accumulate) {
#pragma unroll 1
  for (int h = 0; h < 2; ++h) {
    const uint64_t a = o.a + h * o.a_m64;
    int c = 0;
#pragma unroll 1
    for (; c + 64 <= n; c += 64)
      wg_mma_piece<64, TB>(t, h * 64, col0 + c, a, o.b + (c / 64) * o.b_n64, o.a_k, o.b_k, ksteps, accumulate);
    if (c + 32 <= n) {
      wg_mma_piece<32, TB>(t, h * 64, col0 + c, a, o.b + (c / 64) * o.b_n64, o.a_k, o.b_k, ksteps, accumulate);
      c += 32;
    }
    if (c < n)
      wg_mma_piece<16, TB>(t, h * 64, col0 + c, a, o.b + (c / 64) * o.b_n64 + ((c % 64) / 16) * o.b_n16, o.a_k, o.b_k,
                           ksteps, accumulate);
  }
}

// A value every lane of the warp already agrees on, made visibly warp-uniform to ptxas.  A branch around a wgmma whose condition it cannot
// prove uniform makes it serialise the whole wgmma pipeline of the kernel (C7520); one read from lane 0 avoids that.
__device__ __forceinline__ int warp_uniform(int v) { return __shfl_sync(0xffffffffu, v, 0); }

// The MMA warpgroup has finished with what it read and wrote: one thread arrives on `bar` (expected count 1).
// Named barrier 15 is reserved for the MMA warpgroup.
__device__ __forceinline__ void wg_sync() { asm volatile("bar.sync 15, 128;" ::: "memory"); }
__device__ __forceinline__ void wg_arrive(uint64_t* bar) {
  if ((threadIdx.x & 127) == 0) mbar_arrive(bar);
}

// ------------------------------------------------------------------------------------------
// descriptors
// ------------------------------------------------------------------------------------------
// Shared-memory matrix descriptor (64 bit):
//   [ 0,14) start address >> 4        [16,30) leading-dim byte offset >> 4
//   [32,46) stride-dim byte offset>>4 [49,52) base offset
//   [62,64) layout: 0 none, 1 = 128B swizzle, 2 = 64B, 3 = 32B
// The swizzle is a function of the absolute shared-memory address bits, so a start address moved by whole 128-byte
// rows or by 32-byte K steps inside a row addresses the same TMA-written tile.
//
// K-major, 128B swizzle (what TMA SWIZZLE_128B writes for a [rows][64 x fp16] box): rows are 128 B
// apart, 8-row groups are SBO = 1024 B apart, the 16 B chunk index is XORed with (row & 7).
// Advancing K by 16 elements inside the 64-element swizzle row = +32 B on the start address.
__device__ __forceinline__ uint64_t make_desc_sw128_kmajor(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>(1) << 16;            // LBO (unused for swizzled K-major; 1 like CuTe)
  d |= static_cast<uint64_t>(1024 >> 4) << 32;    // SBO
  d |= static_cast<uint64_t>(1) << 62;            // SWIZZLE_128B
  return d;
}
// K-major, no swizzle ("interleave"): core matrix = 8 rows x 16 B with rows 16 B apart;
// LBO = byte distance between K-adjacent core matrices, SBO = between 8-row groups.
__device__ __forceinline__ uint64_t make_desc_noswz_kmajor(uint32_t smem_addr, uint32_t lbo_bytes,
                                                           uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFF) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFF) << 32;
  return d;
}

// Cheap descriptor arithmetic for issue loops: the high word of a K-major SWIZZLE_128B descriptor is a
// constant, the low word is (addr >> 4) | LBO; stepping K by 16 elements (+32 B) is "+2" on the low word.
constexpr uint32_t kSw128DescHi = (1024u >> 4) | (1u << 30);
__device__ __forceinline__ uint32_t sw128_desc_lo(uint32_t smem_addr) {
  return ((smem_addr & 0x3FFFFu) >> 4) | (1u << 16);
}
__device__ __forceinline__ uint64_t desc_from(uint32_t hi, uint32_t lo) {
  return (static_cast<uint64_t>(hi) << 32) | lo;
}

// One lane of a fully converged warp (TMA issue from a whole producer warp with warp-uniform operands).
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile(
      "{\n"
      ".reg .pred P;\n"
      "elect.sync _|P, 0xffffffff;\n"
      "selp.u32 %0, 1, 0, P;\n"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

// ------------------------------------------------------------------------------------------
// small numeric helpers
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ float2 unpack_half2(uint32_t u) {
  __half2 h = *reinterpret_cast<__half2*>(&u);
  return __half22float2(h);
}

// Division by a run-time constant as a 64-bit multiply + shift (exact for 0 <= n < 2^31): the work-item decode and the
// epilogue's position -> (row, column) split run once per item in every warp; with few-tap 2-D filters an item is short
// enough that the ~25-instruction integer division sequences show up in the issue-slot budget.
struct FastDiv {
  unsigned long long M;
  int s, d;
};
inline FastDiv make_fastdiv(int d) {
  FastDiv f; f.d = d; f.s = 0;
  while ((1ll << f.s) < d) ++f.s;
  const unsigned __int128 one = 1;
  f.M = (unsigned long long)(((one << (32 + f.s)) + (unsigned)d - 1) / (unsigned)d);
  return f;
}
__device__ __forceinline__ int fdiv(int n, const FastDiv& f) {
  return static_cast<int>((static_cast<unsigned long long>(static_cast<unsigned>(n)) * f.M) >> (32 + f.s));
}

}  // namespace b2
