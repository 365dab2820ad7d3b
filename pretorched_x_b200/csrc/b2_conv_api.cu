// b2_conv_api.cu -- C-ABI entry points for the wgmma implicit-GEMM convolution and the dense GEMM,
// plus library-wide error/launch bookkeeping and the CUtensorMap builder.
#include <atomic>
#include <limits.h>
#include <mutex>
#include <stdlib.h>
#include <string.h>

#include "b2_host.h"
#include "b2_igemm.cuh"
#include "b2_densem.cuh"
#include "b2_pgemm.cuh"
#include "b2_slabconv.cuh"
#include "b2_slab_t128.cuh"
#include "b2_tstack.cuh"
#include "b2_stemconv.cuh"

namespace b2 {

// ------------------------------------------------------------------------------------------
// error + launch bookkeeping
// ------------------------------------------------------------------------------------------
static thread_local char g_err[512] = "";
static std::atomic<uint64_t> g_launches{0};

int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}
void count_launch(int n) { g_launches.fetch_add(static_cast<uint64_t>(n), std::memory_order_relaxed); }

static int g_last_kernel = KID_NONE;
static int g_last_info[5] = {0, 0, 0, 0, 0};
void set_last_kernel(int id, int i0, int i1, int i2, int i3, int i4) {
  g_last_kernel = id;
  g_last_info[0] = i0; g_last_info[1] = i1; g_last_info[2] = i2; g_last_info[3] = i3; g_last_info[4] = i4;
}

int require_sm90() {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return set_error(B2_ERR_CUDA, "no CUDA device: %s", cudaGetErrorString(e));
  int major = 0;
  e = cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev);
  if (e != cudaSuccess) return set_error(B2_ERR_CUDA, "cudaDeviceGetAttribute: %s", cudaGetErrorString(e));
  int minor = 0;
  e = cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev);
  if (e != cudaSuccess) return set_error(B2_ERR_CUDA, "cudaDeviceGetAttribute: %s", cudaGetErrorString(e));
  if (major != 9 || minor != 0)
    return set_error(B2_ERR_UNSUPPORTED, "this library targets sm_90a (H100); device is sm_%d%d and there is no fallback",
                     major, minor);
  return B2_OK;
}

int current_device() {
  int dev = 0;
  cudaGetDevice(&dev);
  return dev;
}

int sm_count() {               // per device ordinal (a process may drive several GPUs)
  static std::atomic<int> cache[64];
  const int dev = current_device() & 63;
  int n = cache[dev].load(std::memory_order_relaxed);
  if (n == 0) {
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    cache[dev].store(n, std::memory_order_relaxed);
  }
  return n;
}

// ------------------------------------------------------------------------------------------
// tensor maps
// ------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static PFN_encodeTiled get_encode_tiled() {
  static PFN_encodeTiled fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(p);
  });
  return fn;
}

int make_tmap_2d_f16(CUtensorMap* out, const void* base, uint64_t inner, uint64_t outer, uint64_t pitch_elems,
                     uint32_t box_inner, uint32_t box_outer, bool swizzle128) {
  PFN_encodeTiled enc = get_encode_tiled();
  if (!enc) return set_error(B2_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable (no driver?)");
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) return set_error(B2_ERR_INVALID, "tensor base not 16-byte aligned");
  if ((pitch_elems * 2) % 16 != 0) return set_error(B2_ERR_INVALID, "row pitch %llu elements is not a multiple of 8",
                                                    (unsigned long long)pitch_elems);
  cuuint64_t dims[2] = {inner, outer};
  cuuint64_t strides[1] = {pitch_elems * 2};
  cuuint32_t box[2] = {box_inner, box_outer};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return set_error(B2_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d) inner=%llu outer=%llu pitch=%llu box=%ux%u", (int)r,
                     (unsigned long long)inner, (unsigned long long)outer, (unsigned long long)pitch_elems, box_inner,
                     box_outer);
  return B2_OK;
}

int make_tmap_ndhwc_slab(CUtensorMap* out, const void* base, uint64_t C, uint64_t W, uint64_t H, uint64_t planes,
                         uint32_t box_w, uint32_t box_h, uint32_t stride_hw, uint32_t box_planes) {
  PFN_encodeTiled enc = get_encode_tiled();
  if (!enc) return set_error(B2_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable (no driver?)");
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) return set_error(B2_ERR_INVALID, "tensor base not 16-byte aligned");
  cuuint64_t dims[4] = {C, W, H, planes};
  cuuint64_t strides[3] = {C * 2, W * C * 2, H * W * C * 2};
  // with element strides the box is given in traversed (full-resolution) elements; smem receives every
  // stride_hw-th pixel / row, i.e. box_w x box_h dense pixels
  cuuint32_t box[4] = {64, stride_hw * (box_w - 1) + 1, stride_hw * (box_h - 1) + 1, box_planes};
  cuuint32_t estr[4] = {1, stride_hw, stride_hw, 1};
  if (box[1] > 256 || box[2] > 256) return set_error(B2_ERR_UNSUPPORTED, "slab box %ux%u exceeds the TMA box limit", box[1], box[2]);
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return set_error(B2_ERR_CUDA, "cuTensorMapEncodeTiled(4d) failed (%d) C=%llu W=%llu H=%llu planes=%llu box=%ux%u", (int)r,
                     (unsigned long long)C, (unsigned long long)W, (unsigned long long)H, (unsigned long long)planes, box_w, box_h);
  return B2_OK;
}

int make_tmap_ndhwc_5d(CUtensorMap* out, const void* base, uint64_t C, uint64_t ld, uint64_t W, uint64_t H, uint64_t T,
                       uint64_t N, uint32_t box_w, uint32_t box_h, uint32_t stride_hw) {
  PFN_encodeTiled enc = get_encode_tiled();
  if (!enc) return set_error(B2_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable (no driver?)");
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) return set_error(B2_ERR_INVALID, "tensor base not 16-byte aligned");
  if (ld % 8 != 0 || ld < C) return set_error(B2_ERR_INVALID, "channel pitch %llu must be a multiple of 8 and >= %llu",
                                              (unsigned long long)ld, (unsigned long long)C);
  cuuint64_t dims[5] = {C, W, H, T, N};
  cuuint64_t strides[4] = {ld * 2, W * ld * 2, H * W * ld * 2, T * H * W * ld * 2};
  cuuint32_t box[5] = {64, stride_hw * (box_w - 1) + 1, stride_hw * (box_h - 1) + 1, 1, 1};
  cuuint32_t estr[5] = {1, stride_hw, stride_hw, 1, 1};
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 5, const_cast<void*>(base), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS)
    return set_error(B2_ERR_CUDA, "cuTensorMapEncodeTiled(5d) failed (%d) C=%llu ld=%llu W=%llu H=%llu T=%llu N=%llu", (int)r,
                     (unsigned long long)C, (unsigned long long)ld, (unsigned long long)W, (unsigned long long)H,
                     (unsigned long long)T, (unsigned long long)N);
  return B2_OK;
}

// ------------------------------------------------------------------------------------------
// slab convolution launcher (stride 1 or 2, in-plane padding from 0 to "same")
// ------------------------------------------------------------------------------------------
static int g_conv_algo = 0;   // 0 auto, 1 force gather (debug / A-B comparisons)
static int g_slab_wide = -1;       // 1: request 256-column N tiles for channel counts that are multiples of 256 (tuning; they only run
                                   // where MT * 256 fits kSlabAccCols, which the current register budget never allows), otherwise the
                                   // 128-column rule
static int g_slab_force_mt = -1;   // M tiles per slab work item: -1 read B2_SLAB_MT once, 0 cost model, > 0 forced (tuning)

static int slab_naff(int ldy) { return (ldy + 31) / 32 * 32 + 256; }   // chunk reads may run past ldy inside the last N tile

static int slab_rows(int MT, int PW, int reach, int P) {
  int R = 0;
  for (int q0 = 0; q0 < P; q0 += MT * 128) {
    int lo = q0 - reach;
    lo = (lo >= 0) ? lo / PW : -((-lo + PW - 1) / PW);
    const int hi = (q0 + MT * 128 - 1 + reach) / PW;
    R = (hi - lo + 1) > R ? (hi - lo + 1) : R;
  }
  return R;
}

// Fills the geometry part of SlabParams (sub-image / tap tables).  Returns false when the convolution is not of a
// shape the slab kernel handles.
static bool slab_geometry(const b2_conv_args* a, SlabParams* p, int wc_hint) {
  if (a->mode != B2_CONV_AUTO || a->out_f32) return false;
  if ((a->kt & 1) == 0 || (a->kh & 1) == 0 || (a->kw & 1) == 0) return false;
  // temporal padding "same"; in-plane padding anywhere from "valid" (0) to "same" ((k - 1) / 2)
  if (a->pt != (a->kt - 1) / 2 || a->ph < 0 || a->ph > (a->kh - 1) / 2 || a->pw < 0 || a->pw > (a->kw - 1) / 2) return false;
  if (a->sh != a->sw || (a->sh != 1 && a->sh != 2) || (a->st != 1 && a->st != 2)) return false;
  if (a->kh * a->kw > kSlabMaxTaps) return false;
  const int ss = a->sh;
  if (a->kt * a->kh * a->kw == 1) return false;   // 1x1x1: persistent GEMM (stride 1) / gather kernel (strided): no tap reuse to exploit
  memset(p, 0, sizeof(*p));
  p->T = a->T; p->C = a->C;
  p->To = (a->T + 2 * a->pt - a->kt) / a->st + 1;
  p->Ho = (a->H + 2 * a->ph - a->kh) / ss + 1;
  p->Wo = (a->W + 2 * a->pw - a->kw) / ss + 1;
  p->kt = a->kt; p->khw = a->kh * a->kw; p->st = a->st; p->ss = ss; p->pt = a->pt;
  p->cchunks = (a->C + 63) / 64;
  // tap (dh, dw) reads input (ss*ho + dh - ph, ss*wo + dw - pw) = phase (rh, rw), sub-image pixel (ho + oi, wo + oj)
  int oi[8], rh[8], oj[8], rw[8];
  int min_oj = 0, max_oj = 0, min_oi = 0, max_oi = 0;
  for (int d = 0; d < a->kh; ++d) {
    int v = d - a->ph; rh[d] = ((v % ss) + ss) % ss; oi[d] = (v - rh[d]) / ss;
    if (oi[d] < min_oi) min_oi = oi[d];
    if (oi[d] > max_oi) max_oi = oi[d];
  }
  // Row offsets are taken relative to the middle row of the taps, so that the slab rows an item loads (reach above and below its
  // positions) are not doubled by a one-sided window: below-"same" padding (valid 3x3: rows +0..+2) becomes -1..+1 with the
  // slab starting one sub-image row lower.  Every "same" window is already centred (|min + max| <= 1 truncates to 0).
  const int row_c = (min_oi + max_oi) / 2;
  for (int d = 0; d < a->kw; ++d) {
    int v = d - a->pw; rw[d] = ((v % ss) + ss) % ss; oj[d] = (v - rw[d]) / ss;
    if (oj[d] < min_oj) min_oj = oj[d];
    if (oj[d] > max_oj) max_oj = oj[d];
  }
  p->halo_l = -min_oj;
  // W chunking: rows longer than a TMA box (256 pixels incl. halo) are cut into chunks of WC output columns.  For the
  // temporal remap (kw = 1, "rows" are H*W positions of one frame) a short chunk keeps MT+kt-1 frames in one slab.
  p->WC = p->Wo; p->wchunks = 1;
  const int wc_box = (ss == 1 ? 256 : 128) - p->halo_l - max_oj;                            // TMA box <= 256 traversed pixels
  const int wc_max = (wc_hint > 0 && wc_hint < wc_box) ? wc_hint : wc_box;
  if (p->Wo > wc_max) {
    int best = 0;
    for (int c = wc_max; c >= (wc_max * 3) / 4; --c) if (p->Wo % c == 0) { best = c; break; }   // prefer an exact divisor
    p->WC = best ? best : wc_max;
    p->wchunks = (p->Wo + p->WC - 1) / p->WC;
  }
  p->PW = p->WC + p->halo_l + max_oj;
  p->P = p->Ho * p->PW;
  p->n_sub = 0;
  p->reach = 0;
  for (int ph_ = 0; ph_ < ss; ++ph_)
    for (int pw_ = 0; pw_ < ss; ++pw_) {
      int n = 0;
      const int sidx = p->n_sub;
      for (int dh = 0; dh < a->kh; ++dh)
        for (int dw = 0; dw < a->kw; ++dw)
          if (rh[dh] == ph_ && rw[dw] == pw_) {
            const int off = (oi[dh] - row_c) * p->PW + oj[dw];
            p->sub_off[sidx][n] = (short)off;
            p->sub_tap[sidx][n] = (unsigned char)(dh * a->kw + dw);
            if (off > p->reach) p->reach = off;
            if (-off > p->reach) p->reach = -off;
            ++n;
          }
      if (n == 0) continue;
      p->sub_ntaps[sidx] = n;
      p->sub_h0[sidx] = ph_ + ss * row_c;                  // + ss * r_lo at run time
      p->sub_w0[sidx] = pw_ - ss * p->halo_l;              // slab column 0 = sub-image column -halo_l
      ++p->n_sub;
    }
  if (a->upsample) {
    // 3x3 conv of the nearest-2x upsampled image: output (2h + py, 2w + px) reads low-res rows {h - 1, h} (py = 0) or
    // {h, h + 1} (py = 1), same for columns; the folded 2x2 filters of phase ph are weight taps ph*4 .. ph*4 + 3
    const int s_h0 = p->sub_h0[0], s_w0 = p->sub_w0[0];
    for (int ph = 0; ph < 4; ++ph) {
      const int py = ph >> 1, px = ph & 1;
      for (int ai = 0; ai < 2; ++ai)
        for (int bi = 0; bi < 2; ++bi) {
          const int ro = ai - 1 + py, co = bi - 1 + px;
          p->sub_off[ph][ai * 2 + bi] = (short)(ro * p->PW + co);
          p->sub_tap[ph][ai * 2 + bi] = (unsigned char)(ph * 4 + ai * 2 + bi);
        }
      p->sub_ntaps[ph] = 4; p->sub_h0[ph] = s_h0; p->sub_w0[ph] = s_w0;
    }
    p->khw = 16; p->up = 1; p->n_sub = 1;
  }
  return p->n_sub > 0 && p->PW <= 256;
}

template <int BNT, int TMT, int G = 0>
static int run_slab(int grid, int smem_bytes, const CUtensorMap& tmX, const CUtensorMap& tmB, const SlabParams& p, cudaStream_t stream) {
  if constexpr (G == 0) {
    if (p.ldo) {                    // column-slice output (b2_conv_ndhwc_fprop_slice)
      auto kernel = slabconv_kernel<BNT, TMT, kSlabSlice>;
      B2_OPT_IN_SMEM(kernel, 227 * 1024);
      B2_CHECK_CUDA(launch_pdl(kernel, dim3(grid), dim3(kSlabThreads), smem_bytes, stream, tmX, tmB, p));
      B2_CHECK_LAUNCH("slabconv_kernel");
      return B2_OK;
    }
  }
  auto kernel = slabconv_kernel<BNT, TMT, G>;
  B2_OPT_IN_SMEM(kernel, 227 * 1024);
  B2_CHECK_CUDA(launch_pdl(kernel, dim3(grid), dim3(kSlabThreads), smem_bytes, stream, tmX, tmB, p));
  B2_CHECK_LAUNCH("slabconv_kernel");
  return B2_OK;
}

// BNT = 0: runtime N tile p.bn (set by the caller).  G != 0: grouped convolution (b2_groupconv.cuh) -- N tiles are the K / 64
// channel slices, a.w is the packed grouped filter
// ldo > 0: y is a column slice of rows of pitch ldo; a->ldy is then the slice width (the columns written)
template <int BNT, int G = 0>
static int launch_slab(const b2_conv_args* a, SlabParams& p, int MT, int R, cudaStream_t stream, int ldo = 0) {
  if (BNT) { p.bn = BNT; p.wbytes = BNT * 128; p.accs = BNT; }
  if (G) { p.wbytes = G * 128; p.cchunks = 1; }
  const int BN = p.bn;
  p.R = R;
  p.planes_total = a->N * p.To;
  p.plane_stride = R * p.PW * 128;
  p.slab_bytes = ((R * p.PW * 128 * (p.mp > 1 ? p.mp : 1)) + 1023) / 1024 * 1024;
  p.MT = MT;
  if (MT * BN > kSlabAccCols)
    return set_error(B2_ERR_INVALID, "slab plan MT=%d x N=%d exceeds the %d register accumulator columns", MT, BN, kSlabAccCols);
  if (!BNT && BN != 16 && BN != 32 && BN != 48 && (BN < 144 || BN > kSlabAccCols || BN % 16 != 0))
    return set_error(B2_ERR_INVALID, "slab runtime N tile %d is not one of the compiled widths", BN);
  p.Ncols = a->K;
  p.scale = a->scale; p.shift = a->shift;
  p.residual = reinterpret_cast<const __half*>(a->residual);
  p.ldr = a->ldr;
  p.y = reinterpret_cast<__half*>(a->y);
  p.ldy = a->ldy;
  p.ldo = ldo;
  p.relu = a->relu;
  p.aff_ld = a->aff_ld;
  p.naff = slab_naff(a->ldy);
  p.tiles_n = G ? a->K / 64 : (a->ldy + BN - 1) / BN;
  p.tiles_q = p.mp > 1 ? 1 : (p.P + MT * 128 - 1) / (MT * 128);
  const long long plane_items = p.mp > 1 ? ((long long)a->N * p.To + p.mp - 1) / p.mp : (long long)a->N * p.To;
  const long long items = (long long)p.tiles_n * p.tiles_q * p.wchunks * plane_items * (p.up ? 4 : 1);
  if (items >= (1ll << 31)) return set_error(B2_ERR_INVALID, "slab problem too large");
  p.items_total = (int)items;
  p.fd_tiles_n = make_fastdiv(p.tiles_n); p.fd_tiles_q = make_fastdiv(p.tiles_q); p.fd_wchunks = make_fastdiv(p.wchunks);
  p.fd_To = make_fastdiv(p.To); p.fd_PW = make_fastdiv(p.PW);
  if (a->aff_ld && ((a->aff_ld & 3) || (reinterpret_cast<uintptr_t>(a->scale) & 15) || (reinterpret_cast<uintptr_t>(a->shift) & 15)))
    return set_error(B2_ERR_INVALID, "per-sample scale/shift must be 16-byte aligned with a pitch that is a multiple of 4 floats");
  const int smem_bytes = kSlabSStages * p.slab_bytes + kSlabWStages * p.wbytes + 256 + 2 * slab_naff(a->ldy) * 4 + 1024 +
                         acc_bytes(MT * p.accs);
  CUtensorMap tmX, tmB;
  int rc;
  const int taps = p.up ? 16 : a->kt * a->kh * a->kw;
  if ((rc = make_tmap_ndhwc_slab(&tmX, a->x, (uint64_t)a->C, (uint64_t)a->W, (uint64_t)a->H, (uint64_t)a->N * a->T,
                                 (uint32_t)p.PW, (uint32_t)R, (uint32_t)p.ss, (uint32_t)(p.mp > 1 ? p.mp : 1))) != B2_OK)
    return rc;
  if ((rc = G ? make_tmap_2d_f16(&tmB, a->w, 64, (uint64_t)(a->K / 64) * taps * G, 64, 64, G, true)
              : make_tmap_2d_f16(&tmB, a->w, (uint64_t)taps * a->C, (uint64_t)a->K, (uint64_t)taps * a->C, 64, BN, true)) != B2_OK)
    return rc;
  const int grid = p.items_total < sm_count() ? p.items_total : sm_count();
  if constexpr (G != 0) return run_slab<64, 0, G>(grid, smem_bytes, tmX, tmB, p, stream);
  // the 64-wide tile's MMA form (b2_slabconv.cuh): one N = 128 MMA over a warpgroup's two chunks, otherwise one per chunk.  (MT = 3
  // is never planned outside multi-plane items: its 192-column accumulator tile and two slabs of 384 positions plus halo exceed
  // 227 KB.)
  if constexpr (BNT == 64)
    if (p.mp <= 1 && MT == 2) return run_slab<64, 2>(grid, smem_bytes, tmX, tmB, p, stream);
  return run_slab<BNT, 0>(grid, smem_bytes, tmX, tmB, p, stream);
}

// Picks the N tile (fixed 64 / 128 or runtime), the M tiles per work item and the slab rows for a geometry; *best_mt == 0
// when no configuration fits in shared memory.
// G != 0 (grouped convolution): the N tiles are the K / 64 channel slices, each with a G-row weight stage per tap.
// allow_flex = false: fixed 64 / 128 tiles only (the slice path's retry when the runtime-N tile finds no fit).
// narrow = 32 / 48 (b2_conv_ndhwc_fprop_slice_narrow, a->ldy == narrow): one runtime N tile of exactly the output width.
static double slab_pick_tiles(const b2_conv_args* a, SlabParams& p, int* BN_out, bool* flex_out, int* best_mt_out, int* best_R_out,
                              int G = 0, bool allow_flex = true, int narrow = 0) {
  int BN = (G || a->ldy <= 64) ? 64 : 128;
  const int planes = a->N * p.To;
  int ntn = G ? a->K / 64 : (a->ldy + BN - 1) / BN;
  // Channel counts that tile badly by 128 (144, 288, 576 ... of R(2+1)D) take the runtime-N instance: the fewest
  // tiles of <= 256 columns, each a multiple of 16 wide.
  bool flex = false;
  if (G) {
  } else if (narrow) {
    flex = true; BN = narrow; ntn = 1;
    p.bn = narrow; p.wbytes = (narrow * 128 + 1023) / 1024 * 1024; p.accs = (narrow + 31) / 32 * 32;
  } else if (a->ldy > 128 && allow_flex) {
    const int tn = (a->ldy + 255) / 256;
    const int bn = (((a->ldy + tn - 1) / tn) + 15) / 16 * 16;
    if (bn <= kSlabAccCols && ((long long)bn * tn * 21 <= (long long)ntn * 128 * 20 || (g_slab_wide == 1 && a->ldy % 256 == 0))) {
      flex = true; BN = bn; ntn = tn;
      p.bn = bn; p.wbytes = (bn * 128 + 1023) / 1024 * 1024; p.accs = (bn + 31) / 32 * 32;
    }
  } else if (a->ldy <= 16) {
    // a handful of output channels (the generator's RGB head): the narrowest MMA (N = 16) instead of a 64-wide tile
    // that is 95% padding -- the A operand still streams through shared memory once per tap, so this saves a third
    flex = true; BN = 16; ntn = 1;
    p.bn = 16; p.wbytes = 2048; p.accs = 32;
  }
  const int acc_stride = flex ? p.accs : BN;
  const int w_stage = G ? G * 128 : flex ? p.wbytes : BN * 128;
  // Pick the M tiles per work item from a cycle model of one SM's share: rounds of items x the slower of the MMA
  // stream and the slab/weight loads (the epilogue of an item overlaps the next item's MMAs).  MT * N is bounded by the
  // consumers' register accumulators (kSlabAccCols).  (Model constants:
  // a 128xNx16 MMA retires in ~40 + N/2 cycles, TMA delivers ~48 B/cycle/SM out of L2; not re-fitted on H100.)
  int best_mt = 0, best_R = 0;
  double best_cost = 0.0;
  int& force_mt = g_slab_force_mt;
  if (force_mt < 0) { const char* e = getenv("B2_SLAB_MT"); force_mt = e ? atoi(e) : 0; }   // debug / tuning only
  int ksteps = 0;
  for (int cc = 0; cc < p.cchunks; ++cc) { const int k = (a->C - cc * 64 + 15) / 16; ksteps += k > 4 ? 4 : k; }
  int taps_hw = 0;
  for (int sidx = 0; sidx < p.n_sub; ++sidx) taps_hw += p.sub_ntaps[sidx];
  // planes of at most one M tile whose temporal taps do not differ from plane to plane: the MT accumulators of an item are MT
  // consecutive PLANES (SlabParams::mp), see b2_slabconv.cuh
  static int mp_env = -1;
  if (mp_env < 0) { const char* e = getenv("B2_SLAB_MP"); mp_env = (e && e[0] == '0') ? 0 : 1; }
  const bool mp_ok = mp_env && p.P <= 128 && (a->kt == 1 || a->T == 1) && p.ss == 1 && !p.up && p.wchunks == 1 && planes > 1 &&
                     !a->aff_ld;      // (a per-sample affine is read once per item: its tiles must belong to one image)
  p.mp = 0;
  for (int MT = 4; MT >= 1; --MT) {
    if (force_mt > 0 && MT != force_mt && MT != 1) continue;
    if (MT * BN > kSlabAccCols) continue;
    // (multi-plane: rows one plane's positions and taps can touch -- slab_rows assumes a full 128-position tile)
    const int R = mp_ok ? (p.P - 1 + p.reach) / p.PW + (p.reach + p.PW - 1) / p.PW + 1 : slab_rows(MT, p.PW, p.reach, p.P);
    if (p.ss * (R - 1) + 1 > 256) continue;
    const long long slab_b = ((long long)R * p.PW * 128 * (mp_ok ? MT : 1) + 1023) / 1024 * 1024;
    const long long smem_one = 2ll * slab_b + kSlabWStages * w_stage + 256 + 2 * slab_naff(a->ldy) * 4 + 1024;
    if (smem_one + acc_bytes(MT * acc_stride) > 227 * 1024) continue;
    const long long tq = mp_ok ? 1 : (p.P + MT * 128 - 1) / (MT * 128);
    const long long items = (long long)ntn * tq * (mp_ok ? (planes + MT - 1) / MT : planes) * p.wchunks * (p.up ? 4 : 1);
    const double rounds = (double)((items + sm_count() - 1) / sm_count());
    const double tiles_per_item = mp_ok ? (double)MT : (double)((p.P + 127) / 128) / (double)tq;   // average (the last item of a plane is short)
    const double mma = tiles_per_item * p.kt * taps_hw * ksteps * (40.0 + 0.5 * BN);
    // small planes: every SM streams the whole filter per item at the same time, and what bounds that is the aggregate L2 -> SM rate
    // (modelled as 26 B/cycle/SM), not one SM's TMA rate
    const double bpc = mp_ok ? 26.0 : 48.0;
    const double load = (double)p.kt * p.n_sub * p.cchunks * slab_b / bpc + (double)p.kt * taps_hw * p.cchunks * w_stage / bpc;
    const double cost = rounds * ((mma > load ? mma : load) + 1500.0);
    if (force_mt == -1) {                                   // previous rule (A/B): largest power-of-two MT with >= 2 rounds of items
      if ((MT & (MT - 1)) != 0 && !flex) continue;
      best_mt = MT; best_R = R;
      if (items >= 2 * sm_count()) break;
      continue;
    }
    if (best_mt == 0 || cost < best_cost || (force_mt > 0 && MT == force_mt)) { best_mt = MT; best_R = R; best_cost = cost; }
    if (force_mt > 0 && MT == force_mt) break;
  }
  if (mp_ok && best_mt >= 2 && best_mt < 4 && force_mt <= 0 && 4 * BN <= kSlabAccCols) {
    // four planes per item share each weight tile twice as often as two, as long as a full wave of items remains
    const int R4 = (p.P - 1 + p.reach) / p.PW + (p.reach + p.PW - 1) / p.PW + 1;
    const long long slab4 = ((long long)R4 * p.PW * 128 * 4 + 1023) / 1024 * 1024;
    const long long items4 = (long long)ntn * ((planes + 3) / 4);
    if (2ll * slab4 + kSlabWStages * w_stage + 256 + 2 * slab_naff(a->ldy) * 4 + 1024 + acc_bytes(4 * acc_stride) <= 227 * 1024 &&
        items4 >= sm_count()) { best_mt = 4; best_R = R4; }
  }
  p.mp = (mp_ok && best_mt > 1) ? best_mt : 0;
  *BN_out = BN; *flex_out = flex; *best_mt_out = best_mt; *best_R_out = best_R;
  return best_cost;
}

// The slab kernel's plan of a convolution (a: after the temporal remap).  Returns false when the kernel does not apply or no tiling
// fits in shared memory.
struct SlabChoice {
  SlabParams p;
  int BN, MT, R;
  bool flex;
};
static bool slab_choose(const b2_conv_args* a, int wc_hint, int G, int ldo, SlabChoice* c, int narrow = 0) {
  // W chunking candidates: the default (whole rows, or <= 256-pixel chunks) and narrower chunks.  Narrow chunks make the
  // slab of a work item shorter, which (a) lets 256-pixel rows fit the two slab stages at all and (b) admits more M tiles
  // per item for wide images -- with few-tap 2-D filters the per-item costs (decode, epilogue set-up, slab latency) are
  // what the cycle model trades against the extra halo columns.  The cheapest modelled configuration wins.
  const int wc_try[3] = {wc_hint, 128, 64};
  int best_mt = 0;
  double best_cost = 0.0;
  for (int attempt = 0; attempt < 3; ++attempt) {
    if (attempt > 0 && (wc_hint > 0 || wc_try[attempt] >= a->W)) continue;
    SlabParams q;
    if (!slab_geometry(a, &q, wc_try[attempt])) { if (attempt == 0) return false; else continue; }
    if (attempt > 0 && q.wchunks == 1) continue;              // same geometry as the default
    if (g_conv_algo == 2 && q.ss != 1 && !G) return false;    // debug: strided convs through the gather kernel
    if (G) q.cchunks = 1;                                     // an item reads its own 64-channel slice only
    int bn_c = 0, mt_c = 0, r_c = 0;
    bool flex_c = false;
    const SlabParams q0 = q;
    double cost = slab_pick_tiles(a, q, &bn_c, &flex_c, &mt_c, &r_c, G, true, narrow);
    if (mt_c == 0 && ldo && flex_c && !narrow) {
      // a slice has no other kernel to fall back on: when the wide runtime-N tile does not fit, take 128-column tiles
      q = q0;
      cost = slab_pick_tiles(a, q, &bn_c, &flex_c, &mt_c, &r_c, G, false);
    }
    if (mt_c == 0) continue;
    if (best_mt == 0 || cost < best_cost) { c->p = q; c->BN = bn_c; c->flex = flex_c; c->MT = best_mt = mt_c; c->R = r_c; best_cost = cost; }
  }
  return best_mt != 0;
}

// ------------------------------------------------------------------------------------------
// 128- and 64-wide slab tiles as the transposed product (b2_slab_t128.cuh)
// ------------------------------------------------------------------------------------------
static int g_slab_t128 = -1;       // -1 the rule (slab_t128_wanted), 0 never, 1 wherever the form applies (tests, A/B sweeps)
static int g_slab_t64 = -1;        // the same for the 64-wide form (slab_t64_wanted)
static const int kT128Widths[3] = {216, 224, 256};   // compiled item widths NP of the 128-wide form
static const int kT64Width = 168;  // positions per warpgroup of the 64-wide form: 20 half-items cover a 56 x 58 padded plane

struct TPlan {
  SlabParams p;                    // geometry (slab_geometry) + qitem
  int np, rows, R, items, smem;    // rows: whole output rows per item (128-wide form), 0 for the 64-wide form
};

static int slab_t_smem(int BN, int slab_bytes, int np, int ldy) {
  return kSlabSStages * slab_bytes + kSlabWStages * BN * 128 + np * 256 + 256 + 2 * slab_naff(ldy) * 4 + 1024;
}

// Whether the BN-wide form takes the convolution at all, and its plan.  BN = 128: the fewest row groups per plane whose padded
// positions fit 256, and the narrowest compiled width that holds one.  BN = 64: items of 2 NP consecutive positions.  Then the slab
// rows that every item's MMA columns and taps reach.
static bool slab_t_geometry(const b2_conv_args* a, int BN, TPlan* t) {
  if (a->upsample || a->aff_ld || a->residual || a->y2 || a->residual_up || a->residual_pre || a->in_scale || a->mask) return false;
  if (a->kh != 3 || a->kw != 3 || (a->kt != 1 && a->kt != 3)) return false;
  if (a->C % 64 != 0 || (BN == 128 ? a->K % 128 != 0 : a->ldy > 64)) return false;
  SlabParams& p = t->p;
  if (!slab_geometry(a, &p, 0) || p.wchunks != 1 || p.up) return false;
  int groups, span;                // position groups per plane, MMA columns from each item start
  if (BN == 128) {
    const int max_rows = 256 / p.PW;
    if (max_rows < 1) return false;
    groups = (p.Ho + max_rows - 1) / max_rows;
    t->rows = (p.Ho + groups - 1) / groups;
    p.qitem = t->rows * p.PW;
    t->np = 0;
    for (int np : kT128Widths)
      if (np >= p.qitem) { t->np = np; break; }
    if (t->np == 0) return false;
    span = t->np;
  } else {
    t->np = kT64Width;
    t->rows = 0;
    p.qitem = span = 2 * t->np;
    groups = (p.P + p.qitem - 1) / p.qitem;
  }
  int R = 0;
  for (int q0 = 0; q0 < p.P; q0 += p.qitem) {
    int lo = q0 - p.reach;
    lo = (lo >= 0) ? lo / p.PW : -((-lo + p.PW - 1) / p.PW);
    const int hi = (q0 + span - 1 + p.reach) / p.PW;
    R = (hi - lo + 1) > R ? (hi - lo + 1) : R;
  }
  if (p.ss * (R - 1) + 1 > 256) return false;
  t->R = R;
  p.R = R;
  p.slab_bytes = (R * p.PW * 128 + 1023) / 1024 * 1024;
  p.MT = 1;
  p.tiles_n = (a->ldy + BN - 1) / BN;
  p.tiles_q = groups;
  const long long items = (long long)p.tiles_n * groups * a->N * p.To;
  if (items >= (1ll << 31)) return false;
  t->items = (int)items;
  t->smem = slab_t_smem(BN, p.slab_bytes, t->np, a->ldy);
  return t->smem <= 227 * 1024;
}

// Items the slab kernel's plan c runs for the convolution
static long long slab_items(const b2_conv_args* a, const SlabChoice& c) {
  const SlabParams& p = c.p;
  const long long planes = p.mp > 1 ? ((long long)a->N * p.To + p.mp - 1) / p.mp : (long long)a->N * p.To;
  const long long tq = p.mp > 1 ? 1 : (p.P + c.MT * 128 - 1) / (c.MT * 128);
  return (long long)((a->ldy + c.BN - 1) / c.BN) * tq * p.wchunks * planes * (p.up ? 4 : 1);
}

// The rule: an item of the form runs NP / 128 times the MMA columns of a one-tile slab item and there are fewer of them, so it
// is taken where rounds of items x MMA columns per item -- the critical path of the persistent grid -- is not longer than the slab
// kernel's plan: ceil(items / SMs) * NP / 128 <= ceil(slab items / SMs) * MT.  At small sizes halving the items idles SMs and the
// rule declines.  A forced slab plan (set_slab_mt, set_slab_wide) and multi-plane slab items stay on the slab kernel.
static bool slab_t128_wanted(const b2_conv_args* a, const SlabChoice& c, TPlan* t) {
  if (g_slab_t128 == 0 || !slab_t_geometry(a, 128, t)) return false;
  if (g_slab_t128 == 1) return true;
  if (g_slab_force_mt != 0 || g_slab_wide == 1 || c.p.mp > 1) return false;
  const long long sms = sm_count();
  const long long cur = slab_items(a, c);
  return ((t->items + sms - 1) / sms) * t->np <= ((cur + sms - 1) / sms) * c.MT * 128;
}

// The 64-wide form's rule.  Its items hold 2 NP = 336 positions against the slab kernel's MT * 128, and one of its MMA columns
// costs less: a weight stage serves 1.3x the positions, and the consumers store fp16 through stmatrix instead of fp32 scalars into an
// accumulator tile.  Measured per column (kernel time / (rounds of items x columns per item), H100 SXM at 700 W, 1980 MHz) on 64 ->
// 64 3x3 convolutions over 56 x 56 planes, the form's column cost 0.64 - 0.75 of the slab kernel's at 2 - 32 clips of 8 frames and
// 32 - 256 images, so it is taken where rounds x columns x kT64ColCost % is not longer than the slab plan's rounds x columns.  Below
// kT64MinItemsPerSm items per SM (fewer than ~26 planes of 56 x 56) the slab kernel keeps the convolution: there a launch is a
// round or two of items, and the form's larger items gain at most a few microseconds.  A forced slab plan and multi-plane slab
// items stay on the slab kernel.
static const int kT64ColCost = 75;
static const int kT64MinItemsPerSm = 2;
static bool slab_t64_wanted(const b2_conv_args* a, const SlabChoice& c, TPlan* t) {
  if (g_slab_t64 == 0 || !slab_t_geometry(a, 64, t)) return false;
  if (g_slab_t64 == 1) return true;
  if (g_slab_force_mt != 0 || g_slab_wide == 1 || c.p.mp > 1) return false;
  const long long sms = sm_count();
  const long long cur = slab_items(a, c);
  return t->items >= kT64MinItemsPerSm * sms &&
         ((t->items + sms - 1) / sms) * 2 * t->np * kT64ColCost <= ((cur + sms - 1) / sms) * c.MT * 128 * 100;
}

template <int BN, int NP>
static int run_slab_t(int grid, int smem_bytes, const CUtensorMap& tmX, const CUtensorMap& tmB, const SlabParams& p,
                      cudaStream_t stream) {
  B2_OPT_IN_SMEM((slab_t_kernel<BN, NP>), 227 * 1024);
  B2_CHECK_CUDA(launch_pdl(slab_t_kernel<BN, NP>, dim3(grid), dim3(kSlabThreads), smem_bytes, stream, tmX, tmB, p));
  B2_CHECK_LAUNCH("slab_t_kernel");
  return B2_OK;
}

template <int BN>
static int launch_slab_t(const b2_conv_args* a, TPlan& t, cudaStream_t stream) {
  SlabParams& p = t.p;
  p.bn = BN; p.wbytes = BN * 128; p.accs = BN;
  p.mp = 0;
  p.planes_total = a->N * p.To;
  p.plane_stride = p.R * p.PW * 128;
  p.Ncols = a->K;
  p.scale = a->scale; p.shift = a->shift;
  p.residual = nullptr; p.ldr = 0;
  p.y = reinterpret_cast<__half*>(a->y);
  p.ldy = a->ldy;
  p.ldo = 0;
  p.relu = a->relu;
  p.aff_ld = 0;
  p.naff = slab_naff(a->ldy);
  p.items_total = t.items;
  p.fd_tiles_n = make_fastdiv(p.tiles_n); p.fd_tiles_q = make_fastdiv(p.tiles_q); p.fd_wchunks = make_fastdiv(p.wchunks);
  p.fd_To = make_fastdiv(p.To); p.fd_PW = make_fastdiv(p.PW);
  CUtensorMap tmX, tmB;
  int rc;
  const int taps = a->kt * a->kh * a->kw;
  if ((rc = make_tmap_ndhwc_slab(&tmX, a->x, (uint64_t)a->C, (uint64_t)a->W, (uint64_t)a->H, (uint64_t)a->N * a->T, (uint32_t)p.PW,
                                 (uint32_t)t.R, (uint32_t)p.ss)) != B2_OK)
    return rc;
  if ((rc = make_tmap_2d_f16(&tmB, a->w, (uint64_t)taps * a->C, (uint64_t)a->K, (uint64_t)taps * a->C, 64, BN, true)) != B2_OK)
    return rc;
  const int grid = p.items_total < sm_count() ? p.items_total : sm_count();
  switch (BN * 1000 + t.np) {
    case 128216: return run_slab_t<128, 216>(grid, t.smem, tmX, tmB, p, stream);
    case 128224: return run_slab_t<128, 224>(grid, t.smem, tmX, tmB, p, stream);
    case 128256: return run_slab_t<128, 256>(grid, t.smem, tmX, tmB, p, stream);
    case 64168: return run_slab_t<64, 168>(grid, t.smem, tmX, tmB, p, stream);
    default: return set_error(B2_ERR_INVALID, "slab item width %d is not one of the compiled widths of the %d-wide form", t.np, BN);
  }
}

// returns 1 when the slab kernel (or one of its transposed forms) took the convolution, 0 when it does not apply, <0 on error
// G != 0: grouped convolution inside the contract of b2_conv_grouped_ndhwc_fprop (3x3 in plane, so never the temporal remap)
// ldo > 0: column-slice output, see launch_slab
// narrow: see slab_pick_tiles
static int try_slab(const b2_conv_args* a_in, cudaStream_t stream, int G = 0, int ldo = 0, int narrow = 0) {
  if (g_conv_algo == 1 && !G && !ldo) return 0;
  b2_conv_args remap = *a_in;
  const b2_conv_args* a = a_in;
  int wc_hint = 0;
  if (a_in->kt > 1 && a_in->kh == 1 && a_in->kw == 1 && a_in->st == 1 && a_in->sh == 1 && a_in->sw == 1 &&
      a_in->ph == 0 && a_in->pw == 0 && g_conv_algo != 3) {
    // (kt,1,1) over [N][T][H][W] == (1,kt,1) over N images of T rows x (H*W) columns
    remap.T = 1; remap.H = a_in->T; remap.W = a_in->H * a_in->W;
    remap.kt = 1; remap.kh = a_in->kt; remap.kw = 1;
    remap.pt = 0; remap.ph = a_in->pt; remap.pw = 0;
    a = &remap;
    wc_hint = 64;
  }
  SlabChoice c;
  if (!slab_choose(a, wc_hint, G, ldo, &c, narrow)) return 0;
  if (!G && !ldo) {
    TPlan t;
    if (slab_t128_wanted(a, c, &t)) {
      const int rc = launch_slab_t<128>(a, t, stream);
      if (rc == B2_OK) set_last_kernel(KID_SLAB_T128, t.np, t.rows, 128, t.p.ss, t.R);
      return rc == B2_OK ? 1 : rc;
    }
    if (slab_t64_wanted(a, c, &t)) {
      const int rc = launch_slab_t<64>(a, t, stream);
      if (rc == B2_OK) set_last_kernel(KID_SLAB_T64, t.np, t.items, t.R);
      return rc == B2_OK ? 1 : rc;
    }
  }
  SlabParams& p = c.p;
  const int BN = c.BN, best_mt = c.MT, best_R = c.R;
  const bool flex = c.flex;
  int rc = G == 16 ? launch_slab<64, 16>(a, p, best_mt, best_R, stream)
           : G == 32 ? launch_slab<64, 32>(a, p, best_mt, best_R, stream)
           : flex ? launch_slab<0>(a, p, best_mt, best_R, stream, ldo)
                  : (BN == 64) ? launch_slab<64>(a, p, best_mt, best_R, stream, ldo) : launch_slab<128>(a, p, best_mt, best_R, stream, ldo);
  if (rc == B2_OK && G) set_last_kernel(KID_GROUPCONV, G, best_mt, p.mp, p.wchunks);
  else if (rc == B2_OK && ldo) set_last_kernel(KID_SLAB_SLICE, BN, best_mt, flex, p.wchunks);
  else if (rc == B2_OK) set_last_kernel(KID_SLAB, BN, best_mt, flex, p.wchunks, a != a_in);
  return rc == B2_OK ? 1 : rc;
}


// ------------------------------------------------------------------------------------------
// temporal stack kernel (b2_tstack.cuh): (kt,1,1) stride-1 "same" convolutions with <= 64 output channels, resident filter
// ------------------------------------------------------------------------------------------
static int g_last_conv_path = 0;   // which launcher took the last b2_conv_ndhwc_fprop call: 0 generic, 1 tstack (tests pin the dispatch)
static int g_tstack = -2;     // -2: read B2_TSTACK once (0 = never); -1 rule below, 0 never, 1 whenever the shape is eligible (tests / sweeps)
// Shape test + work decomposition (host only).  Returns false when the kernel does not take the convolution.
static bool tstack_plan(const b2_conv_args* a, TstackParams* out, size_t* smem_out) {
  if (a->mode != B2_CONV_AUTO || a->out_f32 || a->upsample || a->aff_ld || a->y2 || a->residual_up || a->residual_pre || a->in_scale) return false;
  if (a->kh != 1 || a->kw != 1 || a->kt < 3 || !(a->kt & 1) || a->st != 1 || a->sh != 1 || a->sw != 1 || a->pt != a->kt / 2 || a->ph != 0 ||
      a->pw != 0 || a->ldy > 64 || a->T < 2)
    return false;
  const int cchunks = (a->C + 63) / 64;
  const long long wbytes = (long long)cchunks * a->kt * kTkWBlock;
  if (wbytes > 112 * 1024) return false;                     // the filter must stay resident next to the A ring and the accumulators
  const long long HW = (long long)a->H * a->W;
  if (HW >= (1ll << 24)) return false;
  TstackParams p;
  p.T = a->T; p.HW = (int)HW; p.C = a->C;
  p.kt = a->kt; p.pt = a->pt;
  p.cchunks = cchunks;
  p.groups = (a->T + kTkG - 1) / kTkG;
  p.tiles_q = (int)((HW + 127) / 128);
  const long long items = (long long)a->N * p.groups * p.tiles_q;
  if (items >= (1ll << 31)) return false;
  // Below one work item per SM the frames-as-rows form of the slab kernel (more, smaller items) keeps more SMs busy.
  if (g_tstack < 0 && items < sm_count()) return false;
  p.items_total = (int)items;
  p.Ncols = a->K; p.ldy = a->ldy; p.ldr = a->ldr; p.relu = a->relu;
  p.scale = a->scale; p.shift = a->shift;
  p.residual = reinterpret_cast<const __half*>(a->residual);
  p.y = reinterpret_cast<__half*>(a->y);
  p.fd_tiles_q = make_fastdiv(p.tiles_q); p.fd_groups = make_fastdiv(p.groups);
  *out = p;
  *smem_out = 1024 + (size_t)kTkStages * kTkABytes + (size_t)wbytes + 128 + 512 + acc_bytes(kTkSetCols);
  return true;
}

static int try_tstack(const b2_conv_args* a, cudaStream_t stream) {
  if (g_tstack == -2) { const char* e = getenv("B2_TSTACK"); g_tstack = (e && e[0] == '0') ? 0 : -1; }
  if (g_tstack == 0 || g_conv_algo != 0) return 0;
  TstackParams p;
  size_t smem = 0;
  if (!tstack_plan(a, &p, &smem)) return 0;
  const long long HW = p.HW;
  B2_OPT_IN_SMEM(tstack_kernel, 227 * 1024);
  CUtensorMap tmX, tmB;
  int rc;
  if ((rc = make_tmap_ndhwc_slab(&tmX, a->x, (uint64_t)a->C, (uint64_t)HW, 1, (uint64_t)a->N * a->T, 128u, 1u, 1u)) != B2_OK) return rc;
  if ((rc = make_tmap_2d_f16(&tmB, a->w, (uint64_t)a->kt * a->C, (uint64_t)a->K, (uint64_t)a->kt * a->C, 64, 64, true)) != B2_OK) return rc;
  const int grid = p.items_total < sm_count() ? p.items_total : sm_count();
  B2_CHECK_CUDA(launch_pdl(tstack_kernel, dim3(grid), dim3(kTkThreads), smem, stream, tmX, tmB, p));
  B2_CHECK_LAUNCH("tstack_kernel");
  g_last_conv_path = 1;
  set_last_kernel(KID_TSTACK);
  return 1;
}

// ------------------------------------------------------------------------------------------
// stem convolution launcher (Toeplitz-descriptor kernel)
// ------------------------------------------------------------------------------------------
// Instance of the BN = 64 stem: -2 = not read yet, -1 = the rule; 2 / 4 = forced two- / four-row instance with positions along
// M, kStemForceT = the transposed four-row instance (each only where eligible).  B2_STEM_ROWS=2 / 4 / 4t in the environment (read
// once) or b2_debug_set_stem_rows() force an instance, for A/B comparisons.
constexpr int kStemForceT = 4 | 16;
static int g_stem_rows = -2;
static int g_last_stem_rows = 0;
template <int BN, int G, bool kT>
static int launch_stem_g(cudaStream_t stream, const StemParams& p, const CUtensorMap& tmX, int smem_bytes) {
  B2_OPT_IN_SMEM((stemconv_kernel<BN, G, false, kT>), 227 * 1024);
  if constexpr (G != 4) B2_OPT_IN_SMEM((stemconv_kernel<BN, G, true, false>), 227 * 1024);
  const int grid = p.items_total < sm_count() ? p.items_total : sm_count();
  if constexpr (G != 4)
    if (p.nstages == 1) {
      B2_CHECK_CUDA(launch_pdl(stemconv_kernel<BN, G, true, false>, dim3(grid), dim3(stem_threads(G)), smem_bytes, stream, tmX, p));
      B2_CHECK_LAUNCH("stemconv_kernel");
      return B2_OK;
    }
  B2_CHECK_CUDA(launch_pdl(stemconv_kernel<BN, G, false, kT>, dim3(grid), dim3(stem_threads(G)), smem_bytes, stream, tmX, p));
  B2_CHECK_LAUNCH("stemconv_kernel");
  return B2_OK;
}

// Which instance a stem runs with: returns G, *transposed for the transposed four-row one.  G = 4 is eligible at BN = 64 outside
// pair mode when its slab (2 * 3 + kh rows) and weight image leave room for three ring stages next to its staging tile, i.e.
// kh <= 7; taller filters keep G = 2 and its deeper ring.  The rule takes it for temporal filters (kt > 1): on an H100 the 7x7x7
// stems of resnet3d50 / nonlocal50 run 15-17 % faster than with G = 2.  A 2-D stem (kt == 1, resnet18) has one tap per item, so the
// item-end drain and the single staging tile are exposed: G = 4 measured 16 % slower there and it keeps G = 2.  Where G = 4 runs
// and a row has at most kStemTileT = 112 output columns, the transposed instance computes it (one N = 112 MMA per output row
// instead of two 64-row halves of a 128-row tile; 112 / Wo columns of waste instead of 128 / Wo).
static int stem_rows_for(int BN, int kt, int kh, int Wo, bool pair, bool* transposed) {
  *transposed = false;
  if (BN != 64) return 1;
  if (g_stem_rows == -2) {
    const char* e = getenv("B2_STEM_ROWS");
    g_stem_rows = (e && e[0] == '2') ? 2 : (e && e[0] == '4') ? ((e[1] == 't' || e[1] == 'T') ? kStemForceT : 4) : -1;
  }
  const int stage4 = ((2 * 3 + kh) * kStemPitch + kh * 64 * 64 + 127) / 128 * 128;
  const bool eligible = !pair && (227 * 1024 - stem_tail_bytes(4, 64) - 128) / stage4 >= 3;
  if (!eligible || g_stem_rows == 2) return 2;
  if (g_stem_rows == -1 && kt == 1) return 2;
  *transposed = Wo <= kStemTileT && g_stem_rows != 4;
  return 4;
}

template <int BN>
static int launch_stem(const b2_conv_args* a, cudaStream_t stream) {
  PFN_encodeTiled enc = get_encode_tiled();
  if (!enc) return set_error(B2_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable (no driver?)");
  StemParams p;
  memset(&p, 0, sizeof(p));
  p.T = a->T; p.H = a->H; p.W = a->W;
  p.To = (a->T + 2 * a->pt - a->kt) / a->st + 1;
  p.Ho = (a->H + 2 * a->ph - a->kh) / 2 + 1;
  p.Wo = (a->W + 6 - 7) / 2 + 1;
  p.kt = a->kt; p.kh = a->kh; p.pt = a->pt; p.ph = a->ph;
  // with pt >= kt the first output frames see no input frame at all; the kernel expects every item to have a tap inside the clip
  if (a->pt >= a->kt) return set_error(B2_ERR_UNSUPPORTED, "stem convolution needs temporal padding < kt (got pt=%d, kt=%d)", a->pt, a->kt);
  static int pair_env = -1;
  if (pair_env < 0) { const char* e = getenv("B2_STEM_PAIR"); pair_env = (e && e[0] == '0') ? 0 : 1; }
  p.pair = (pair_env && a->kt == 1 && a->pt == 0 && p.Wo <= 60 && !a->pool_w && a->W <= 120) ? 1 : 0;
  bool transposed = false;
  p.G = stem_rows_for(BN, a->kt, a->kh, p.Wo, p.pair != 0, &transposed);
  p.rows = 2 * (p.G - 1) + a->kh;
  if (p.rows > kStemMaxRows) return set_error(B2_ERR_UNSUPPORTED, "stem kernel height %d too large", a->kh);
  for (int i = 0; i < p.rows; ++i) {
    int g_lo, g_hi, slot;
    stem_row_plan(p.G, a->kh, i, &g_lo, &g_hi, &slot);
    p.row_glo[i] = (signed char)g_lo;
    p.row_ghi[i] = (signed char)g_hi;
    p.row_slot[i] = (signed char)slot;
  }
  p.w_bytes = a->kh * BN * 64;
  p.stage_bytes = ((p.rows * kStemPitch + p.w_bytes) + 127) / 128 * 128;
  const int tail_bytes = stem_tail_bytes(p.G, BN) + 128;        // + alignment of the dynamic shared-memory base
  p.nstages = (227 * 1024 - tail_bytes) / p.stage_bytes;
  if (p.nstages > kStemMaxStages) p.nstages = kStemMaxStages;
  if (p.nstages < 1) return set_error(B2_ERR_UNSUPPORTED, "stem slab does not fit in shared memory (kh=%d)", a->kh);
  p.Ncols = a->K;
  p.ntiles_n = (a->ldy + BN - 1) / BN;
  if (p.ntiles_n * BN > 256) return set_error(B2_ERR_UNSUPPORTED, "stem convolution supports at most 256 output channels");
  p.tiles_w = (p.Wo + kStemTileW - 1) / kStemTileW;
  p.tiles_h = (p.Ho + p.G - 1) / p.G;
  p.planes_total = a->N * p.To;
  const long long plane_items = p.pair ? (p.planes_total + 1) / 2 : p.planes_total;
  const long long items = (long long)p.tiles_w * p.tiles_h * p.ntiles_n * plane_items;
  if (items >= (1ll << 31)) return set_error(B2_ERR_INVALID, "stem problem too large");
  p.items_total = (int)items;
  p.wimg = reinterpret_cast<const __half*>(a->w);
  p.scale = a->scale; p.shift = a->shift;
  p.y = reinterpret_cast<__half*>(a->y);
  p.ldy = a->ldy;
  p.relu = a->relu;
  p.pool_w = a->pool_w; p.Wp = (p.Wo - 1) / 2 + 1;
  if (a->pool_w && (!a->relu || p.tiles_w != 1))
    return set_error(B2_ERR_UNSUPPORTED, "fused W pooling needs ReLU and an output row of at most %d columns (got %d)", kStemTileW, p.Wo);
  const int smem_bytes = p.nstages * p.stage_bytes + tail_bytes;
  // input viewed as 8-byte pixels (W, H, N*T); box (256, rows, 1); no swizzle -> dense 2 KB rows in smem
  CUtensorMap tmX;
  cuuint64_t dims[3] = {(cuuint64_t)a->W, (cuuint64_t)a->H, (cuuint64_t)a->N * a->T};
  cuuint64_t strides[2] = {(cuuint64_t)a->W * 8, (cuuint64_t)a->H * a->W * 8};
  cuuint32_t box[3] = {(cuuint32_t)kStemRowPx, (cuuint32_t)p.rows, 1};
  if (p.pair) {      // (W, plane, H): box (128 pixels, 2 planes, rows) -> smem [row][plane][1024 B]
    dims[1] = (cuuint64_t)a->N * a->T; dims[2] = (cuuint64_t)a->H;
    strides[0] = (cuuint64_t)a->H * a->W * 8; strides[1] = (cuuint64_t)a->W * 8;
    box[0] = 128; box[1] = 2; box[2] = (cuuint32_t)p.rows;
  }
  cuuint32_t estr[3] = {1, 1, 1};
  CUresult r = enc(&tmX, CU_TENSOR_MAP_DATA_TYPE_UINT64, 3, const_cast<void*>(a->x), dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return set_error(B2_ERR_CUDA, "cuTensorMapEncodeTiled(stem) failed (%d)", (int)r);
  g_last_stem_rows = p.G;
  set_last_kernel(KID_STEM, p.G, transposed);
  if constexpr (BN == 128) return launch_stem_g<128, 1, false>(stream, p, tmX, smem_bytes);
  else if (p.G == 2) return launch_stem_g<64, 2, false>(stream, p, tmX, smem_bytes);
  else return transposed ? launch_stem_g<64, 4, true>(stream, p, tmX, smem_bytes) : launch_stem_g<64, 4, false>(stream, p, tmX, smem_bytes);
}

// ------------------------------------------------------------------------------------------
// launcher shared by conv and gemm
// ------------------------------------------------------------------------------------------
struct IgemmLaunch {
  IgemmParams p;
  // optional second operand pair (persistent GEMM only): D += A2[M][k2] . B2[N][k2]^T
  const void* a2 = nullptr; int lda2 = 0; const void* w2 = nullptr; int ldb2 = 0; int k2 = 0;
  const void* a_mat;      // AMODE_TMA: A as [M][lda]
  int lda;
  int a_cols;             // logical K extent of A (columns readable)
  const void* w;          // B as [Ncols][ldb]
  int ldb;
  int b_cols;             // logical K extent of B
};

template <int BN, int MASK>
static int launch_igemm(const IgemmLaunch& L, cudaStream_t stream) {
  using S = IgemmSmem<BN>;
  B2_OPT_IN_SMEM((igemm_kernel<BN, MASK>), S::kTotalBytes);
  const IgemmParams& p = L.p;
  CUtensorMap tmA, tmB, tmC, tmR;
  memset(&tmA, 0, sizeof(tmA)); memset(&tmC, 0, sizeof(tmC)); memset(&tmR, 0, sizeof(tmR));
  int rc;
  if ((rc = make_tmap_2d_f16(&tmB, L.w, (uint64_t)L.b_cols, (uint64_t)p.Ncols, (uint64_t)L.ldb, kBK, BN, true)) != B2_OK)
    return rc;
  if (p.amode == AMODE_TMA) {
    if ((rc = make_tmap_2d_f16(&tmA, L.a_mat, (uint64_t)L.a_cols, (uint64_t)p.M_total, (uint64_t)L.lda, kBK, kBM, true)) != B2_OK)
      return rc;
  } else {
    tmA = tmB;
  }
  if (p.epi == EPI_TMA_F16) {
    if ((rc = make_tmap_2d_f16(&tmC, p.y, (uint64_t)p.ldy, (uint64_t)p.M_total, (uint64_t)p.ldy, 64, kBM, true)) != B2_OK)
      return rc;
    if (p.residual) {
      // column extent Ncols, not ldr: residual columns >= K are never read (TMA zero-fills them), so y's padding stays zero
      if ((rc = make_tmap_2d_f16(&tmR, p.residual, (uint64_t)p.Ncols, (uint64_t)p.M_total, (uint64_t)p.ldr, 64, kBM, true)) != B2_OK)
        return rc;
    } else {
      tmR = tmC;
    }
  } else {
    tmC = tmB; tmR = tmB;
  }
  dim3 grid((p.epi == EPI_TMA_F16 ? (p.ldy + BN - 1) / BN : (p.Ncols + BN - 1) / BN), (p.M_total + kBM - 1) / kBM, 1);
  B2_CHECK_CUDA(launch_pdl(igemm_kernel<BN, MASK>, grid, dim3(kThreads), S::kTotalBytes, stream, tmA, tmB, tmC, tmR, p));
  B2_CHECK_LAUNCH("igemm_kernel");
  set_last_kernel(KID_IGEMM, BN, MASK);
  return B2_OK;
}


// ------------------------------------------------------------------------------------------
// small-M path: dense-M implicit GEMM, split-K over a thread-block cluster (b2_densem.cuh)
// ------------------------------------------------------------------------------------------
// Which layers take the dense-M kernel (tools/conv_sweep.py times single layers as CUDA-graph replays to re-check the rule):
// it beats the slab kernel only where a plane fills a small part of a 128-row tile AND the K loop is long enough to split --
// stride-1 multi-tap convolutions with M <= 1024 output positions (4x4 planes: 12% tile fill), strided multi-tap convolutions
// (whose slab form needs four phase sub-images per tap) with M <= 8192.  1x1x1 convolutions stay on the persistent GEMM.
// B2_DENSEM_MAXM = 0 disables the path, a positive value replaces BOTH thresholds (debug / sweeps).
static int g_densem_maxm = -1;
static int densem_maxm_env() {
  if (g_densem_maxm < 0) {
    const char* e = getenv("B2_DENSEM_MAXM");
    g_densem_maxm = e ? atoi(e) : -2;               // -2: no override
    if (g_densem_maxm == -1) g_densem_maxm = -2;
  }
  return g_densem_maxm;
}
static bool densem_wanted(long long M, int taps, bool strided) {
  const int ov = densem_maxm_env();
  if (ov >= 0) return ov > 0 && M <= ov;
  if (taps <= 1) return false;
  return strided ? M <= 8192 : M <= 1024;
}

// N tile (multiple of 32, <= 128, least padding then widest) and cluster size S (bn / S a multiple of 32, >= 2 K blocks per CTA):
// the smallest S that gives every SM a work unit, else the largest admissible one.  128 columns at most: the shared-memory
// accumulator tile of a wider N tile leaves too little room for the operand ring and for the peers' partials, which alias it.
static bool densem_split_ok(int bn, int S, int nkb) {      // bn / S a multiple of 32 and every CTA of the cluster gets >= 1 K block
  if (S < 1 || bn % (32 * S) != 0 || S > nkb) return false;
  const int per = (nkb + S - 1) / S;
  return (S - 1) * per < nkb;
}
static int g_densem_force_s = -1;
static void densem_plan(int M, int ldy, int nkb, int* bn_out, int* S_out) {
  int best_bn = 128, best_waste = 1 << 30;
  for (int bn = 128; bn >= 64; bn -= 32) {
    const int tn = (ldy + bn - 1) / bn;
    const int waste = tn * bn - ldy;
    if (waste < best_waste) { best_waste = waste; best_bn = bn; }
  }
  if (ldy <= 32) best_bn = 32;
  const int tiles = ((M + 127) / 128) * ((ldy + best_bn - 1) / best_bn);
  if (g_densem_force_s < 0) { const char* e = getenv("B2_DENSEM_S"); g_densem_force_s = e ? atoi(e) : 0; }
  int S = 1;
  for (int cand = 1; cand <= 8; ++cand) {
    if (!densem_split_ok(best_bn, cand, nkb) || (cand > 1 && nkb / cand < 2)) continue;
    if (g_densem_force_s > 0) { if (cand <= g_densem_force_s) S = cand; continue; }
    S = cand;
    if (tiles * cand >= 64) break;                  // beyond ~half the SMs the cluster / DSMEM cost outgrows the gain
  }
  *bn_out = best_bn; *S_out = S;
}

static int launch_densem(const IgemmLaunch& L, cudaStream_t stream) {
  DensemParams dp;
  memset(&dp, 0, sizeof(dp));
  dp.g = L.p;
  const IgemmParams& p = L.p;
  const int width = (p.epi == EPI_DIRECT_F32) ? p.Ncols : p.ldy;
  int bn = 0, S = 1;
  densem_plan(p.M_total, width, p.nkb, &bn, &S);
  dp.bn = bn; dp.bbytes = bn * 128; dp.stage_bytes = kBM * kBK * 2 + dp.bbytes;
  dp.ksplit = S;
  dp.kb_per = (p.nkb + S - 1) / S;
  dp.nstages = (227 * 1024 - 256 - 1024 - acc_bytes(bn)) / dp.stage_bytes;
  if (dp.nstages > kDmMaxStages) dp.nstages = kDmMaxStages;
  dp.acc_off = dp.nstages * dp.stage_bytes + 256;
  const int smem_bytes = dp.acc_off + acc_bytes(bn) + 1024;
  B2_OPT_IN_SMEM(densem_kernel, 227 * 1024);
  CUtensorMap tmA, tmB;
  int rc;
  if ((rc = make_tmap_2d_f16(&tmB, L.w, (uint64_t)L.b_cols, (uint64_t)p.Ncols, (uint64_t)L.ldb, kBK, (uint32_t)bn, true)) != B2_OK) return rc;
  if (p.amode == AMODE_TMA) {
    if ((rc = make_tmap_2d_f16(&tmA, L.a_mat, (uint64_t)L.a_cols, (uint64_t)p.M_total, (uint64_t)L.lda, kBK, kBM, true)) != B2_OK) return rc;
  } else {
    tmA = tmB;
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((width + bn - 1) / bn, (p.M_total + kBM - 1) / kBM, dp.ksplit);
  cfg.blockDim = dim3(kDmThreads);
  cfg.dynamicSmemBytes = smem_bytes;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
  attr[1].id = cudaLaunchAttributeClusterDimension;
  attr[1].val.clusterDim.x = 1; attr[1].val.clusterDim.y = 1; attr[1].val.clusterDim.z = dp.ksplit;
  cfg.attrs = attr; cfg.numAttrs = 2;
  B2_CHECK_CUDA(cudaLaunchKernelEx(&cfg, densem_kernel, tmA, tmB, dp));
  B2_CHECK_LAUNCH("densem_kernel");
  set_last_kernel(KID_DENSEM, bn, S);
  return B2_OK;
}

// does the dense-M kernel take this launch?  (plain per-column affine, no generator extras, few output positions)
static bool densem_applies(const IgemmParams& p, int k2) {
  if (p.in_scale) return false;
  const bool gather = p.amode != AMODE_TMA;
  const int taps = gather ? p.kt * p.kh * p.kw : 1;
  const bool strided = gather && (p.st > 1 || p.sh > 1 || p.sw > 1);
  return k2 == 0 && !p.aff_ld && !p.res_up && !p.res_pre && !p.y2 && densem_wanted(p.M_total, taps, strided) &&
         (p.epi == EPI_DIRECT_F32 || !p.per_row);
}

static int g_gemm_algo = 0;   // 0 auto (persistent kernel where it applies), 1 force the per-tile kernel

template <int BN, int GAN, int MASK = 0>
static int launch_pgemm(const IgemmLaunch& L, cudaStream_t stream) {
  using S = PgemmSmem<BN, GAN>;
  B2_OPT_IN_SMEM((pgemm_kernel<BN, GAN, MASK>), S::kTotal);
  const IgemmParams& ip = L.p;
  CUtensorMap tmA, tmB, tmC, tmR;
  int rc;
  if ((rc = make_tmap_2d_f16(&tmA, L.a_mat, (uint64_t)L.a_cols, (uint64_t)ip.M_total, (uint64_t)L.lda, 64, 128, true)) != B2_OK) return rc;
  if ((rc = make_tmap_2d_f16(&tmB, L.w, (uint64_t)L.b_cols, (uint64_t)ip.Ncols, (uint64_t)L.ldb, 64, BN, true)) != B2_OK) return rc;
  // outputs are stored per consumer warpgroup: boxes of 64 rows
  if ((rc = make_tmap_2d_f16(&tmC, ip.y, (uint64_t)ip.ldy, (uint64_t)ip.M_total, (uint64_t)ip.ldy, 64, 64, true)) != B2_OK) return rc;
  const int up_W = ip.up_W > 0 ? ip.up_W : 2;
  const int res_rows = up_W >= 128 ? 64 : 32;
  // residual maps span Ncols columns, not ldr: columns >= K (a skip tensor's dropped channels, whatever lies in the pitch gap) are
  // never read -- TMA zero-fills them -- so the output's padding columns stay zero
  if (ip.residual && ip.res_up) {
    // low-res skip tensor: a tile's 128 output rows read res_rows consecutive rows of it (see PgemmParams::res_up)
    if (!(up_W % 128 == 0 || (up_W <= 64 && 64 % up_W == 0)))
      return set_error(B2_ERR_UNSUPPORTED, "residual_up needs an output width that is a multiple of 128 or divides 64 (got %d)", up_W);
    if ((rc = make_tmap_2d_f16(&tmR, ip.residual, (uint64_t)ip.Ncols, (uint64_t)ip.M_total / 4, (uint64_t)ip.ldr, 64, res_rows, true)) != B2_OK) return rc;
  } else if (ip.residual) {
    if ((rc = make_tmap_2d_f16(&tmR, ip.residual, (uint64_t)ip.Ncols, (uint64_t)ip.M_total, (uint64_t)ip.ldr, 64, 128, true)) != B2_OK) return rc;
  } else {
    tmR = tmC;
  }
  CUtensorMap tmC2 = tmC;
  if (ip.y2 && (rc = make_tmap_2d_f16(&tmC2, ip.y2, (uint64_t)ip.ldy, (uint64_t)ip.M_total, (uint64_t)ip.ldy, 64, 64, true)) != B2_OK) return rc;
  CUtensorMap tmA2 = tmA, tmB2 = tmB;
  if (L.k2 > 0) {
    if ((rc = make_tmap_2d_f16(&tmA2, L.a2, (uint64_t)L.k2, (uint64_t)ip.M_total, (uint64_t)L.lda2, 64, 128, true)) != B2_OK) return rc;
    if ((rc = make_tmap_2d_f16(&tmB2, L.w2, (uint64_t)L.k2, (uint64_t)ip.Ncols, (uint64_t)L.ldb2, 64, BN, true)) != B2_OK) return rc;
  }
  PgemmParams p;
  p.M = ip.M_total; p.Ncols = ip.Ncols; p.ldy = ip.ldy; p.nkb = ip.nkb;
  p.nkb2 = (L.k2 + 63) / 64;
  p.tiles_n = (ip.ldy + BN - 1) / BN;
  p.tiles_total = p.tiles_n * ((ip.M_total + 127) / 128);
  p.scale = ip.scale; p.shift = ip.shift;
  p.has_residual = ip.residual != nullptr;
  p.relu = ip.relu;
  p.aff_ld = ip.aff_ld; p.aff_rows = ip.aff_rows;
  p.res_up = ip.res_up ? ip.residual : nullptr;
  p.res_ld = ip.ldr; p.Wh = up_W; p.Hh = ip.up_H > 0 ? ip.up_H : 2; p.res_rows = res_rows;
  p.fd_Wh = make_fastdiv(p.Wh); p.fd_Hh = make_fastdiv(p.Hh);
  p.res_pre = ip.res_pre;
  p.in_scale = GAN ? ip.in_scale : nullptr; p.in_shift = ip.in_shift; p.in_ld = ip.in_ld; p.in_rows = ip.in_rows > 0 ? ip.in_rows : 128;
  p.dual = ip.y2 != nullptr; p.scale2 = ip.scale2; p.shift2 = ip.shift2; p.aff2_ld = ip.aff2_ld; p.aff2_rows = ip.aff2_rows > 0 ? ip.aff2_rows : 128;
  p.mask = ip.mask; p.ldm = ip.ldm;
  p.fd_aff = make_fastdiv(ip.aff_rows > 0 ? ip.aff_rows : 1);
  const int grid = p.tiles_total < sm_count() ? p.tiles_total : sm_count();
  B2_CHECK_CUDA(launch_pdl(pgemm_kernel<BN, GAN, MASK>, dim3(grid), dim3(GAN ? kPgThreadsGan : kPgThreads), S::kTotal, stream, tmA, tmB, tmA2, tmB2, tmC, tmR, tmC2, p));
  B2_CHECK_LAUNCH("pgemm_kernel");
  set_last_kernel(KID_PGEMM, BN, MASK, GAN);
  return B2_OK;
}

// The chained instance (b2_gemm_chain_f16): closing GEMM of width N = ldd, then h1 = relu(scale1 * (y . W1^T) + shift1).  Its
// N tile and the chained MMA width are the ones the two stand-alone launches pick (64 for a pitch <= 64, else 128).
template <int BN, int BN1>
static int launch_pgemm_chain(const b2_gemm_args* g, const void* a2, int lda2, const void* b2, int ldb2, int k2, const void* w1, int ldw1,
                              int n1, const float* scale1, const float* shift1, void* d1, int ldd1, cudaStream_t stream) {
  using S = PgemmChainSmem<BN, BN1>;
  B2_OPT_IN_SMEM((pgemm_chain_kernel<BN, BN1>), S::kTotal);
  CUtensorMap tmA, tmB, tmA2, tmB2, tmC, tmR, tmW1, tmH;
  int rc;
  if ((rc = make_tmap_2d_f16(&tmA, g->a, (uint64_t)g->Kd, (uint64_t)g->M, (uint64_t)g->lda, 64, 128, true)) != B2_OK) return rc;
  if ((rc = make_tmap_2d_f16(&tmB, g->b, (uint64_t)g->Kd, (uint64_t)g->N, (uint64_t)g->ldb, 64, BN, true)) != B2_OK) return rc;
  if ((rc = make_tmap_2d_f16(&tmC, g->d, (uint64_t)g->ldd, (uint64_t)g->M, (uint64_t)g->ldd, 64, 64, true)) != B2_OK) return rc;
  tmA2 = tmA; tmB2 = tmB; tmR = tmC;
  if (k2 > 0) {
    if ((rc = make_tmap_2d_f16(&tmA2, a2, (uint64_t)k2, (uint64_t)g->M, (uint64_t)lda2, 64, 128, true)) != B2_OK) return rc;
    if ((rc = make_tmap_2d_f16(&tmB2, b2, (uint64_t)k2, (uint64_t)g->N, (uint64_t)ldb2, 64, BN, true)) != B2_OK) return rc;
  }
  if (g->residual && (rc = make_tmap_2d_f16(&tmR, g->residual, (uint64_t)g->N, (uint64_t)g->M, (uint64_t)g->ldr, 64, 128, true)) != B2_OK)
    return rc;
  if ((rc = make_tmap_2d_f16(&tmW1, w1, (uint64_t)g->N, (uint64_t)n1, (uint64_t)ldw1, 64, BN1, true)) != B2_OK) return rc;
  if ((rc = make_tmap_2d_f16(&tmH, d1, (uint64_t)ldd1, (uint64_t)g->M, (uint64_t)ldd1, 64, 64, true)) != B2_OK) return rc;
  PgemmChainParams p;
  p.M = g->M; p.Ncols = g->N;
  p.nkb = (g->Kd + 63) / 64; p.nkb2 = (k2 + 63) / 64;
  p.npass = (g->N + BN - 1) / BN;
  p.tiles_total = (g->M + 127) / 128;
  p.scale = g->scale; p.shift = g->shift;
  p.has_residual = g->residual != nullptr; p.relu = g->relu;
  p.N1 = n1; p.ld1 = ldd1; p.scale1 = scale1; p.shift1 = shift1;
  const int grid = p.tiles_total < sm_count() ? p.tiles_total : sm_count();
  B2_CHECK_CUDA(launch_pdl(pgemm_chain_kernel<BN, BN1>, dim3(grid), dim3(kPgThreads), S::kTotal, stream, tmA, tmB, tmA2, tmB2, tmC, tmR,
                           tmW1, tmH, p));
  B2_CHECK_LAUNCH("pgemm_chain_kernel");
  set_last_kernel(KID_PGEMM_CHAIN, BN, BN1);
  return B2_OK;
}

// The split instance (b2_gemm_split_f16): pgemm_kernel<BN, 0, 3> with one tensor map per column-slice destination.
template <int BN>
static int launch_pgemm_split(const b2_gemm_args* g, int nd, void* const* y, const int* ldy, const int* cols, const int* box0,
                              cudaStream_t stream) {
  using S = PgemmSmem<BN, 0>;
  B2_OPT_IN_SMEM((pgemm_kernel<BN, 0, 3>), S::kTotal);
  CUtensorMap tmA, tmB, tmD[4];
  int rc;
  const int Npad = box0[nd] * 64;
  if ((rc = make_tmap_2d_f16(&tmA, g->a, (uint64_t)g->Kd, (uint64_t)g->M, (uint64_t)g->lda, 64, 128, true)) != B2_OK) return rc;
  if ((rc = make_tmap_2d_f16(&tmB, g->b, (uint64_t)g->Kd, (uint64_t)Npad, (uint64_t)g->ldb, 64, BN, true)) != B2_OK) return rc;
  for (int d = 0; d < 4; ++d) {
    const int s = d < nd ? d : 0;       // unused slots repeat destination 0 (never selected)
    if ((rc = make_tmap_2d_f16(&tmD[d], y[s], (uint64_t)cols[s], (uint64_t)g->M, (uint64_t)ldy[s], 64, 64, true)) != B2_OK) return rc;
  }
  PgemmParams p;
  memset(&p, 0, sizeof(p));
  p.M = g->M; p.Ncols = Npad; p.ldy = Npad; p.nkb = (g->Kd + 63) / 64; p.nkb2 = 0;
  p.tiles_n = (Npad + BN - 1) / BN;
  p.tiles_total = p.tiles_n * ((g->M + 127) / 128);
  p.scale = g->scale; p.shift = g->shift;
  p.relu = g->relu;
  p.fd_Wh = make_fastdiv(2); p.fd_Hh = make_fastdiv(2); p.fd_aff = make_fastdiv(1);
  for (int d = 0; d < 4; ++d) p.split_box[d] = d < nd ? box0[d] : INT_MAX;
  const int grid = p.tiles_total < sm_count() ? p.tiles_total : sm_count();
  B2_CHECK_CUDA(launch_pdl(pgemm_kernel<BN, 0, 3>, dim3(grid), dim3(kPgThreads), S::kTotal, stream, tmA, tmB, tmD[3], tmB, tmD[0], tmD[1],
                           tmD[2], p));
  B2_CHECK_LAUNCH("pgemm_kernel");
  set_last_kernel(KID_PGEMM_SPLIT, BN, nd, Npad);
  return B2_OK;
}

// The dual instance (b2_gemm_dual_f16): pgemm_kernel<BN, 0, 4>, d through tmC as b2_gemm_f16 writes it, d2 through tmC2.
template <int BN>
static int launch_pgemm_dual(const b2_gemm_args* g, const float* scale2, const float* shift2, void* d2, int ldd2, cudaStream_t stream) {
  using S = PgemmSmem<BN, 0, 1>;
  B2_OPT_IN_SMEM((pgemm_kernel<BN, 0, 4>), S::kTotal);
  CUtensorMap tmA, tmB, tmC, tmR, tmC2;
  int rc;
  if ((rc = make_tmap_2d_f16(&tmA, g->a, (uint64_t)g->Kd, (uint64_t)g->M, (uint64_t)g->lda, 64, 128, true)) != B2_OK) return rc;
  if ((rc = make_tmap_2d_f16(&tmB, g->b, (uint64_t)g->Kd, (uint64_t)g->N, (uint64_t)g->ldb, 64, BN, true)) != B2_OK) return rc;
  if ((rc = make_tmap_2d_f16(&tmC, g->d, (uint64_t)g->ldd, (uint64_t)g->M, (uint64_t)g->ldd, 64, 64, true)) != B2_OK) return rc;
  if ((rc = make_tmap_2d_f16(&tmC2, d2, (uint64_t)ldd2, (uint64_t)g->M, (uint64_t)ldd2, 64, 64, true)) != B2_OK) return rc;
  tmR = tmC;
  if (g->residual && (rc = make_tmap_2d_f16(&tmR, g->residual, (uint64_t)g->N, (uint64_t)g->M, (uint64_t)g->ldr, 64, 128, true)) != B2_OK)
    return rc;
  PgemmParams p;
  memset(&p, 0, sizeof(p));
  p.M = g->M; p.Ncols = g->N; p.ldy = g->ldd; p.nkb = (g->Kd + 63) / 64; p.nkb2 = 0;
  p.tiles_n = (g->ldd + BN - 1) / BN;
  p.tiles_total = p.tiles_n * ((g->M + 127) / 128);
  p.scale = g->scale; p.shift = g->shift;
  p.has_residual = g->residual != nullptr;
  p.relu = g->relu;
  p.dual = 1; p.scale2 = scale2; p.shift2 = shift2; p.aff2_ld = 0; p.aff2_rows = 128;   // one per-column row for every tile
  p.fd_Wh = make_fastdiv(2); p.fd_Hh = make_fastdiv(2); p.fd_aff = make_fastdiv(1);
  const int grid = p.tiles_total < sm_count() ? p.tiles_total : sm_count();
  B2_CHECK_CUDA(launch_pdl(pgemm_kernel<BN, 0, 4>, dim3(grid), dim3(kPgThreads), S::kTotal, stream, tmA, tmB, tmA, tmB, tmC, tmR, tmC2, p));
  B2_CHECK_LAUNCH("pgemm_kernel");
  set_last_kernel(KID_PGEMM, BN, 4, 0);
  return B2_OK;
}

// The split-K instance (b2_gemm_splitk_f16): pgemm_kernel<BN, 0, 5> writes the fp32 partial accumulators of every (split, tile)
// into the workspace, splitk_reduce_kernel sums them in split order and applies the epilogue.
template <int BN>
static int launch_pgemm_splitk(const b2_gemm_args* g, int splits, float* ws, int ldw, cudaStream_t stream) {
  using S = PgemmSmem<BN, 0, 0>;
  B2_OPT_IN_SMEM((pgemm_kernel<BN, 0, 5>), S::kTotal);
  CUtensorMap tmA, tmB;
  int rc;
  if ((rc = make_tmap_2d_f16(&tmA, g->a, (uint64_t)g->Kd, (uint64_t)g->M, (uint64_t)g->lda, 64, 128, true)) != B2_OK) return rc;
  if ((rc = make_tmap_2d_f16(&tmB, g->b, (uint64_t)g->Kd, (uint64_t)g->N, (uint64_t)g->ldb, 64, BN, true)) != B2_OK) return rc;
  PgemmParams p;
  memset(&p, 0, sizeof(p));
  p.M = g->M; p.Ncols = g->N; p.ldy = ldw; p.nkb = (g->Kd + 63) / 64; p.nkb2 = 0;
  p.tiles_n = (ldw + BN - 1) / BN;
  p.tiles_mn = p.tiles_n * ((g->M + 127) / 128);
  p.splits = splits;
  p.tiles_total = p.tiles_mn * splits;
  p.ldw = ldw; p.ws = ws;
  p.aff2_rows = 128;
  p.fd_Wh = make_fastdiv(2); p.fd_Hh = make_fastdiv(2); p.fd_aff = make_fastdiv(1);
  const int grid = p.tiles_total < sm_count() ? p.tiles_total : sm_count();
  // the maps this instance never reads are given tmA (every map argument must be a valid descriptor)
  B2_CHECK_CUDA(launch_pdl(pgemm_kernel<BN, 0, 5>, dim3(grid), dim3(kPgThreads), S::kTotal, stream, tmA, tmB, tmA, tmB, tmA, tmA, tmA, p));
  B2_CHECK_LAUNCH("pgemm_kernel");
  const int width = g->out_f32 ? g->N : g->ldd;
  const int quads = (width + 3) / 4;
  const long long threads = (long long)g->M * quads;
  splitk_reduce_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, stream>>>(ws, splits, g->M, g->N, ldw, g->scale, g->shift, g->relu, g->d,
                                                                             g->ldd, g->out_f32, quads);
  B2_CHECK_LAUNCH("splitk_reduce_kernel");
  set_last_kernel(KID_PGEMM_SPLITK, BN, splits);
  return B2_OK;
}

static int g_last_gemm_path = 0;   // kernel of the last GEMM-family launch: 1 dense-M, 2 persistent GEMM, 3 implicit GEMM (tests pin it)

static int dispatch_igemm(const IgemmLaunch& L, cudaStream_t stream) {
  if (L.p.mask) {
    // ReLU-derivative mask (fine-tuning backward): the persistent GEMM and the implicit-GEMM kernel carry the masked epilogue
    if (L.p.epi != EPI_TMA_F16 || L.p.per_row || L.p.relu || L.p.aff_ld || L.p.res_up || L.p.res_pre || L.p.y2 || L.p.in_scale)
      return set_error(B2_ERR_UNSUPPORTED, "a masked output needs fp16 output without ReLU, per-row / per-sample affines or generator extras");
    if (L.p.ldm % 8 || L.p.ldm < L.p.ldy) return set_error(B2_ERR_INVALID, "mask pitch %d must be a multiple of 8 and >= ldy %d", L.p.ldm, L.p.ldy);
    if (g_gemm_algo == 0 && L.p.amode == AMODE_TMA) { g_last_gemm_path = 2; return launch_pgemm<64, 0, 1>(L, stream); }
    if (L.k2 > 0) return set_error(B2_ERR_UNSUPPORTED, "two-operand GEMM needs the persistent kernel");
    g_last_gemm_path = 3;
    return L.p.ldy <= 64 ? launch_igemm<64, 1>(L, stream) : launch_igemm<128, 1>(L, stream);
  }
  if (g_gemm_algo == 0 && densem_applies(L.p, L.k2)) { g_last_gemm_path = 1; return launch_densem(L, stream); }
  if (g_gemm_algo == 0 && L.p.amode == AMODE_TMA && L.p.epi == EPI_TMA_F16 && !L.p.per_row) {
    // 64-wide N tiles for narrow outputs, 128 otherwise
    g_last_gemm_path = 2;
    const bool gan = L.p.y2 || L.p.res_up || L.p.res_pre || L.p.in_scale;
    if (L.p.ldy <= 64) return gan ? launch_pgemm<64, 1>(L, stream) : launch_pgemm<64, 0>(L, stream);
    return gan ? launch_pgemm<128, 1>(L, stream) : launch_pgemm<128, 0>(L, stream);
  }
  if (L.p.aff_ld)
    return set_error(B2_ERR_UNSUPPORTED, "per-sample affine is implemented by the slab convolution and the persistent GEMM only");
  if (L.p.res_up || L.p.res_pre || L.p.y2 || L.p.in_scale)
    return set_error(B2_ERR_UNSUPPORTED, "upsampled / pre-scale residuals, second outputs and input affines are implemented by the persistent GEMM (1x1 convolutions, fp16) only");
  // 64-wide tiles for narrow outputs, 128 otherwise
  const int width = (L.p.epi == EPI_TMA_F16) ? L.p.ldy : L.p.Ncols;
  g_last_gemm_path = 3;
  if (width <= 64) return launch_igemm<64, 0>(L, stream);
  return launch_igemm<128, 0>(L, stream);
}

bool pdl_enabled() {
  static int v = -1;
  if (v < 0) { const char* e = getenv("B2_PDL"); v = (e && e[0] == '0') ? 0 : 1; }
  return v != 0;
}

}  // namespace b2

using namespace b2;

extern "C" {

int b2_version(void) { return 103; }   // 103: split-K / fused (2+1)D / pooled-stem entry points (round 2); 102: generator fields
/* debug knob (not in the public header): 0 = auto, 1 = never use the slab kernel */
int b2_debug_set_conv_algo(int algo) { g_conv_algo = algo; return B2_OK; }
int b2_debug_set_gemm_algo(int algo) { g_gemm_algo = algo; return B2_OK; }
/* host-only view of the slab kernel's tiling decision for a convolution (no launch, no GPU needed): out = {applies, BN, MT, R, PW,
   WC, wchunks, items, flex, remapped}.  Used by tests/test_host_logic.py and by tuning scripts.  slice != 0: the plan of
   b2_conv_ndhwc_fprop_slice (a->ldy the slice width), which takes 128-column tiles where the runtime-N tile finds no fit. */
static int slab_plan_view(const b2_conv_args* a_in, int* out, bool slice, int narrow = 0) {
  b2_conv_args remap = *a_in;
  const b2_conv_args* a = a_in;
  int wc_hint = 0, remapped = 0;
  if (a_in->kt > 1 && a_in->kh == 1 && a_in->kw == 1 && a_in->st == 1 && a_in->sh == 1 && a_in->sw == 1 && a_in->ph == 0 && a_in->pw == 0) {
    remap.T = 1; remap.H = a_in->T; remap.W = a_in->H * a_in->W; remap.kt = 1; remap.kh = a_in->kt; remap.kw = 1;
    remap.pt = 0; remap.ph = a_in->pt; remap.pw = 0; a = &remap; wc_hint = 64; remapped = 1;
  }
  SlabChoice c;
  memset(&c, 0, sizeof(c));
  const bool ok = slab_choose(a, wc_hint, 0, slice ? 1 : 0, &c, narrow);   // the launchers' own planner (ldo only selects the slice rules)
  const int BN = ok ? c.BN : 0, best_mt = ok ? c.MT : 0;
  out[0] = ok; out[1] = BN; out[2] = best_mt; out[3] = ok ? c.R : 0; out[4] = c.p.PW; out[5] = c.p.WC; out[6] = c.p.wchunks;
  const long long tq = best_mt ? (c.p.P + best_mt * 128 - 1) / (best_mt * 128) : 0;
  out[7] = (int)(((a->ldy + BN - 1) / (BN ? BN : 1)) * tq * c.p.wchunks * a->N * c.p.To);
  out[8] = ok && c.flex; out[9] = remapped;
  return B2_OK;
}
int b2_debug_slab_plan(const b2_conv_args* a_in, int* out) { return slab_plan_view(a_in, out, false); }
int b2_debug_slab_slice_plan(const b2_conv_args* a_in, int* out) { return slab_plan_view(a_in, out, true); }
/* the plan of b2_conv_ndhwc_fprop_slice_narrow (a->ldy = a->K = 32 or 48) */
int b2_debug_slab_slice_narrow_plan(const b2_conv_args* a_in, int* out) { return slab_plan_view(a_in, out, true, a_in->K); }
/* debug knobs of the small-M path: layers with M <= maxm take the dense-M kernel (0 = never); force_s > 0 caps the cluster size */
int b2_debug_set_slab_wide(int on) { g_slab_wide = on; return B2_OK; }   /* 1: request 256-column tiles; -1 / 0: the rule */
/* host-only view of the temporal stack kernel's decision for a convolution (no launch, no GPU needed): out = {applies, items, frame
   groups per clip, position tiles per frame, channel chunks, resident filter bytes, dynamic shared memory bytes} */
int b2_debug_tstack_plan(const b2_conv_args* a, int* out) {
  if (g_tstack == -2) { const char* e = getenv("B2_TSTACK"); g_tstack = (e && e[0] == '0') ? 0 : -1; }
  TstackParams p;
  size_t smem = 0;
  memset(&p, 0, sizeof(p));
  const bool ok = g_tstack != 0 && tstack_plan(a, &p, &smem);
  out[0] = ok; out[1] = ok ? p.items_total : 0; out[2] = p.groups; out[3] = p.tiles_q; out[4] = p.cchunks;
  out[5] = ok ? p.cchunks * p.kt * kTkWBlock : 0; out[6] = ok ? (int)smem : 0;
  return B2_OK;
}
int b2_debug_last_conv_path(void) { return g_last_conv_path; }
/* stem convolution: output rows per work item of the last launch (1, 2 or 4; b2_debug_last_kernel's info[1] tells whether the
   four-row instance was the transposed one); rows = 2 / 4 forces the two- / four-row BN = 64 instance with positions along M,
   rows = 20 (4 | 16) the transposed four-row instance (each only where eligible), -1 the rule.  The row plan of (G, kh):
   out[3 i .. 3 i + 2] = {g_lo, g_hi, first weight slot} of slab row i, returns the slab row count. */
int b2_debug_last_stem_rows(void) { return g_last_stem_rows; }
int b2_debug_set_stem_rows(int rows) { g_stem_rows = (rows == 2 || rows == 4 || rows == kStemForceT) ? rows : -1; return B2_OK; }
/* host-only view of the stem's instance choice (no launch, no GPU needed) for K output channels, a kt x kh x 7 filter, Wo output
   columns and pair mode on / off, under the current force knob: out = {G, transposed} */
int b2_debug_stem_plan(int K, int kt, int kh, int Wo, int pair, int* out) {
  bool transposed = false;
  out[0] = stem_rows_for(K <= 64 ? 64 : 128, kt, kh, Wo, pair != 0, &transposed);
  out[1] = transposed;
  return B2_OK;
}
int b2_debug_stem_row_plan(int G, int kh, int* out) {
  const int rows = 2 * (G - 1) + kh;
  if (G < 1 || kh < 1 || rows > kStemMaxRows) return -1;
  for (int i = 0; i < rows; ++i) stem_row_plan(G, kh, i, &out[3 * i], &out[3 * i + 1], &out[3 * i + 2]);
  return rows;
}
int b2_debug_last_gemm_path(void) { return g_last_gemm_path; }   /* 1 dense-M, 2 persistent GEMM, 3 implicit GEMM (last GEMM-family launch) */   /* 1: the temporal stack kernel took the last convolution */
int b2_debug_set_tstack(int mode) { g_tstack = mode < -1 ? -1 : (mode > 1 ? 1 : mode); return B2_OK; }   /* temporal stack kernel: -1 rule, 0 never, 1 whenever eligible */
/* 128-wide slab tiles as the transposed product (b2_slab_t128.cuh): mode -1 = the rule, 0 = never, 1 = wherever the form applies.
   Host-only view of its decision for a convolution (no launch, no GPU needed) under the current knobs: out = {taken, applies, NP,
   rows per item, slab rows R, items, dynamic shared memory bytes, slab kernel items, slab kernel MT, SM count the rule used}.
   b2_debug_last_kernel's info
   of a launch of the form (KID_SLAB_T128): {NP, rows per item, N tile 128, spatial stride, R}. */
int b2_debug_set_slab_t128(int mode) { g_slab_t128 = mode < -1 ? -1 : (mode > 1 ? 1 : mode); return B2_OK; }
int b2_debug_slab_t128_plan(const b2_conv_args* a, int* out) {
  memset(out, 0, 10 * sizeof(int));
  out[9] = sm_count();
  TPlan t;
  memset(&t, 0, sizeof(t));
  SlabChoice c;
  const bool remapped = a->kt > 1 && a->kh == 1 && a->kw == 1;      // the remapped temporal form is never this one's
  if (remapped || !slab_choose(a, 0, 0, 0, &c)) return B2_OK;
  out[0] = slab_t128_wanted(a, c, &t);
  out[1] = slab_t_geometry(a, 128, &t);
  out[2] = t.np; out[3] = t.rows; out[4] = t.R; out[5] = t.items; out[6] = t.smem;
  out[7] = (int)slab_items(a, c); out[8] = c.MT;
  return B2_OK;
}
/* 64-wide slab tiles as the transposed product (b2_slab_t128.cuh): mode -1 = the rule, 0 = never, 1 = wherever the form applies.
   Host-only view of its decision for a convolution (no launch, no GPU needed) under the current knobs: out = {taken, applies, NP,
   slab rows R, items, dynamic shared memory bytes, slab kernel items, slab kernel MT, SM count the rule used}.
   b2_debug_last_kernel's info of a launch of the form (KID_SLAB_T64): {NP, items, R}. */
int b2_debug_set_slab_t64(int mode) { g_slab_t64 = mode < -1 ? -1 : (mode > 1 ? 1 : mode); return B2_OK; }
int b2_debug_slab_t64_plan(const b2_conv_args* a, int* out) {
  memset(out, 0, 9 * sizeof(int));
  out[8] = sm_count();
  TPlan t;
  memset(&t, 0, sizeof(t));
  SlabChoice c;
  const bool remapped = a->kt > 1 && a->kh == 1 && a->kw == 1;      // the remapped temporal form is never this one's
  if (remapped || !slab_choose(a, 0, 0, 0, &c)) return B2_OK;
  out[0] = slab_t64_wanted(a, c, &t);
  out[1] = slab_t_geometry(a, 64, &t);
  out[2] = t.np; out[3] = t.R; out[4] = t.items; out[5] = t.smem;
  out[6] = (int)slab_items(a, c); out[7] = c.MT;
  return B2_OK;
}
int b2_debug_set_slab_mt(int mt) { g_slab_force_mt = mt < 0 ? 0 : mt; return B2_OK; }
int b2_debug_set_densem(int maxm, int force_s) { g_densem_maxm = maxm < 0 ? -2 : maxm; g_densem_force_s = force_s; return B2_OK; }
/* The temporal-group slab kernel this selected is gone (the slab kernel's 64-wide tile does what it was for); the entry point
   stays for the ABI and accepts its argument with no effect. */
int b2_debug_set_slabts(int mode) { (void)mode; return B2_OK; }
/* kernel of the last convolution / GEMM / attention call (a KID_* id of b2_host.h, 0 when the call launched nothing) and its
   tile parameters in info[0..4]: slab {BN, MT, flex, wchunks, remapped}, densem {bn, S}, pgemm {BN, masked, generator instance},
   igemm {BN, masked}, stem {G, transposed},
   attention {online, DVT}, grouped convolution {G, MT, planes per item, wchunks}; unused entries are 0 */
int b2_debug_last_kernel(int* info) {
  if (info) memcpy(info, g_last_info, sizeof(g_last_info));
  return g_last_kernel;
}
const char* b2_last_error(void) { return g_err; }
uint64_t b2_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

static int conv_out_dim(int in, int k, int s, int p) { return (in + 2 * p - k) / s + 1; }

static int validate_conv(const b2_conv_args* a) {
  B2_CHECK_ARG(a != nullptr, "null args");
  B2_CHECK_ARG(a->x && a->w && a->scale && a->shift && a->y, "null tensor pointer");
  B2_CHECK_ARG(a->N > 0 && a->T > 0 && a->H > 0 && a->W > 0 && a->C > 0 && a->K > 0, "non-positive dimension");
  B2_CHECK_ARG(a->kt > 0 && a->kh > 0 && a->kw > 0 && a->st > 0 && a->sh > 0 && a->sw > 0, "bad kernel/stride");
  B2_CHECK_ARG(a->pt >= 0 && a->ph >= 0 && a->pw >= 0, "negative padding");
  B2_CHECK_ARG(a->ldy >= a->K, "ldy < K");
  B2_CHECK_ARG(a->residual == nullptr || a->ldr >= a->K, "ldr < K");
  B2_CHECK_ARG(conv_out_dim(a->T, a->kt, a->st, a->pt) > 0 && conv_out_dim(a->H, a->kh, a->sh, a->ph) > 0 &&
                   conv_out_dim(a->W, a->kw, a->sw, a->pw) > 0,
               "empty output");
  B2_CHECK_ARG(!a->pool_w || a->mode == B2_CONV_STEM7, "pool_w is implemented by the stem convolution only");
  B2_CHECK_ARG(!a->mask || (a->mode == B2_CONV_AUTO && !a->upsample), "a masked output needs a plain (B2_CONV_AUTO) convolution");
  if (a->mode == B2_CONV_STEM7) {
    B2_CHECK_ARG(a->C == 4, "STEM7 needs NDHWC4 input (C == 4), got %d", a->C);
    B2_CHECK_ARG(a->kw == 7 && a->sw == 2 && a->pw == 3, "STEM7 needs kw=7, sw=2, pw=3");
    B2_CHECK_ARG(a->W % 2 == 0, "STEM7 needs an even input width, got %d", a->W);
  } else {
    B2_CHECK_ARG(a->mode == B2_CONV_AUTO, "unknown conv mode %d", a->mode);
    B2_CHECK_ARG(a->C % 8 == 0, "channel pitch %d is not a multiple of 8", a->C);
  }
  if (a->residual_up || a->residual_pre) {
    B2_CHECK_ARG(a->residual != nullptr && a->kt * a->kh * a->kw == 1 && a->st == 1 && a->sh == 1 && a->sw == 1 && a->T == 1 &&
                     !a->out_f32 && a->mode == B2_CONV_AUTO,
                 "residual_up / residual_pre need a residual and a 1x1 stride-1 2-D convolution with fp16 output");
    B2_CHECK_ARG(!a->residual_up || (a->H % 2 == 0 && a->W % 2 == 0), "residual_up needs even output height and width");
  }
  if (a->upsample)
    B2_CHECK_ARG(a->upsample == 1 && a->mode == B2_CONV_AUTO && !a->out_f32 && a->kt == 1 && a->kh == 3 && a->kw == 3 && a->st == 1 &&
                     a->sh == 1 && a->sw == 1 && a->pt == 0 && a->ph == 1 && a->pw == 1,
                 "fused upsampling is implemented for 1x3x3 stride-1 'same' convolutions with fp16 output only");
  B2_CHECK_ARG(a->aff_ld >= 0 && (a->aff_ld == 0 || (a->aff_ld >= a->K && !a->out_f32 && a->mode == B2_CONV_AUTO)),
               "bad per-sample affine pitch %d", a->aff_ld);
  if (!a->out_f32) {
    B2_CHECK_ARG(a->ldy % 8 == 0, "ldy %d is not a multiple of 8", a->ldy);
    B2_CHECK_ARG(a->residual == nullptr || a->ldr % 8 == 0, "ldr %d is not a multiple of 8", a->ldr);
    B2_CHECK_ARG(!a->accumulate, "accumulate requires out_f32");
  }
  return B2_OK;
}

int b2_conv_ndhwc_fprop(const b2_conv_args* a, void* stream) {
  set_last_kernel(KID_NONE);
  int rc = validate_conv(a);
  if (rc != B2_OK) return rc;
  if ((rc = require_sm90()) != B2_OK) return rc;
  const long long M_out = (long long)a->N * conv_out_dim(a->T, a->kt, a->st, a->pt) * conv_out_dim(a->H, a->kh, a->sh, a->ph) *
                          conv_out_dim(a->W, a->kw, a->sw, a->pw);
  const bool small_m = a->mode == B2_CONV_AUTO && !a->upsample && !a->aff_ld && !a->out_f32 && !a->y2 && !a->residual_up &&
                       !a->residual_pre && !a->in_scale && g_gemm_algo == 0 &&
                       densem_wanted(M_out, a->kt * a->kh * a->kw, a->st > 1 || a->sh > 1 || a->sw > 1);
  g_last_conv_path = 0;
  g_last_gemm_path = 0;
  const bool skip_slab = small_m || a->mask != nullptr;     // the slab / temporal kernels have no masked epilogue
  rc = skip_slab ? 0 : try_tstack(a, reinterpret_cast<cudaStream_t>(stream));
  if (rc != 0) return rc < 0 ? rc : B2_OK;
  rc = skip_slab ? 0 : try_slab(a, reinterpret_cast<cudaStream_t>(stream));
  if (rc != 0) return rc < 0 ? rc : B2_OK;
  if (a->upsample) return set_error(B2_ERR_UNSUPPORTED, "fused upsampling needs the slab kernel, which does not take this shape");

  IgemmLaunch L;
  memset(&L, 0, sizeof(L));
  IgemmParams& p = L.p;
  p.x = reinterpret_cast<const __half*>(a->x);
  p.N = a->N; p.T = a->T; p.H = a->H; p.W = a->W; p.C = a->C;
  p.To = conv_out_dim(a->T, a->kt, a->st, a->pt);
  p.Ho = conv_out_dim(a->H, a->kh, a->sh, a->ph);
  p.Wo = conv_out_dim(a->W, a->kw, a->sw, a->pw);
  p.kt = a->kt; p.kh = a->kh; p.kw = a->kw;
  p.st = a->st; p.sh = a->sh; p.sw = a->sw;
  p.pt = a->pt; p.ph = a->ph; p.pw = a->pw;
  const long long M = (long long)a->N * p.To * p.Ho * p.Wo;
  B2_CHECK_ARG(M < (1ll << 31), "output too large");
  p.M_total = (int)M;
  p.Ncols = a->K;
  p.scale = a->scale; p.shift = a->shift;
  p.residual = reinterpret_cast<const __half*>(a->residual);
  p.ldr = a->ldr;
  p.y = a->y; p.ldy = a->ldy;
  p.relu = a->relu; p.per_row = 0; p.accumulate = a->accumulate;
  p.epi = a->out_f32 ? EPI_DIRECT_F32 : EPI_TMA_F16;
  p.aff_ld = a->aff_ld;
  p.res_up = a->residual_up; p.res_pre = a->residual_pre; p.up_H = p.Ho; p.up_W = p.Wo;
  p.y2 = a->y2; p.scale2 = a->scale2; p.shift2 = a->shift2; p.aff2_ld = a->aff2_ld; p.aff2_rows = p.To * p.Ho * p.Wo;
  if (a->y2) {
    B2_CHECK_ARG(a->scale2 && a->shift2 && a->aff2_ld >= a->K && !a->out_f32 && a->kt * a->kh * a->kw == 1,
                 "second output needs scale2 / shift2 (fp32 [N][aff2_ld >= K]) and a 1x1 convolution with fp16 output");
    if (p.aff2_rows % 128 != 0)
      return set_error(B2_ERR_UNSUPPORTED, "second output with a per-sample affine needs To*Ho*Wo %% 128 == 0 (got %d)", p.aff2_rows);
  }
  if (a->in_scale) {
    B2_CHECK_ARG(a->in_shift && a->in_aff_ld >= a->C && (a->in_aff_ld & 3) == 0 && !a->out_f32 && a->kt * a->kh * a->kw == 1 && a->st == 1 &&
                     a->sh == 1 && a->sw == 1 && (reinterpret_cast<uintptr_t>(a->in_scale) & 15) == 0 &&
                     (reinterpret_cast<uintptr_t>(a->in_shift) & 15) == 0,
                 "input affine needs in_shift, a 16-byte aligned fp32 [N][in_aff_ld >= C] pair (pitch %% 4 == 0) and a 1x1 stride-1 convolution with fp16 output");
    if ((p.To * p.Ho * p.Wo) % 128 != 0 || a->C % 64 != 0)
      return set_error(B2_ERR_UNSUPPORTED, "input affine needs To*Ho*Wo %% 128 == 0 and a channel pitch that is a multiple of 64 (got %d, %d)",
                       p.To * p.Ho * p.Wo, a->C);
    p.in_scale = a->in_scale; p.in_shift = a->in_shift; p.in_ld = a->in_aff_ld; p.in_rows = p.To * p.Ho * p.Wo;
  }
  p.aff_rows = p.To * p.Ho * p.Wo;
  p.mask = reinterpret_cast<const __half*>(a->mask); p.ldm = a->ldm;
  if (a->aff_ld && p.aff_rows % 128 != 0)
    return set_error(B2_ERR_UNSUPPORTED, "per-sample affine on a 1x1x1 convolution needs To*Ho*Wo %% 128 == 0 (got %d)", p.aff_rows);
  L.w = a->w;

  const int taps = a->kt * a->kh * a->kw;
  if (a->mode == B2_CONV_STEM7) {
    B2_CHECK_ARG(!a->out_f32 && a->residual == nullptr, "stem convolution has no residual / fp32 output");
    B2_CHECK_ARG(a->st == 1 && a->sh == 2, "stem convolution needs strides (1, 2, 2)");
    const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    return a->K <= 64 ? launch_stem<64>(a, st) : launch_stem<128>(a, st);
  } else if (taps == 1 && a->st == 1 && a->sh == 1 && a->sw == 1 && a->pt == 0 && a->ph == 0 && a->pw == 0) {
    // 1x1x1 stride-1: A is literally the [M][C] activation matrix -> TMA on both operands
    p.amode = AMODE_TMA;
    p.nkb = (a->C + kBK - 1) / kBK;
    L.a_mat = a->x; L.lda = a->C; L.a_cols = a->C;
    L.ldb = a->C; L.b_cols = a->C;
  } else {
    p.amode = AMODE_GATHER;
    p.cchunks = (a->C + kBK - 1) / kBK;
    p.nkb = taps * p.cchunks;
    L.ldb = taps * a->C;
    L.b_cols = L.ldb;
    // When C % 64 != 0 the last K block of a tap also covers the first columns of the next tap's
    // weights; the activation side zero-fills channels >= C, so those products vanish.
  }
  return dispatch_igemm(L, reinterpret_cast<cudaStream_t>(stream));
}

// ------------------------------------------------------------------------------------------
// grouped convolution (b2_groupconv.cuh)
// ------------------------------------------------------------------------------------------
static bool grouped_filter_ok(int K, int cg, int groups, int kt, int kh, int kw) {
  return K > 0 && groups > 0 && K % 64 == 0 && (cg == 4 || cg == 8 || cg == 16 || cg == 32) && (long long)cg * groups == K &&
         kh == 3 && kw == 3 && (kt == 1 || kt == 3);
}

size_t b2_pack_grouped_conv_weight_elems(int K, int Cin_per_group, int groups, int kt, int kh, int kw) {
  if (!grouped_filter_ok(K, Cin_per_group, groups, kt, kh, kw)) return 0;
  return (size_t)K * group_block(Cin_per_group) * kt * kh * kw;
}

int b2_pack_grouped_conv_weight(const float* w, void* out, int K, int Cin_per_group, int groups, int kt, int kh, int kw, void* stream) {
  B2_CHECK_ARG(w && out, "null pointer");
  const long long total = (long long)b2_pack_grouped_conv_weight_elems(K, Cin_per_group, groups, kt, kh, kw);
  if (total == 0)
    return set_error(B2_ERR_UNSUPPORTED, "grouped packing needs K == C, K %% 64 == 0, 4 / 8 / 16 / 32 channels per group and a 3x3x3 or "
                                         "1x3x3 filter (got K=%d, %d per group, %d groups, %dx%dx%d)", K, Cin_per_group, groups, kt, kh, kw);
  pack_grouped_weight_kernel<<<(unsigned)((total + 255) / 256), 256, 0, reinterpret_cast<cudaStream_t>(stream)>>>(
      w, reinterpret_cast<__half*>(out), Cin_per_group, kt * kh * kw, group_block(Cin_per_group), total);
  B2_CHECK_LAUNCH("pack_grouped_weight_kernel");
  return B2_OK;
}

int b2_conv_grouped_ndhwc_fprop(const b2_conv_args* a, int groups, void* stream) {
  set_last_kernel(KID_NONE);
  int rc = validate_conv(a);
  if (rc != B2_OK) return rc;
  B2_CHECK_ARG(a->mode == B2_CONV_AUTO && !a->out_f32 && !a->accumulate && !a->aff_ld && !a->upsample && !a->residual_up &&
                   !a->residual_pre && !a->y2 && !a->scale2 && !a->shift2 && !a->aff2_ld && !a->pool_w && !a->in_scale && !a->in_shift &&
                   !a->in_aff_ld && !a->mask && !a->ldm,
               "the grouped convolution takes a plain fp16 call: mode, fp32 output, per-sample affines, generator and fine-tuning fields must be zero");
  B2_CHECK_ARG(groups > 0, "groups must be positive");
  const int cg = a->C / groups;
  if (a->C != a->K || a->C % groups || !grouped_filter_ok(a->K, cg, groups, a->kt, a->kh, a->kw) || a->pt != a->kt / 2 || a->ph != 1 ||
      a->pw != 1 || a->sh != a->sw || (a->sh != 1 && a->sh != 2) || (a->st != 1 && a->st != 2))
    return set_error(B2_ERR_UNSUPPORTED, "grouped convolution needs C == K, C %% 64 == 0, 4 / 8 / 16 / 32 channels per group, a 3x3x3 or 1x3x3 "
                                         "'same' filter and strides 1 or 2 (got C=%d K=%d groups=%d, %dx%dx%d, stride %d%d%d, padding %d%d%d)",
                     a->C, a->K, groups, a->kt, a->kh, a->kw, a->st, a->sh, a->sw, a->pt, a->ph, a->pw);
  if ((rc = require_sm90()) != B2_OK) return rc;
  rc = try_slab(a, reinterpret_cast<cudaStream_t>(stream), group_block(cg));
  if (rc == 0) return set_error(B2_ERR_UNSUPPORTED, "no slab tiling of this image fits in shared memory (H=%d W=%d)", a->H, a->W);
  return rc < 0 ? rc : B2_OK;
}

static int gemm_common(const b2_gemm_args* g, const void* a2, int lda2, const void* b2, int ldb2, int k2, void* stream,
                       bool sample_rows = false);

int b2_gemm_f16(const b2_gemm_args* g, void* stream) { return gemm_common(g, nullptr, 0, nullptr, 0, 0, stream); }

int b2_gemm_sample_affine_f16(const b2_gemm_args* g, void* stream) {
  set_last_kernel(KID_NONE);
  B2_CHECK_ARG(g != nullptr && g->scale && g->shift, "null args");
  B2_CHECK_ARG(g->aff_ld > 0 && g->aff_ld % 4 == 0 && g->aff_ld >= g->N && g->aff_rows > 0 &&
                   (reinterpret_cast<uintptr_t>(g->scale) & 15) == 0 && (reinterpret_cast<uintptr_t>(g->shift) & 15) == 0,
               "per-sample affine needs 16-byte aligned fp32 [M / aff_rows][aff_ld] rows, aff_ld %% 4 == 0, aff_ld >= N, aff_rows > 0 "
               "(got pitch %d, rows per sample %d)", g->aff_ld, g->aff_rows);
  B2_CHECK_ARG(g->M > 0 && g->M % g->aff_rows == 0, "M %d is not a whole number of samples of %d rows", g->M, g->aff_rows);
  B2_CHECK_ARG(g->N % 8 == 0, "N %d is not a multiple of 8", g->N);
  B2_CHECK_ARG(!g->out_f32 && !g->per_row && !g->accumulate && !g->d2 && !g->mask,
               "the per-sample-affine GEMM takes fp16 output without per-row affine, accumulation, second output or mask");
  if (g_gemm_algo != 0) return set_error(B2_ERR_UNSUPPORTED, "the per-sample-affine GEMM needs the persistent kernel");
  return gemm_common(g, nullptr, 0, nullptr, 0, 0, stream, true);
}

int b2_gemm2_f16(const b2_gemm_args* g, const void* a2, int lda2, const void* b2, int ldb2, int k2, void* stream) {
  B2_CHECK_ARG(g != nullptr && a2 && b2 && k2 > 0, "null / empty second operand pair");
  B2_CHECK_ARG(lda2 % 8 == 0 && ldb2 % 8 == 0 && lda2 >= k2 && ldb2 >= k2, "bad second operand pitch");
  B2_CHECK_ARG(!g->out_f32 && !g->per_row, "the fused two-operand GEMM produces fp16 output with per-column affine");
  return gemm_common(g, a2, lda2, b2, ldb2, k2, stream);
}

int b2_gemm_chain_f16(const b2_gemm_args* g, const void* a2, int lda2, const void* b2, int ldb2, int k2, const void* w1, int ldw1, int n1,
                      const float* scale1, const float* shift1, void* d1, int ldd1, void* stream) {
  set_last_kernel(KID_NONE);
  B2_CHECK_ARG(g != nullptr && g->a && g->b && g->scale && g->shift && g->d, "null tensor pointer");
  B2_CHECK_ARG(w1 && scale1 && shift1 && d1, "null chained-GEMM pointer");
  B2_CHECK_ARG(g->M > 0 && g->N > 0 && g->Kd > 0 && n1 > 0, "non-positive dimension");
  B2_CHECK_ARG(g->lda % 8 == 0 && g->ldb % 8 == 0 && g->lda >= g->Kd && g->ldb >= g->Kd, "bad operand pitch");
  B2_CHECK_ARG(g->ldd >= g->N && (g->residual == nullptr || (g->ldr % 8 == 0 && g->ldr >= g->N)), "bad output / residual pitch");
  B2_CHECK_ARG(k2 >= 0 && (k2 == 0 || (a2 && b2 && lda2 % 8 == 0 && ldb2 % 8 == 0 && lda2 >= k2 && ldb2 >= k2)), "bad second operand pair");
  B2_CHECK_ARG(ldw1 % 8 == 0 && ldw1 >= g->N && ldd1 % 8 == 0 && ldd1 >= n1, "bad chained-GEMM pitch");
  if (g->out_f32 || g->per_row || g->accumulate || g->aff_ld || g->d2 || g->mask)
    return set_error(B2_ERR_UNSUPPORTED, "the chained GEMM takes fp16 output with a per-column affine, no mask and no second output");
  if (g->N % 64 || g->N > 256 || g->ldd != g->N || ldd1 > 128)
    return set_error(B2_ERR_UNSUPPORTED, "the chained GEMM needs N %% 64 == 0, N <= 256, ldd == N and a chained pitch <= 128 (got %d, %d, %d)",
                     g->N, g->ldd, ldd1);
  if (g_gemm_algo != 0) return set_error(B2_ERR_UNSUPPORTED, "the chained GEMM needs the persistent kernel");
  int rc;
  if ((rc = require_sm90()) != B2_OK) return rc;
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  if (g->N <= 64)
    return ldd1 <= 64 ? launch_pgemm_chain<64, 64>(g, a2, lda2, b2, ldb2, k2, w1, ldw1, n1, scale1, shift1, d1, ldd1, st)
                      : launch_pgemm_chain<64, 128>(g, a2, lda2, b2, ldb2, k2, w1, ldw1, n1, scale1, shift1, d1, ldd1, st);
  return ldd1 <= 64 ? launch_pgemm_chain<128, 64>(g, a2, lda2, b2, ldb2, k2, w1, ldw1, n1, scale1, shift1, d1, ldd1, st)
                    : launch_pgemm_chain<128, 128>(g, a2, lda2, b2, ldb2, k2, w1, ldw1, n1, scale1, shift1, d1, ldd1, st);
}

static int gemm_common(const b2_gemm_args* g, const void* a2, int lda2, const void* b2, int ldb2, int k2, void* stream,
                       bool sample_rows) {
  set_last_kernel(KID_NONE);
  B2_CHECK_ARG(g != nullptr, "null args");
  B2_CHECK_ARG(g->a && g->b && g->scale && g->shift && g->d, "null tensor pointer");
  B2_CHECK_ARG(g->M > 0 && g->N > 0 && g->Kd > 0, "non-positive dimension");
  B2_CHECK_ARG(g->lda % 8 == 0 && g->ldb % 8 == 0 && g->lda >= g->Kd && g->ldb >= g->Kd, "bad operand pitch");
  B2_CHECK_ARG(g->ldd >= g->N, "ldd < N");
  if (!g->out_f32) {
    B2_CHECK_ARG(g->ldd % 8 == 0, "ldd not a multiple of 8");
    B2_CHECK_ARG(!g->accumulate, "accumulate requires out_f32");
    B2_CHECK_ARG(g->residual == nullptr || (g->ldr % 8 == 0 && g->ldr >= g->N), "bad residual pitch");
  }
  int rc;
  if ((rc = require_sm90()) != B2_OK) return rc;

  IgemmLaunch L;
  memset(&L, 0, sizeof(L));
  IgemmParams& p = L.p;
  p.amode = AMODE_TMA;
  p.M_total = g->M;
  p.Ncols = g->N;
  p.nkb = (g->Kd + kBK - 1) / kBK;
  p.scale = g->scale; p.shift = g->shift;
  p.residual = reinterpret_cast<const __half*>(g->residual);
  p.ldr = g->ldr;
  p.y = g->d; p.ldy = g->ldd;
  p.relu = g->relu; p.per_row = g->per_row; p.accumulate = g->accumulate;
  p.epi = g->out_f32 ? EPI_DIRECT_F32 : EPI_TMA_F16;
  B2_CHECK_ARG(sample_rows || (g->aff_ld >= 0 && (g->aff_ld == 0 || (g->aff_ld >= g->N && g->aff_rows > 0 && g->aff_rows % 128 == 0 &&
                                                                     !g->out_f32 && !g->per_row))),
               "bad per-sample affine (pitch %d, rows per sample %d)", g->aff_ld, g->aff_rows);
  p.aff_ld = g->aff_ld; p.aff_rows = g->aff_rows;
  p.mask = reinterpret_cast<const __half*>(g->mask); p.ldm = g->ldm;
  if (g->d2) {
    B2_CHECK_ARG(g->scale2 && g->shift2 && g->aff2_ld >= g->N && g->aff2_rows > 0 && g->aff2_rows % 128 == 0 && !g->out_f32 && !g->per_row,
                 "second output needs scale2 / shift2 (fp32 [M / aff2_rows][aff2_ld >= N], aff2_rows %% 128 == 0) and fp16 output");
    p.y2 = g->d2; p.scale2 = g->scale2; p.shift2 = g->shift2; p.aff2_ld = g->aff2_ld; p.aff2_rows = g->aff2_rows;
  }
  p.x = reinterpret_cast<const __half*>(g->a);
  L.a_mat = g->a; L.lda = g->lda; L.a_cols = g->Kd;
  L.w = g->b; L.ldb = g->ldb; L.b_cols = g->Kd;
  L.a2 = a2; L.lda2 = lda2; L.w2 = b2; L.ldb2 = ldb2; L.k2 = k2;
  if (k2 > 0 && g_gemm_algo != 0) return set_error(B2_ERR_UNSUPPORTED, "two-operand GEMM needs the persistent kernel");
  if (sample_rows) {
    // the only kernel with the per-row sample decode; the dense-M and per-tile kernels never see this epilogue
    g_last_gemm_path = 2;
    const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
    return g->ldd <= 64 ? launch_pgemm<64, 0, 2>(L, st) : launch_pgemm<128, 0, 2>(L, st);
  }
  return dispatch_igemm(L, reinterpret_cast<cudaStream_t>(stream));
}

int b2_gemm_preact_f16(const b2_gemm_args* g, const float* in_scale, const float* in_shift, void* stream) {
  set_last_kernel(KID_NONE);
  B2_CHECK_ARG(g != nullptr && g->a && g->b && g->scale && g->shift && g->d && in_scale && in_shift, "null tensor pointer");
  B2_CHECK_ARG(g->M > 0 && g->N > 0 && g->Kd > 0 && g->Kd % 8 == 0, "non-positive dimension or Kd %d not a multiple of 8", g->Kd);
  B2_CHECK_ARG(g->lda % 8 == 0 && g->ldb % 8 == 0 && g->lda >= g->Kd && g->ldb >= g->Kd, "bad operand pitch");
  B2_CHECK_ARG(g->ldd % 8 == 0 && g->ldd >= g->N, "bad output pitch %d", g->ldd);
  B2_CHECK_ARG((reinterpret_cast<uintptr_t>(in_scale) & 15) == 0 && (reinterpret_cast<uintptr_t>(in_shift) & 15) == 0,
               "in_scale / in_shift must be 16-byte aligned fp32 arrays of round_up(Kd, 64) entries");
  B2_CHECK_ARG(!g->residual && !g->ldr && !g->per_row && !g->out_f32 && !g->accumulate && !g->aff_ld && !g->aff_rows && !g->d2 && !g->mask,
               "the pre-activated GEMM takes fp16 output with a per-column affine: residual, per_row, out_f32, accumulate, aff_ld, d2 "
               "and mask must be zero");
  if (g_gemm_algo != 0) return set_error(B2_ERR_UNSUPPORTED, "the pre-activated GEMM needs the persistent kernel");
  int rc;
  if ((rc = require_sm90()) != B2_OK) return rc;
  IgemmLaunch L;
  memset(&L, 0, sizeof(L));
  IgemmParams& p = L.p;
  p.amode = AMODE_TMA;
  p.M_total = g->M;
  p.Ncols = g->N;
  p.nkb = (g->Kd + kBK - 1) / kBK;
  p.scale = g->scale; p.shift = g->shift;
  p.y = g->d; p.ldy = g->ldd;
  p.relu = g->relu;
  p.epi = EPI_TMA_F16;
  // one per-channel row for every tile: in_ld = 0 makes the transform warps' row offset (m0 / in_rows) * in_ld zero
  p.in_scale = in_scale; p.in_shift = in_shift; p.in_ld = 0; p.in_rows = 128;
  p.x = reinterpret_cast<const __half*>(g->a);
  L.a_mat = g->a; L.lda = g->lda; L.a_cols = g->Kd;
  L.w = g->b; L.ldb = g->ldb; L.b_cols = g->Kd;
  g_last_gemm_path = 2;
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  return g->ldd <= 64 ? launch_pgemm<64, 1>(L, st) : launch_pgemm<128, 1>(L, st);
}

static bool spans_overlap(const void* p, size_t pn, const void* q, size_t qn) {
  const uintptr_t a = reinterpret_cast<uintptr_t>(p), b = reinterpret_cast<uintptr_t>(q);
  return p && q && a < b + qn && b < a + pn;
}

int b2_gemm_dual_f16(const b2_gemm_args* g, const float* scale2, const float* shift2, void* d2, int ldd2, void* stream) {
  set_last_kernel(KID_NONE);
  B2_CHECK_ARG(g != nullptr && g->a && g->b && g->scale && g->shift && g->d && scale2 && shift2 && d2, "null tensor pointer");
  B2_CHECK_ARG(g->M > 0 && g->N > 0 && g->Kd > 0, "non-positive dimension");
  B2_CHECK_ARG(g->lda % 8 == 0 && g->ldb % 8 == 0 && g->lda >= g->Kd && g->ldb >= g->Kd, "bad operand pitch");
  B2_CHECK_ARG(g->ldd % 8 == 0 && g->ldd >= g->N && ldd2 == g->ldd, "bad output pitch (ldd %d, ldd2 %d, N %d): d2 has d's pitch",
               g->ldd, ldd2, g->N);
  B2_CHECK_ARG(g->residual == nullptr || (g->ldr % 8 == 0 && g->ldr >= g->N), "bad residual pitch");
  B2_CHECK_ARG((reinterpret_cast<uintptr_t>(d2) & 15) == 0, "d2 must be 16-byte aligned");
  if (g->out_f32 || g->per_row || g->accumulate || g->aff_ld || g->aff_rows || g->d2 || g->scale2 || g->shift2 || g->aff2_ld ||
      g->aff2_rows || g->mask || g->ldm)
    return set_error(B2_ERR_UNSUPPORTED, "the dual GEMM takes fp16 output with per-column affines: out_f32, per_row, accumulate, "
                     "aff_ld / aff_rows, the args' own d2 / scale2 / shift2 / aff2 fields and mask must be zero");
  // d2 is written while A, the residual and d are live: it may share no byte with them
  const size_t d2n = static_cast<size_t>(g->M) * ldd2 * 2;
  B2_CHECK_ARG(!spans_overlap(d2, d2n, g->d, static_cast<size_t>(g->M) * g->ldd * 2) &&
                   !spans_overlap(d2, d2n, g->a, (static_cast<size_t>(g->M - 1) * g->lda + g->Kd) * 2) &&
                   !spans_overlap(d2, d2n, g->b, (static_cast<size_t>(g->N - 1) * g->ldb + g->Kd) * 2) &&
                   !spans_overlap(d2, d2n, g->residual, (static_cast<size_t>(g->M - 1) * g->ldr + g->N) * 2),
               "d2 overlaps d, A, B or the residual");
  if (g_gemm_algo != 0) return set_error(B2_ERR_UNSUPPORTED, "the dual GEMM needs the persistent kernel");
  int rc;
  if ((rc = require_sm90()) != B2_OK) return rc;
  g_last_gemm_path = 2;
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  // the N tile b2_gemm_f16 picks for an output of this pitch
  return g->ldd <= 64 ? launch_pgemm_dual<64>(g, scale2, shift2, d2, ldd2, st) : launch_pgemm_dual<128>(g, scale2, shift2, d2, ldd2, st);
}

// The split-K planner: N tile as b2_gemm_f16 picks it for an output of pitch round_up(N, 8), at least kSplitkMinKb K blocks of 64 per
// split, at most kSplitkMaxSplits splits.
static constexpr int kSplitkMinKb = 8;
static constexpr int kSplitkMaxSplits = 16;

static int splitk_bn(int N) { return (N + 7) / 8 * 8 <= 64 ? 64 : 128; }

int b2_gemm_splitk_plan(int M, int N, int Kd, int sms) {
  B2_CHECK_ARG(M > 0 && N > 0 && Kd > 0 && sms > 0, "non-positive dimension or SM count");
  const int BN = splitk_bn(N);
  const long long tiles = (long long)((M + 127) / 128) * (((N + 7) / 8 * 8 + BN - 1) / BN);
  if (tiles >= sms) return 1;                    // the output tiles alone fill the SMs
  long long s = sms / tiles;
  const int nkb = (Kd + 63) / 64;
  if (s > nkb / kSplitkMinKb) s = nkb / kSplitkMinKb;
  if (s > kSplitkMaxSplits) s = kSplitkMaxSplits;
  return s < 1 ? 1 : (int)s;
}

size_t b2_gemm_splitk_workspace_elems(int M, int N, int splits) {
  if (M <= 0 || N <= 0 || splits <= 0) return 0;
  return (size_t)splits * M * ((N + 7) / 8 * 8);
}

int b2_gemm_splitk_f16(const b2_gemm_args* g, int splits, float* ws, size_t ws_elems, void* stream) {
  set_last_kernel(KID_NONE);
  B2_CHECK_ARG(g != nullptr && g->a && g->b && g->scale && g->shift && g->d && ws, "null tensor pointer");
  B2_CHECK_ARG(g->M > 0 && g->N > 0 && g->Kd > 0, "non-positive dimension");
  B2_CHECK_ARG(g->lda % 8 == 0 && g->ldb % 8 == 0 && g->lda >= g->Kd && g->ldb >= g->Kd, "bad operand pitch");
  B2_CHECK_ARG(g->out_f32 ? g->ldd >= g->N : (g->ldd % 8 == 0 && g->ldd >= g->N), "bad output pitch (ldd %d, N %d)", g->ldd, g->N);
  const int nkb = (g->Kd + 63) / 64;
  B2_CHECK_ARG(splits >= 1 && splits <= nkb && splits <= 64, "splits %d outside [1, min(64, K blocks %d)]", splits, nkb);
  B2_CHECK_ARG((reinterpret_cast<uintptr_t>(ws) & 15) == 0, "workspace must be 16-byte aligned");
  B2_CHECK_ARG(ws_elems >= b2_gemm_splitk_workspace_elems(g->M, g->N, splits), "workspace of %zu floats, %zu needed", ws_elems,
               b2_gemm_splitk_workspace_elems(g->M, g->N, splits));
  B2_CHECK_ARG(g->residual == nullptr && g->ldr == 0, "the split-K GEMM takes no residual");
  B2_CHECK_ARG(g->mask == nullptr && g->ldm == 0, "the split-K GEMM takes no mask");
  B2_CHECK_ARG(!g->per_row && !g->aff_ld && !g->aff_rows, "the split-K GEMM takes a per-column affine only (no per-row or per-sample affine)");
  B2_CHECK_ARG(!g->d2 && !g->scale2 && !g->shift2 && !g->aff2_ld && !g->aff2_rows, "the split-K GEMM has no second output");
  B2_CHECK_ARG(!g->accumulate, "the split-K GEMM does not accumulate into its output");
  int rc;
  if ((rc = require_sm90()) != B2_OK) return rc;
  g_last_gemm_path = 2;
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  const int ldw = (g->N + 7) / 8 * 8;
  return splitk_bn(g->N) == 64 ? launch_pgemm_splitk<64>(g, splits, ws, ldw, st) : launch_pgemm_splitk<128>(g, splits, ws, ldw, st);
}

int b2_gemm_split_plan(int nd, const int* cols, int* box0) {
  B2_CHECK_ARG(nd >= 1 && nd <= 4 && cols && box0, "a split GEMM has 1 to 4 destinations (got %d)", nd);
  box0[0] = 0;
  for (int d = 0; d < nd; ++d) {
    B2_CHECK_ARG(cols[d] > 0 && cols[d] % 8 == 0, "destination %d: width %d is not a positive multiple of 8", d, cols[d]);
    box0[d + 1] = box0[d] + (cols[d] + 63) / 64;
  }
  return box0[nd] * 64;
}

int b2_gemm_split_f16(const b2_gemm_args* g, int nd, void* const* y, const int* ldy, const int* cols, void* stream) {
  set_last_kernel(KID_NONE);
  int box0[5];
  const int Npad = b2_gemm_split_plan(nd, cols, box0);
  if (Npad < 0) return Npad;
  B2_CHECK_ARG(g != nullptr && g->a && g->b && g->scale && g->shift && y && ldy, "null tensor pointer");
  B2_CHECK_ARG(g->M > 0 && g->Kd > 0, "non-positive dimension");
  B2_CHECK_ARG(g->N == Npad, "N %d is not the packed width %d of the destinations (whole 64-column boxes each)", g->N, Npad);
  B2_CHECK_ARG(g->lda % 8 == 0 && g->ldb % 8 == 0 && g->lda >= g->Kd && g->ldb >= g->Kd, "bad operand pitch");
  B2_CHECK_ARG(!g->d && !g->ldd && !g->residual && !g->out_f32 && !g->per_row && !g->accumulate && !g->aff_ld && !g->d2 && !g->mask,
               "the split GEMM writes fp16 through its destinations with a per-column affine: d, ldd, residual, out_f32, per_row, "
               "accumulate, aff_ld, d2 and mask must be zero");
  for (int d = 0; d < nd; ++d) {
    B2_CHECK_ARG(y[d] != nullptr && (reinterpret_cast<uintptr_t>(y[d]) & 15) == 0, "destination %d is null or not 16-byte aligned", d);
    B2_CHECK_ARG(ldy[d] % 8 == 0 && ldy[d] >= cols[d], "destination %d: pitch %d is not a multiple of 8 >= its width %d", d, ldy[d], cols[d]);
  }
  if (g_gemm_algo != 0) return set_error(B2_ERR_UNSUPPORTED, "the split GEMM needs the persistent kernel");
  int rc;
  if ((rc = require_sm90()) != B2_OK) return rc;
  g_last_gemm_path = 2;
  const cudaStream_t st = reinterpret_cast<cudaStream_t>(stream);
  // the N tile b2_gemm_f16 picks for an output of this width
  return Npad <= 64 ? launch_pgemm_split<64>(g, nd, y, ldy, cols, box0, st) : launch_pgemm_split<128>(g, nd, y, ldy, cols, box0, st);
}

static int conv_slice(const b2_conv_args* a, void* stream, int narrow) {
  set_last_kernel(KID_NONE);
  int rc = validate_conv(a);
  if (rc != B2_OK) return rc;
  B2_CHECK_ARG(a->mode == B2_CONV_AUTO && !a->mask && !a->ldm && !a->aff_ld && !a->upsample && !a->y2 && !a->scale2 && !a->shift2 &&
                   !a->aff2_ld && !a->pool_w && !a->residual_up && !a->residual_pre && !a->in_scale && !a->in_shift && !a->in_aff_ld &&
                   !a->out_f32 && !a->accumulate,
               "the slice convolution takes a plain fp16 call: stem mode, mask, per-sample affine, upsampling, second output, pool_w, "
               "generator fields and fp32 output must be zero");
  B2_CHECK_ARG(a->kt == 1 && a->pt == 0 && a->st == 1 && (a->kh & 1) && (a->kw & 1) && a->kh * a->kw > 1 && a->kh * a->kw <= kSlabMaxTaps &&
                   a->ph >= 0 && 2 * a->ph <= a->kh - 1 && a->pw >= 0 && 2 * a->pw <= a->kw - 1 && a->sh == a->sw && (a->sh == 1 || a->sh == 2),
               "the slice convolution is a 2-D convolution with an odd kh x kw filter other than 1x1 (at most %d taps), padding from 0 to "
               "(k - 1) / 2 per axis and stride 1 or 2 (got %dx%dx%d, stride %d%d%d, padding %d%d%d)",
               kSlabMaxTaps, a->kt, a->kh, a->kw, a->st, a->sh, a->sw, a->pt, a->ph, a->pw);
  B2_CHECK_ARG(a->K % 8 == 0, "slice width K %d is not a multiple of 8", a->K);
  B2_CHECK_ARG(!narrow || a->K == narrow, "the narrow slice convolution takes K = 32 or 48 output channels (got %d)", a->K);
  B2_CHECK_ARG((reinterpret_cast<uintptr_t>(a->y) & 15) == 0, "slice start is not 16-byte aligned");
  if ((rc = require_sm90()) != B2_OK) return rc;
  g_last_conv_path = 0;
  g_last_gemm_path = 0;
  b2_conv_args s = *a;
  s.ldy = a->K;                         // the slab planner and epilogue see the slice width; ldo carries the row pitch
  rc = try_slab(&s, reinterpret_cast<cudaStream_t>(stream), 0, a->ldy, narrow);
  if (rc == 0) return set_error(B2_ERR_UNSUPPORTED, "no slab tiling of this image fits in shared memory (H=%d W=%d)", a->H, a->W);
  return rc < 0 ? rc : B2_OK;
}

int b2_conv_ndhwc_fprop_slice(const b2_conv_args* a, void* stream) { return conv_slice(a, stream, 0); }

int b2_conv_ndhwc_fprop_slice_narrow(const b2_conv_args* a, void* stream) {
  if (a != nullptr && a->K != 32 && a->K != 48) {
    set_last_kernel(KID_NONE);
    return set_error(B2_ERR_INVALID, "the narrow slice convolution takes K = 32 or 48 output channels (got %d)", a->K);
  }
  return conv_slice(a, stream, a ? a->K : 0);
}

}  // extern "C"
