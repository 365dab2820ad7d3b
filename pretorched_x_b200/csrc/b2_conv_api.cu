// b2_conv_api.cu -- C-ABI entry points for the wgmma implicit-GEMM convolution and the dense GEMM,
// plus library-wide error/launch bookkeeping and the CUtensorMap builder.
#include <atomic>
#include <mutex>
#include <stdlib.h>
#include <string.h>

#include "b2_host.h"
#include "b2_igemm.cuh"
#include "b2_densem.cuh"
#include "b2_pgemm.cuh"
#include "b2_slabconv.cuh"
#include "b2_slabts.cuh"
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
// slab convolution launcher (stride 1, "same" padding)
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
  if (a->pt != (a->kt - 1) / 2 || a->ph != (a->kh - 1) / 2 || a->pw != (a->kw - 1) / 2) return false;
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
  int min_oj = 0, max_oj = 0;
  for (int d = 0; d < a->kh; ++d) { int v = d - a->ph; rh[d] = ((v % ss) + ss) % ss; oi[d] = (v - rh[d]) / ss; }
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
            const int off = oi[dh] * p->PW + oj[dw];
            p->sub_off[sidx][n] = (short)off;
            p->sub_tap[sidx][n] = (unsigned char)(dh * a->kw + dw);
            if (off > p->reach) p->reach = off;
            if (-off > p->reach) p->reach = -off;
            ++n;
          }
      if (n == 0) continue;
      p->sub_ntaps[sidx] = n;
      p->sub_h0[sidx] = ph_;                               // + ss * r_lo at run time
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

template <int BNT>   // BNT = 0: runtime N tile p.bn (set by the caller)
static int launch_slab(const b2_conv_args* a, SlabParams& p, int MT, int R, cudaStream_t stream) {
  if (BNT) { p.bn = BNT; p.wbytes = BNT * 128; p.accs = BNT; }
  const int BN = p.bn;
  p.R = R;
  p.planes_total = a->N * p.To;
  p.plane_stride = R * p.PW * 128;
  p.slab_bytes = ((R * p.PW * 128 * (p.mp > 1 ? p.mp : 1)) + 1023) / 1024 * 1024;
  p.MT = MT;
  if (MT * BN > kSlabAccCols)
    return set_error(B2_ERR_INVALID, "slab plan MT=%d x N=%d exceeds the %d register accumulator columns", MT, BN, kSlabAccCols);
  if (!BNT && BN != 16 && (BN < 144 || BN > kSlabAccCols || BN % 16 != 0))
    return set_error(B2_ERR_INVALID, "slab runtime N tile %d is not one of the compiled widths", BN);
  p.Ncols = a->K;
  p.scale = a->scale; p.shift = a->shift;
  p.residual = reinterpret_cast<const __half*>(a->residual);
  p.ldr = a->ldr;
  p.y = reinterpret_cast<__half*>(a->y);
  p.ldy = a->ldy;
  p.relu = a->relu;
  p.aff_ld = a->aff_ld;
  p.naff = slab_naff(a->ldy);
  p.tiles_n = (a->ldy + BN - 1) / BN;
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
  B2_OPT_IN_SMEM(slabconv_kernel<BNT>, 227 * 1024);
  CUtensorMap tmX, tmB;
  int rc;
  const int taps = p.up ? 16 : a->kt * a->kh * a->kw;
  if ((rc = make_tmap_ndhwc_slab(&tmX, a->x, (uint64_t)a->C, (uint64_t)a->W, (uint64_t)a->H, (uint64_t)a->N * a->T,
                                 (uint32_t)p.PW, (uint32_t)R, (uint32_t)p.ss, (uint32_t)(p.mp > 1 ? p.mp : 1))) != B2_OK)
    return rc;
  if ((rc = make_tmap_2d_f16(&tmB, a->w, (uint64_t)taps * a->C, (uint64_t)a->K, (uint64_t)taps * a->C, 64, BN, true)) != B2_OK)
    return rc;
  const int grid = p.items_total < sm_count() ? p.items_total : sm_count();
  B2_CHECK_CUDA(launch_pdl(slabconv_kernel<BNT>, dim3(grid), dim3(kSlabThreads), smem_bytes, stream, tmX, tmB, p));
  B2_CHECK_LAUNCH("slabconv_kernel");
  return B2_OK;
}

// Picks the N tile (fixed 64 / 128 or runtime), the M tiles per work item and the slab rows for a geometry; *best_mt == 0
// when no configuration fits in shared memory.
static double slab_pick_tiles(const b2_conv_args* a, SlabParams& p, int* BN_out, bool* flex_out, int* best_mt_out, int* best_R_out) {
  int BN = (a->ldy <= 64) ? 64 : 128;
  const int planes = a->N * p.To;
  int ntn = (a->ldy + BN - 1) / BN;
  // Channel counts that tile badly by 128 (144, 288, 576 ... of R(2+1)D) take the runtime-N instance: the fewest
  // tiles of <= 256 columns, each a multiple of 16 wide.
  bool flex = false;
  if (a->ldy > 128) {
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
  const int w_stage = flex ? p.wbytes : BN * 128;
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

// returns 1 when the slab kernel took the convolution, 0 when it does not apply, <0 on error
static int try_slab(const b2_conv_args* a_in, cudaStream_t stream) {
  if (g_conv_algo == 1) return 0;
  SlabParams p;
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
  // W chunking candidates: the default (whole rows, or <= 256-pixel chunks) and narrower chunks.  Narrow chunks make the
  // slab of a work item shorter, which (a) lets 256-pixel rows fit the two slab stages at all and (b) admits more M tiles
  // per item for wide images -- with few-tap 2-D filters the per-item costs (decode, epilogue set-up, slab latency) are
  // what the cycle model trades against the extra halo columns.  The cheapest modelled configuration wins.
  const int wc_try[3] = {wc_hint, 128, 64};
  int BN = 0, best_mt = 0, best_R = 0;
  bool flex = false;
  double best_cost = 0.0;
  SlabParams best_p;
  for (int attempt = 0; attempt < 3; ++attempt) {
    if (attempt > 0 && (wc_hint > 0 || wc_try[attempt] >= a->W)) continue;
    SlabParams q;
    if (!slab_geometry(a, &q, wc_try[attempt])) { if (attempt == 0) return 0; else continue; }
    if (attempt > 0 && q.wchunks == 1) continue;              // same geometry as the default
    if (g_conv_algo == 2 && q.ss != 1) return 0;              // debug: strided convs through the gather kernel
    int bn_c = 0, mt_c = 0, r_c = 0;
    bool flex_c = false;
    const double cost = slab_pick_tiles(a, q, &bn_c, &flex_c, &mt_c, &r_c);
    if (mt_c == 0) continue;
    if (best_mt == 0 || cost < best_cost) { best_p = q; BN = bn_c; flex = flex_c; best_mt = mt_c; best_R = r_c; best_cost = cost; }
  }
  if (best_mt != 0) p = best_p;
  if (best_mt == 0) return 0;
  int rc = flex ? launch_slab<0>(a, p, best_mt, best_R, stream)
                : (BN == 64) ? launch_slab<64>(a, p, best_mt, best_R, stream) : launch_slab<128>(a, p, best_mt, best_R, stream);
  return rc == B2_OK ? 1 : rc;
}


// ------------------------------------------------------------------------------------------
// temporal-group slab kernel (b2_slabts.cuh): 3 x kh x kw stride-1 "same" convolutions with <= 64 output channels
// ------------------------------------------------------------------------------------------
static int g_slabts = -1;     // B2_SLABTS=0 disables (A/B measurements)
static int try_slabts(const b2_conv_args* a, cudaStream_t stream) {
  if (g_slabts < 0) { const char* e = getenv("B2_SLABTS"); g_slabts = (e && e[0] == '0') ? 0 : 1; }
  if (!g_slabts || g_conv_algo != 0) return 0;
  if (a->mode != B2_CONV_AUTO || a->out_f32 || a->upsample || a->aff_ld || a->y2 || a->residual_up || a->residual_pre || a->in_scale) return 0;
  if (a->kt != 3 || a->st != 1 || a->pt != 1 || a->sh != 1 || a->sw != 1 || a->ldy > 64 || a->T < 3) return 0;
  // The operand traffic it saves in shared memory comes back as 2.5x more weight bytes per output tile from L2 (one 24 KB stack per
  // tap and input frame), the single accumulator set exposes a residual read, and with a 1x1 in-plane filter the frames-as-rows remap
  // of the slab kernel has less to gain from.  So: true 3-D filters without a residual only.
  if (a->kh * a->kw < 9 || a->residual) return 0;
  SlabParams p;
  if (!slab_geometry(a, &p, 0) || p.n_sub != 1) return 0;
  // one M tile per item: its 3 x 64 accumulator columns are what the consumers' registers hold (kSlabAccCols)
  const int R = slab_rows(1, p.PW, p.reach, p.P);
  const long long slab_b = ((long long)R * p.PW * 128 + 1023) / 1024 * 1024;
  const long long smem = kSlabSStages * slab_b + kSlabWStages * kTsWBytes + 256 + 2 * slab_naff(a->ldy) * 4 + 1024 +
                         acc_bytes(kTsGroup * kTsBN);
  if (R > 256 || smem > 227 * 1024) return 0;
  p.R = R;
  p.planes_total = a->N * p.To;
  p.plane_stride = R * p.PW * 128;
  p.slab_bytes = (int)slab_b;
  p.MT = 1; p.bn = kTsBN; p.wbytes = kTsWBytes; p.accs = kTsBN;
  p.Ncols = a->K;
  p.scale = a->scale; p.shift = a->shift;
  p.residual = reinterpret_cast<const __half*>(a->residual);
  p.ldr = a->ldr;
  p.y = reinterpret_cast<__half*>(a->y);
  p.ldy = a->ldy;
  p.relu = a->relu;
  p.naff = slab_naff(a->ldy);
  p.tiles_n = 1;
  p.tiles_q = (p.P + 127) / 128;
  const int groups = (p.To + kTsGroup - 1) / kTsGroup;
  const long long items = (long long)p.tiles_q * p.wchunks * a->N * groups;
  if (items >= (1ll << 31)) return 0;
  p.items_total = (int)items;
  p.fd_tiles_n = make_fastdiv(1); p.fd_tiles_q = make_fastdiv(p.tiles_q); p.fd_wchunks = make_fastdiv(p.wchunks);
  p.fd_To = make_fastdiv(groups); p.fd_PW = make_fastdiv(p.PW);
  B2_OPT_IN_SMEM(slabts_kernel, 227 * 1024);
  CUtensorMap tmX, tmB;
  int rc;
  const int taps = a->kt * a->kh * a->kw;
  if ((rc = make_tmap_ndhwc_slab(&tmX, a->x, (uint64_t)a->C, (uint64_t)a->W, (uint64_t)a->H, (uint64_t)a->N * a->T, (uint32_t)p.PW,
                                 (uint32_t)R, 1u)) != B2_OK) return rc;
  if ((rc = make_tmap_2d_f16(&tmB, a->w, (uint64_t)taps * a->C, (uint64_t)a->K, (uint64_t)taps * a->C, 64, kTsBN, true)) != B2_OK) return rc;
  const int grid = p.items_total < sm_count() ? p.items_total : sm_count();
  B2_CHECK_CUDA(launch_pdl(slabts_kernel, dim3(grid), dim3(kSlabThreads), (size_t)smem, stream, tmX, tmB, p));
  B2_CHECK_LAUNCH("slabts_kernel");
  return 1;
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
  return 1;
}

// ------------------------------------------------------------------------------------------
// stem convolution launcher (Toeplitz-descriptor kernel)
// ------------------------------------------------------------------------------------------
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
  p.G = kStemAccCols / BN;
  p.rows = 2 * (p.G - 1) + a->kh;
  if (p.rows > kStemMaxRows) return set_error(B2_ERR_UNSUPPORTED, "stem kernel height %d too large", a->kh);
  for (int i = 0; i < p.rows; ++i) {
    int g_lo = i - (a->kh - 1);
    g_lo = g_lo > 0 ? (g_lo + 1) / 2 : 0;
    int g_hi = i / 2;
    if (g_hi > p.G - 1) g_hi = p.G - 1;
    p.row_glo[i] = (signed char)g_lo;
    p.row_ghi[i] = (signed char)g_hi;
    p.row_slot[i] = (signed char)(g_lo <= g_hi ? stem_slot(i - 2 * g_lo, a->kh) : 0);
  }
  p.w_bytes = a->kh * BN * 64;
  p.stage_bytes = ((p.rows * kStemPitch + p.w_bytes) + 127) / 128 * 128;
  const int tail_bytes = kStemTailBytes + 128;                  // + alignment of the dynamic shared-memory base
  p.nstages = (227 * 1024 - tail_bytes) / p.stage_bytes;
  if (p.nstages > kStemMaxStages) p.nstages = kStemMaxStages;
  if (p.nstages < 1) return set_error(B2_ERR_UNSUPPORTED, "stem slab does not fit in shared memory (kh=%d)", a->kh);
  p.Ncols = a->K;
  p.ntiles_n = (a->ldy + BN - 1) / BN;
  if (p.ntiles_n * BN > 256) return set_error(B2_ERR_UNSUPPORTED, "stem convolution supports at most 256 output channels");
  p.tiles_w = (p.Wo + kStemTileW - 1) / kStemTileW;
  p.tiles_h = (p.Ho + p.G - 1) / p.G;
  static int pair_env = -1;
  if (pair_env < 0) { const char* e = getenv("B2_STEM_PAIR"); pair_env = (e && e[0] == '0') ? 0 : 1; }
  p.planes_total = a->N * p.To;
  p.pair = (pair_env && a->kt == 1 && a->pt == 0 && p.Wo <= 60 && !a->pool_w && a->W <= 120) ? 1 : 0;
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
  B2_OPT_IN_SMEM((stemconv_kernel<BN, false>), 227 * 1024);
  B2_OPT_IN_SMEM((stemconv_kernel<BN, true>), 227 * 1024);
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
  const int grid = p.items_total < sm_count() ? p.items_total : sm_count();
  if (p.nstages == 1) B2_CHECK_CUDA(launch_pdl(stemconv_kernel<BN, true>, dim3(grid), dim3(kStemThreads), smem_bytes, stream, tmX, p));
  else B2_CHECK_CUDA(launch_pdl(stemconv_kernel<BN, false>, dim3(grid), dim3(kStemThreads), smem_bytes, stream, tmX, p));
  B2_CHECK_LAUNCH("stemconv_kernel");
  return B2_OK;
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
      if ((rc = make_tmap_2d_f16(&tmR, p.residual, (uint64_t)p.ldr, (uint64_t)p.M_total, (uint64_t)p.ldr, 64, kBM, true)) != B2_OK)
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
  if (ip.residual && ip.res_up) {
    // low-res skip tensor: a tile's 128 output rows read res_rows consecutive rows of it (see PgemmParams::res_up)
    if (!(up_W % 128 == 0 || (up_W <= 64 && 64 % up_W == 0)))
      return set_error(B2_ERR_UNSUPPORTED, "residual_up needs an output width that is a multiple of 128 or divides 64 (got %d)", up_W);
    if ((rc = make_tmap_2d_f16(&tmR, ip.residual, (uint64_t)ip.ldr, (uint64_t)ip.M_total / 4, (uint64_t)ip.ldr, 64, res_rows, true)) != B2_OK) return rc;
  } else if (ip.residual) {
    if ((rc = make_tmap_2d_f16(&tmR, ip.residual, (uint64_t)ip.ldr, (uint64_t)ip.M_total, (uint64_t)ip.ldr, 64, 128, true)) != B2_OK) return rc;
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
  const int grid = p.tiles_total < sm_count() ? p.tiles_total : sm_count();
  B2_CHECK_CUDA(launch_pdl(pgemm_kernel<BN, GAN, MASK>, dim3(grid), dim3(GAN ? kPgThreadsGan : kPgThreads), S::kTotal, stream, tmA, tmB, tmA2, tmB2, tmC, tmR, tmC2, p));
  B2_CHECK_LAUNCH("pgemm_kernel");
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
   WC, wchunks, items, flex, remapped}.  Used by tests/test_host_logic.py and by tuning scripts. */
int b2_debug_slab_plan(const b2_conv_args* a_in, int* out) {
  b2_conv_args remap = *a_in;
  const b2_conv_args* a = a_in;
  int wc_hint = 0, remapped = 0;
  if (a_in->kt > 1 && a_in->kh == 1 && a_in->kw == 1 && a_in->st == 1 && a_in->sh == 1 && a_in->sw == 1 && a_in->ph == 0 && a_in->pw == 0) {
    remap.T = 1; remap.H = a_in->T; remap.W = a_in->H * a_in->W; remap.kt = 1; remap.kh = a_in->kt; remap.kw = 1;
    remap.pt = 0; remap.ph = a_in->pt; remap.pw = 0; a = &remap; wc_hint = 64; remapped = 1;
  }
  const int wc_try[3] = {wc_hint, 128, 64};
  int BN = 0, best_mt = 0, best_R = 0; bool flex = false; double best_cost = 0.0; SlabParams best_p;
  memset(&best_p, 0, sizeof(best_p));
  for (int attempt = 0; attempt < 3; ++attempt) {
    if (attempt > 0 && (wc_hint > 0 || wc_try[attempt] >= a->W)) continue;
    SlabParams q;
    if (!slab_geometry(a, &q, wc_try[attempt])) { if (attempt == 0) break; else continue; }
    if (attempt > 0 && q.wchunks == 1) continue;
    int bn_c = 0, mt_c = 0, r_c = 0; bool flex_c = false;
    const double cost = slab_pick_tiles(a, q, &bn_c, &flex_c, &mt_c, &r_c);
    if (mt_c == 0) continue;
    if (best_mt == 0 || cost < best_cost) { best_p = q; BN = bn_c; flex = flex_c; best_mt = mt_c; best_R = r_c; best_cost = cost; }
  }
  out[0] = best_mt != 0; out[1] = BN; out[2] = best_mt; out[3] = best_R; out[4] = best_p.PW; out[5] = best_p.WC; out[6] = best_p.wchunks;
  const long long tq = best_mt ? (best_p.P + best_mt * 128 - 1) / (best_mt * 128) : 0;
  out[7] = (int)(((a->ldy + BN - 1) / (BN ? BN : 1)) * tq * best_p.wchunks * a->N * best_p.To);
  out[8] = flex; out[9] = remapped;
  return B2_OK;
}
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
int b2_debug_last_gemm_path(void) { return g_last_gemm_path; }   /* 1 dense-M, 2 persistent GEMM, 3 implicit GEMM (last GEMM-family launch) */   /* 1: the temporal stack kernel took the last convolution */
int b2_debug_set_tstack(int mode) { g_tstack = mode < -1 ? -1 : (mode > 1 ? 1 : mode); return B2_OK; }   /* temporal stack kernel: -1 rule, 0 never, 1 whenever eligible */
int b2_debug_set_slab_mt(int mt) { g_slab_force_mt = mt < 0 ? 0 : mt; return B2_OK; }
int b2_debug_set_densem(int maxm, int force_s) { g_densem_maxm = maxm < 0 ? -2 : maxm; g_densem_force_s = force_s; return B2_OK; }
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
  rc = skip_slab ? 0 : try_slabts(a, reinterpret_cast<cudaStream_t>(stream));
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

static int gemm_common(const b2_gemm_args* g, const void* a2, int lda2, const void* b2, int ldb2, int k2, void* stream);

int b2_gemm_f16(const b2_gemm_args* g, void* stream) { return gemm_common(g, nullptr, 0, nullptr, 0, 0, stream); }

int b2_gemm2_f16(const b2_gemm_args* g, const void* a2, int lda2, const void* b2, int ldb2, int k2, void* stream) {
  B2_CHECK_ARG(g != nullptr && a2 && b2 && k2 > 0, "null / empty second operand pair");
  B2_CHECK_ARG(lda2 % 8 == 0 && ldb2 % 8 == 0 && lda2 >= k2 && ldb2 >= k2, "bad second operand pitch");
  B2_CHECK_ARG(!g->out_f32 && !g->per_row, "the fused two-operand GEMM produces fp16 output with per-column affine");
  return gemm_common(g, a2, lda2, b2, ldb2, k2, stream);
}

static int gemm_common(const b2_gemm_args* g, const void* a2, int lda2, const void* b2, int ldb2, int k2, void* stream) {
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
  B2_CHECK_ARG(g->aff_ld >= 0 && (g->aff_ld == 0 || (g->aff_ld >= g->N && g->aff_rows > 0 && g->aff_rows % 128 == 0 &&
                                                     !g->out_f32 && !g->per_row)),
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
  return dispatch_igemm(L, reinterpret_cast<cudaStream_t>(stream));
}

}  // extern "C"
