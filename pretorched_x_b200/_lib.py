"""ctypes binding of libb2pretorched.so -- the C-ABI boundary declared in include/b2_pretorched.h.

This is the only place Python touches native code.  There is deliberately no fallback: if the shared
library is missing it is built with nvcc (sm_90a); if that is impossible, or a compute entry point
is called without an H100, a RuntimeError carrying b2_last_error() is raised.
"""
import ctypes
import os
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "csrc", "libb2pretorched.so")
_lock = threading.Lock()
_lib = None

B2_OK = 0
# The ABI revision this binding was written against (b2_version() of csrc/b2_conv_api.cu).  The argument structs below
# mirror that revision; a library from another checkout would silently ignore / misread fields, so load() insists on it.
EXPECTED_ABI = 103
B2_CONV_AUTO = 0
B2_CONV_STEM7 = 1

c_void_p = ctypes.c_void_p
c_int = ctypes.c_int
c_i32 = ctypes.c_int32


class ConvArgs(ctypes.Structure):
    """Mirror of `struct b2_conv_args` (include/b2_pretorched.h)."""
    _fields_ = [
        ("x", c_void_p), ("w", c_void_p), ("scale", c_void_p), ("shift", c_void_p),
        ("residual", c_void_p), ("y", c_void_p),
        ("N", c_i32), ("T", c_i32), ("H", c_i32), ("W", c_i32), ("C", c_i32),
        ("K", c_i32), ("ldy", c_i32), ("ldr", c_i32),
        ("kt", c_i32), ("kh", c_i32), ("kw", c_i32),
        ("st", c_i32), ("sh", c_i32), ("sw", c_i32),
        ("pt", c_i32), ("ph", c_i32), ("pw", c_i32),
        ("relu", c_i32), ("out_f32", c_i32), ("accumulate", c_i32), ("mode", c_i32), ("aff_ld", c_i32), ("upsample", c_i32), ("residual_up", c_i32), ("residual_pre", c_i32),
        ("y2", c_void_p), ("scale2", c_void_p), ("shift2", c_void_p), ("aff2_ld", c_i32), ("pool_w", c_i32),
        ("in_scale", c_void_p), ("in_shift", c_void_p), ("in_aff_ld", c_i32),
        ("mask", c_void_p), ("ldm", c_i32),
    ]


class GemmArgs(ctypes.Structure):
    """Mirror of `struct b2_gemm_args`."""
    _fields_ = [
        ("a", c_void_p), ("b", c_void_p), ("scale", c_void_p), ("shift", c_void_p),
        ("residual", c_void_p), ("d", c_void_p),
        ("M", c_i32), ("N", c_i32), ("Kd", c_i32),
        ("lda", c_i32), ("ldb", c_i32), ("ldd", c_i32), ("ldr", c_i32),
        ("per_row", c_i32), ("relu", c_i32), ("out_f32", c_i32), ("accumulate", c_i32),
        ("aff_ld", c_i32), ("aff_rows", c_i32),
        ("d2", c_void_p), ("scale2", c_void_p), ("shift2", c_void_p), ("aff2_ld", c_i32), ("aff2_rows", c_i32),
        ("mask", c_void_p), ("ldm", c_i32),
    ]


# name -> (restype, argtypes); every symbol include/b2_pretorched.h declares
SYMBOLS = {
    "b2_version": (c_int, []),
    "b2_last_error": (ctypes.c_char_p, []),
    "b2_launch_count": (ctypes.c_uint64, []),
    "b2_conv_ndhwc_fprop": (c_int, [ctypes.POINTER(ConvArgs), c_void_p]),
    "b2_conv_ndhwc_fprop_simt": (c_int, [ctypes.POINTER(ConvArgs), c_void_p]),
    "b2_pack_conv_weight_elems": (ctypes.c_size_t, [c_int] * 7),
    "b2_pack_conv_weight": (c_int, [c_void_p, c_void_p] + [c_int] * 7 + [c_void_p]),
    "b2_pack_upconv3x3_weight": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "b2_gemm_f16": (c_int, [ctypes.POINTER(GemmArgs), c_void_p]),
    "b2_gemm2_f16": (c_int, [ctypes.POINTER(GemmArgs), c_void_p, c_int, c_void_p, c_int, c_int, c_void_p]),
    "b2_gemm_chain_f16": (c_int, [ctypes.POINTER(GemmArgs), c_void_p, c_int, c_void_p, c_int, c_int, c_void_p, c_int, c_int,
                                  c_void_p, c_void_p, c_void_p, c_int, c_void_p]),
    "b2_nonlocal_attention": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_void_p, c_int,
                                      c_int, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "b2_maxpool3d_ndhwc": (c_int, [c_void_p, c_void_p] + [c_int] * 14 + [c_void_p]),
    "b2_avgpool_global_ndhwc": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "b2_ncdhw_f32_to_ndhwc_f16": (c_int, [c_void_p, c_void_p] + [c_int] * 6 + [c_void_p]),
    "b2_ncdhw_f16_to_ndhwc_f16": (c_int, [c_void_p, c_void_p] + [c_int] * 6 + [c_void_p]),
    "b2_ndhwc_f16_to_ncdhw_f32": (c_int, [c_void_p, c_void_p] + [c_int] * 6 + [c_void_p]),
    "b2_cast_f32_to_f16": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "b2_shortcut_a_ndhwc": (c_int, [c_void_p, c_void_p] + [c_int] * 7 + [c_void_p]),
    "b2_concat_channels": (c_int, [c_void_p, c_int, c_int, c_void_p, c_int, c_int, c_void_p, c_int, ctypes.c_longlong, c_void_p]),
    "b2_gather_frames": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "b2_gather_frame_tuples": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "b2_transform_image_u8": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_int, c_int,
                                      c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "b2_u8_frames_to_ndhwc4_f16": (c_int, [c_void_p, c_void_p, ctypes.c_longlong, c_int, c_void_p, c_void_p, c_void_p]),
    "b2_embed_concat": (c_int, [c_void_p] * 5 + [c_int] * 6 + [c_void_p]),
    "b2_ccbn_act_ndhwc": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p] + [c_int] * 7 + [c_void_p]),
    "b2_rgb_head_gather_tanh": (c_int, [c_void_p, c_int, c_void_p, c_void_p] + [c_int] * 5 + [c_void_p]),
    "b2_tanh_nhwc_to_nchw": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, ctypes.c_longlong, c_int, c_void_p]),
    "b2_conv_wgrad_workspace_elems": (ctypes.c_size_t, [c_int] * 9),
    "b2_conv_wgrad": (c_int, [c_void_p, c_int, c_void_p, c_int] + [c_void_p] * 6 + [ctypes.c_size_t] + [c_int] * 9 + [c_void_p]),
    "b2_conv_wgrad_thw_workspace_elems": (ctypes.c_size_t, [c_int] * 13),
    "b2_conv_wgrad_thw": (c_int, [c_void_p, c_int, c_void_p, c_int] + [c_void_p] * 6 + [ctypes.c_size_t] + [c_int] * 13 + [c_void_p]),
    "b2_zero_insert_ndhwc": (c_int, [c_void_p, c_int, c_int, c_void_p] + [c_int] * 6 + [c_void_p]),
    "b2_colsum_workspace_elems": (ctypes.c_size_t, [c_int]),
    "b2_colsum_f16": (c_int, [c_void_p, c_int, ctypes.c_longlong, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "b2_loss_scale_f32": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "b2_avgpool_global_backward": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p] + [c_int] * 4 + [c_void_p]),
    "b2_dwconv3x3_ndhwc": (c_int, [c_void_p] * 5 + [c_int] * 8 + [c_void_p]),
    "b2_relu6_inplace_ndhwc": (c_int, [c_void_p, ctypes.c_longlong, c_int, c_void_p]),
    "b2_pack_grouped_conv_weight_elems": (ctypes.c_size_t, [c_int] * 6),
    "b2_pack_grouped_conv_weight": (c_int, [c_void_p, c_void_p] + [c_int] * 6 + [c_void_p]),
    "b2_conv_grouped_ndhwc_fprop": (c_int, [ctypes.POINTER(ConvArgs), c_int, c_void_p]),
    "b2_gemm_sample_affine_f16": (c_int, [ctypes.POINTER(GemmArgs), c_void_p]),
    "b2_maxpool3d_ndhwc_out": (c_int, [c_void_p, c_void_p] + [c_int] * 17 + [c_void_p]),
    "b2_se_excite_workspace_elems": (ctypes.c_size_t, [c_int] * 3),
    "b2_se_excite": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p,
                             c_void_p, c_void_p, c_void_p, c_int, c_void_p, ctypes.c_size_t, c_void_p]),
    "b2_gemm_split_plan": (c_int, [c_int, ctypes.POINTER(c_int), ctypes.POINTER(c_int)]),
    "b2_gemm_split_f16": (c_int, [ctypes.POINTER(GemmArgs), c_int, ctypes.POINTER(c_void_p), ctypes.POINTER(c_int),
                                  ctypes.POINTER(c_int), c_void_p]),
    "b2_conv_ndhwc_fprop_slice": (c_int, [ctypes.POINTER(ConvArgs), c_void_p]),
    "b2_conv_ndhwc_fprop_slice_narrow": (c_int, [ctypes.POINTER(ConvArgs), c_void_p]),
    "b2_pool_ndhwc_slice": (c_int, [c_void_p, c_int, c_void_p] + [c_int] * 19 + [c_void_p]),
    "b2_avgpool_ndhwc_slice_exclude_pad": (c_int, [c_void_p, c_int, c_void_p] + [c_int] * 18 + [c_void_p]),
    "b2_gemm_preact_f16": (c_int, [ctypes.POINTER(GemmArgs), c_void_p, c_void_p, c_void_p]),
    "b2_gemm_dual_f16": (c_int, [ctypes.POINTER(GemmArgs), c_void_p, c_void_p, c_void_p, c_int, c_void_p]),
    "b2_bn_relu_avgpool2_ndhwc": (c_int, [c_void_p, c_int, c_void_p, c_int] + [c_int] * 4 + [c_void_p, c_void_p, c_void_p]),
    "b2_avgpool_global_affine_ndhwc": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "b2_space_to_depth4_nchw": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "b2_gemm_splitk_workspace_elems": (ctypes.c_size_t, [c_int, c_int, c_int]),
    "b2_gemm_splitk_f16": (c_int, [ctypes.POINTER(GemmArgs), c_int, c_void_p, ctypes.c_size_t, c_void_p]),
    "b2_gemm_splitk_plan": (c_int, [c_int, c_int, c_int, c_int]),
}


def lib_path():
    return _LIB_PATH


def load():
    """Return the loaded shared library, building it first if it is not there."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        from .csrc import build as _build
        if _build.sources_present() and _build.have_nvcc():
            _build.build()    # digest check: rebuilds only when a source, header or flag changed since the .so was linked
        elif not os.path.exists(_LIB_PATH):
            raise RuntimeError("libb2pretorched.so is missing and cannot be built here (no nvcc / no sources): the engine has "
                               "no CPU or library fallback")
        lib = ctypes.CDLL(_LIB_PATH)
        lib.b2_version.restype = c_int
        got = lib.b2_version()
        if got != EXPECTED_ABI:
            raise RuntimeError("libb2pretorched.so reports ABI %d, this binding needs %d: stale library from another checkout -- "
                               "run `python -m pretorched_x_b200.csrc.build --force`" % (got, EXPECTED_ABI))
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(lib, name)  # AttributeError if the library does not export the symbol
            fn.restype = res
            fn.argtypes = args
        algo = os.environ.get("B2_CONV_ALGO")          # debug: "gather" disables the slab kernel (A/B timing)
        if algo:
            lib.b2_debug_set_conv_algo.restype = c_int
            lib.b2_debug_set_conv_algo.argtypes = [c_int]
            lib.b2_debug_set_conv_algo(1 if algo == "gather" else 0)
        if os.environ.get("B2_GEMM_ALGO"):             # debug: "tile" disables the persistent GEMM kernel
            lib.b2_debug_set_gemm_algo.restype = c_int
            lib.b2_debug_set_gemm_algo.argtypes = [c_int]
            lib.b2_debug_set_gemm_algo(1 if os.environ["B2_GEMM_ALGO"] == "tile" else 0)
        _lib = lib
    return _lib


def last_error():
    return load().b2_last_error().decode("utf-8", "replace")


def check(rc, what):
    if rc != B2_OK:
        raise RuntimeError("%s failed (code %d): %s" % (what, rc, last_error()))


def launch_count():
    return int(load().b2_launch_count())
