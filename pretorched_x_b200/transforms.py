"""Image preprocessing behind the reference's interface (pretorched/transforms/utils.py:9-105), with the pixel work on the GPU.

``TransformImage(opts, scale=0.875, random_crop=False, random_hflip=False, random_vflip=False, preserve_aspect_ratio=True)``
takes the model (or its settings dict) exactly like the reference and is called with a decoded image; it returns the fp32
``[3, H, W]`` tensor the reference returns -- bit-identical to the Pillow + torchvision pipeline it composes
(transforms/utils.py:53-77) -- but living on the device, produced by ``b2_transform_image_u8`` (csrc/b2_image.cu):
Pillow-exact 8-bit bilinear resampling, crop, flips, ToTensor, ToSpaceBGR, ToRange255 and Normalize in two launches.
``to_stem_input=True`` additionally / instead yields the fp16 NDHWC4 ``Act`` the stem convolution consumes.

Host side of the split: JPEG decode (Pillow, as upstream's ``LoadImage``), the output-size / crop-offset rules and the
fixed-point coefficient tables of the resampling filter (a few hundred integers per axis, cached per size pair).
"""
import ctypes
import math

import numpy as np
import torch

from . import _lib, ops

_PRECISION_BITS = 32 - 8 - 2


class ToSpaceBGR(object):
    """transforms/utils.py:9-20 (tensor op; kept for API compatibility -- TransformImage fuses it into the kernel)."""

    def __init__(self, is_bgr):
        self.is_bgr = is_bgr

    def __call__(self, tensor):
        if self.is_bgr:
            tensor = tensor.flip(0) if tensor.shape[0] == 3 else tensor
        return tensor


class ToRange255(object):
    """transforms/utils.py:23-31."""

    def __init__(self, is_255):
        self.is_255 = is_255

    def __call__(self, tensor):
        if self.is_255:
            tensor.mul_(255)
        return tensor


def _opt(opts, name):
    return opts[name] if isinstance(opts, dict) else getattr(opts, name)


def _has(opts, name):
    return (name in opts) if isinstance(opts, dict) else hasattr(opts, name)


_COEFF_CACHE = {}


def resample_coeffs(in_size, out_size, device):
    """Pillow's bilinear (triangle) resampling window for every output index, as device int32 tables
    (bounds [out][2] = first source index / count, coeffs [out][ksize], 22-bit fixed point).  Vectorised restatement of
    libImaging/Resample.c ``precompute_coeffs`` + ``normalize_coeffs_8bpc``; the CPU oracle (oracle/image.py) holds the
    scalar version and tests/test_image_cpu.py checks both against Pillow itself."""
    key = (in_size, out_size, str(device))
    hit = _COEFF_CACHE.get(key)
    if hit is not None:
        return hit
    scale = in_size / out_size
    fscale = max(scale, 1.0)
    support = fscale
    ksize = int(math.ceil(support)) * 2 + 1
    xx = np.arange(out_size, dtype=np.float64)
    center = (xx + 0.5) * scale
    xmin = np.maximum((center - support + 0.5).astype(np.int64), 0)
    xmax = np.minimum((center + support + 0.5).astype(np.int64), in_size)
    count = xmax - xmin
    taps = np.arange(ksize, dtype=np.float64)[None, :]
    arg = np.abs((taps + xmin[:, None] - center[:, None] + 0.5) * (1.0 / fscale))
    w = np.where(arg < 1.0, 1.0 - arg, 0.0)
    w[taps >= count[:, None]] = 0.0
    # Pillow sums the window left to right in double precision; do the same so the normalisation is bit-identical
    ww = np.zeros(out_size, dtype=np.float64)
    for t in range(ksize):
        ww = ww + w[:, t]
    w = np.where(ww[:, None] != 0.0, w / np.where(ww == 0.0, 1.0, ww)[:, None], w)
    kk = np.trunc(w * (1 << _PRECISION_BITS) + 0.5).astype(np.int32)        # all weights are >= 0 for the triangle filter
    kk[taps.repeat(out_size, 0) >= count[:, None]] = 0
    bounds = np.stack([xmin, count], axis=1).astype(np.int32)
    out = (torch.from_numpy(np.ascontiguousarray(bounds)).to(device), torch.from_numpy(np.ascontiguousarray(kk)).to(device), ksize)
    _COEFF_CACHE[key] = out
    return out


def resized_size(h, w, size):
    """torchvision ``Resize(int)``: the shorter edge becomes ``size``, the longer ``int(size * long / short)``."""
    short, long = (w, h) if w <= h else (h, w)
    new_long = int(size * long / short)
    return (new_long, size) if w <= h else (size, new_long)


class TransformImage(object):
    """transforms/utils.py:34-81, same constructor.  ``__call__(img)``: ``img`` is a PIL image, a uint8 ``[H, W, 3]`` NumPy array
    or tensor (host or device).  Returns a CUDA fp32 ``[3, S, S]`` tensor; ``stem_input(img)`` returns the NDHWC4 ``Act``."""

    def __init__(self, opts, scale=0.875, random_crop=False, random_hflip=False, random_vflip=False,
                 preserve_aspect_ratio=True, device=None):
        self.input_size = list(_opt(opts, 'input_size'))
        self.input_space = _opt(opts, 'input_space')
        self.input_range = list(_opt(opts, 'input_range'))
        self.mean = list(_opt(opts, 'mean'))
        self.std = list(_opt(opts, 'std'))
        self.scale = scale
        self.random_crop, self.random_hflip, self.random_vflip = random_crop, random_hflip, random_vflip
        self.preserve_aspect_ratio = preserve_aspect_ratio
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device()) \
            if torch.cuda.is_available() else None
        self._mean = (ctypes.c_float * 3)(*[float(np.float32(m)) for m in self.mean])
        self._std = (ctypes.c_float * 3)(*[float(np.float32(s)) for s in self.std])

    # -- host-side geometry (torchvision's rules) -----------------------------------------------------------------
    def plan(self, h, w):
        """(resized_h, resized_w, top, left, crop, hflip, vflip) for an h x w image; consumes torch's global RNG in the same
        order as torchvision's RandomCrop / RandomHorizontalFlip / RandomVerticalFlip."""
        crop = max(self.input_size)
        if self.preserve_aspect_ratio:
            rh, rw = resized_size(h, w, int(math.floor(crop / self.scale)))
        else:
            rh, rw = int(self.input_size[1] / self.scale), int(self.input_size[2] / self.scale)
        if self.random_crop:
            if rh < crop or rw < crop:
                raise ValueError("Required crop size %s is larger than input image size %s" % ((crop, crop), (rh, rw)))
            top = int(torch.randint(0, rh - crop + 1, size=(1,)).item()) if (rh, rw) != (crop, crop) else 0
            left = int(torch.randint(0, rw - crop + 1, size=(1,)).item()) if (rh, rw) != (crop, crop) else 0
        else:
            if rh < crop or rw < crop:
                raise NotImplementedError("CenterCrop of an image smaller than the crop (zero padding) is not implemented")
            top, left = int(round((rh - crop) / 2.0)), int(round((rw - crop) / 2.0))
        hflip = bool(torch.rand(1) < 0.5) if self.random_hflip else False
        vflip = bool(torch.rand(1) < 0.5) if self.random_vflip else False
        return rh, rw, top, left, crop, hflip, vflip

    def _to_device_u8(self, img):
        if self.device is None:
            raise RuntimeError("TransformImage runs on a CUDA (sm_90a) device: this engine has no CPU path")
        if isinstance(img, torch.Tensor):
            t = img
        else:
            arr = np.asarray(img)
            if arr.ndim == 2:
                arr = np.repeat(arr[:, :, None], 3, axis=2)
            t = torch.from_numpy(np.ascontiguousarray(arr))
        if t.dtype != torch.uint8 or t.dim() != 3 or t.shape[2] != 3:
            raise ValueError("expected a uint8 [H, W, 3] image, got %s %s" % (t.dtype, tuple(t.shape)))
        return t.to(self.device, non_blocking=True).contiguous()

    def _run(self, img, want_f32, want_h4):
        u8 = self._to_device_u8(img)
        H, W = int(u8.shape[0]), int(u8.shape[1])
        rh, rw, top, left, crop, hflip, vflip = self.plan(H, W)
        dev = u8.device
        hb = hk = vb = vk = tmp = None
        hks = vks = 0
        if rw != W:
            hb, hk, hks = resample_coeffs(W, rw, dev)
            tmp = torch.empty((H, rw, 3), dtype=torch.uint8, device=dev)
        if rh != H:
            vb, vk, vks = resample_coeffs(H, rh, dev)
        out = torch.empty((3, crop, crop), dtype=torch.float32, device=dev) if want_f32 else None
        h4 = torch.empty((crop * crop, 4), dtype=torch.float16, device=dev) if want_h4 else None
        flags = int(hflip) | (int(vflip) << 1) | (int(self.input_space == 'BGR') << 2) | (int(max(self.input_range) == 255) << 3)
        p = ops._ptr
        with torch.cuda.device(dev):
            _lib.check(_lib.load().b2_transform_image_u8(p(u8), H, W, p(hb), p(hk), hks, rw, p(vb), p(vk), vks, rh, p(tmp), top, left,
                                                        crop, crop, flags, self._mean, self._std, p(out), p(h4), ops._stream()),
                       "b2_transform_image_u8")
        return out, (ops.Act(h4, 1, 1, crop, crop, 3) if want_h4 else None)

    def __call__(self, img):
        return self._run(img, True, False)[0]

    def stem_input(self, img):
        """The preprocessed image as the fp16 NDHWC4 activation ``model.features`` / ``model.forward`` accept directly."""
        return self._run(img, False, True)[1]


class LoadImage(object):
    """transforms/utils.py:84-93: decode with Pillow on the host and convert to ``space``."""

    def __init__(self, space='RGB'):
        self.space = space

    def __call__(self, path_img):
        from PIL import Image
        with open(path_img, 'rb') as f:
            with Image.open(f) as img:
                img = img.convert(self.space)
        return img


class LoadTransformImage(object):
    """transforms/utils.py:96-105."""

    def __init__(self, model, scale=0.875):
        self.load = LoadImage()
        self.tf = TransformImage(model, scale=scale)

    def __call__(self, path_img):
        return self.tf(self.load(path_img))


class ClipToStemInput(object):
    """Decoded video clips, uint8 ``[N, T, H, W, 3]`` (channels last, already at network resolution), to the fp16 NDHWC4 ``Act``
    the 3-D stems consume: ToTensor, ToSpaceBGR, ToRange255 and Normalize of the model's settings (transforms/utils.py:72-75)
    applied per pixel on the device.  The reference has no clip loader (SURVEY.md section 8f n4); what this adds is the transfer
    format -- 3 bytes per pixel over PCIe instead of the 12 of an fp32 NCDHW tensor -- with the same arithmetic as
    ``TransformImage``'s tail.  ``model(ClipToStemInput(model)(clips_u8))`` equals ``model(x)`` for
    ``x = ((clips / 255 - mean) / std)`` permuted to NCDHW, bit for bit after the engine's fp16 rounding of the input."""

    def __init__(self, opts):
        self.input_space = _opt(opts, 'input_space') if _has(opts, 'input_space') else 'RGB'
        self.input_range = list(_opt(opts, 'input_range')) if _has(opts, 'input_range') else [0, 1]
        self.mean = list(_opt(opts, 'mean'))
        self.std = list(_opt(opts, 'std'))
        self._mean = (ctypes.c_float * 3)(*[float(np.float32(m)) for m in self.mean])
        self._std = (ctypes.c_float * 3)(*[float(np.float32(s)) for s in self.std])

    def __call__(self, clips_u8, out=None):
        if clips_u8.dtype != torch.uint8 or clips_u8.dim() != 5 or clips_u8.shape[-1] != 3 or not clips_u8.is_cuda:
            raise ValueError("expected a CUDA uint8 [N, T, H, W, 3] tensor, got %s %s" % (clips_u8.dtype, tuple(clips_u8.shape)))
        clips_u8 = clips_u8.contiguous()
        N, T, H, W, _ = clips_u8.shape
        px = N * T * H * W
        y = out if out is not None else torch.empty((px, 4), dtype=torch.float16, device=clips_u8.device)
        flags = (int(self.input_space == 'BGR') << 2) | (int(max(self.input_range) == 255) << 3)
        with torch.cuda.device(clips_u8.device):
            _lib.check(_lib.load().b2_u8_frames_to_ndhwc4_f16(ops._ptr(clips_u8), ops._ptr(y), px, flags, self._mean, self._std,
                                                             ops._stream()), "b2_u8_frames_to_ndhwc4_f16")
        return ops.Act(y, N, T, H, W, 3)
