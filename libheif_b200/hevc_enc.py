"""HEVC-intra encoders: the host encoder (b200_hevc_encode_intra), the GPU encoder (GpuEncoder, b200_gpu_encoder_*), and the
synthetic source images of SURVEY.md 8(d)."""
import ctypes as C

import numpy as np

from . import _lib
from ._lib import EncParams, GpuEncodeStats, GridEncodeInfo


def default_params(**kw) -> EncParams:
    l = _lib.lib()
    p = EncParams()
    l.b200_hevc_enc_params_default(C.byref(p))
    for k, v in kw.items():
        if not hasattr(p, k):
            raise AttributeError(k)
        setattr(p, k, int(v))
    return p


def encode_intra(y, cb=None, cr=None, **kw) -> bytes:
    """Encode one picture; returns the access unit as length-prefixed NALs (what libheif pushes to a decoder plugin)."""
    l = _lib.lib()
    h, w = y.shape
    bd = kw.get("bit_depth", 8)
    dt = np.uint8 if bd == 8 else np.uint16
    y = np.ascontiguousarray(y, dtype=dt)
    chroma = cb is not None
    if chroma:
        cb = np.ascontiguousarray(cb, dtype=dt)
        cr = np.ascontiguousarray(cr, dtype=dt)
    cfmt = 0
    if chroma:                                             # chroma format from the plane shapes (4:2:0 / 4:2:2 / 4:4:4)
        cfmt = 3 if cb.shape == y.shape else (2 if cb.shape[0] == h else 1)
    p = default_params(width=w, height=h, chroma_format_idc=cfmt, **kw)
    out = C.POINTER(C.c_uint8)()
    n = C.c_size_t()
    _lib.check(l.b200_hevc_encode_intra(C.byref(p), y.ctypes.data, cb.ctypes.data if chroma else None,
                                        cr.ctypes.data if chroma else None, y.strides[0], cb.strides[0] if chroma else 0,
                                        C.byref(out), C.byref(n)))
    data = bytes(C.cast(out, C.POINTER(C.c_uint8 * n.value)).contents)
    l.b200_free(out)
    return data


# What the GPU encoder codes (b200_heif.h): no SAO, sign hiding or cu_qp_delta, one WPP sub-stream per CTB row.
GPU_DEFAULTS = dict(sao=0, sign_data_hiding=0, cu_qp_delta=0, wpp=1)


def gpu_params(width, height, chroma, **kw) -> EncParams:
    """b200_hevc_enc_params for b200_gpu_encode_intra_*: the library defaults with GPU_DEFAULTS, then `kw`."""
    return default_params(width=width, height=height, **{"chroma_format_idc": 1 if chroma else 0, **GPU_DEFAULTS, **kw})


def substream_capacity(width, log2_ctb_size, chroma=True) -> int:
    return int(_lib.lib().b200_gpu_encoder_substream_capacity(width, log2_ctb_size, 1 if chroma else 0))


def _grid_args(rgb, tile_w, tile_h, alpha, chroma_downsampling, only_use_preferred, bit_depth, endianness, alpha_bit_depth, params):
    """(b200_rgb_image, params, options, device?) of the b200_gpu_encode_rgb_grid_* calls; rgb: numpy array or CUDA tensor
    [H, W, 3|4], or a tuple (R, G, B) of [H, W] planes with the optional alpha plane in `alpha`."""
    from .color import _HOST, _Cuda, _rgb_image
    planar = isinstance(rgb, (tuple, list))
    if alpha is not None and not planar:
        raise ValueError("alpha= is the alpha plane of planar input; interleaved input carries alpha as RGBA")
    if planar:
        if len(rgb) != 3:
            raise ValueError("planar input: (R, G, B) planes, alpha in alpha=")
        rgb = tuple(rgb) + ((alpha,) if alpha is not None else ())
    first = rgb[0] if planar else rgb
    device = hasattr(first, "is_cuda") and first.is_cuda
    mem = _Cuda(first.device) if device else _HOST
    d, _ = _rgb_image(rgb, bit_depth, endianness, alpha_bit_depth, mem.ptr, mem.stride, mem.is16, mem.packed)
    p = gpu_params(tile_w, tile_h, True, **params)
    opt = _lib.RgbToYCbCrOptions(chroma_downsampling, int(bool(only_use_preferred)))
    return d, p, opt, device


def grid_encode_check(rgb, tile_w, tile_h, alpha=None, chroma_downsampling=2, only_use_preferred=False, input_bit_depth=None, endianness=None,
                      alpha_bit_depth=None, **params):
    """Host only, no CUDA (b200_gpu_encode_rgb_grid_check): raises B200Error with the code and message
    GpuEncoder.encode_rgb_grid would fail with for these arguments (numpy input; no pixel is read).  input_bit_depth /
    endianness / alpha_bit_depth describe uint16 inputs as rgb_to_ycbcr_ex's bit_depth / endianness / alpha_bit_depth do."""
    d, p, opt, _ = _grid_args(rgb, tile_w, tile_h, alpha, chroma_downsampling, only_use_preferred, input_bit_depth, endianness, alpha_bit_depth,
                              params)
    _lib.check(_lib.lib().b200_gpu_encode_rgb_grid_check(C.byref(d), tile_w, tile_h, C.byref(p), C.byref(opt)))


class GpuEncoder:
    """HEVC intra encoder on the GPU (b200_gpu_encoder_*): N same-sized 8-bit 4:2:0 or 4:0:0 pictures per call.

    encode(pictures, **params) takes a list of (y, cb, cr) tuples -- numpy uint8 host planes or uint8 CUDA tensors,
    cb = cr = None for monochrome -- and returns one access unit (length-prefixed NALs) per picture.  speed=0 (default), 1 or
    2 selects the mode decision (b200_heif.h): 1 searches at most 18 of the 35 luma modes per PU, 2 also decides open loop."""

    def __init__(self):
        self._l = _lib.lib()
        self._h = C.c_void_p()
        _lib.check(self._l.b200_gpu_encoder_create(C.byref(self._h)))
        self._shape = None

    def close(self):
        if getattr(self, "_h", None):
            self._l.b200_gpu_encoder_destroy(self._h)
            self._h = C.c_void_p()

    __del__ = close

    def encode(self, pictures, **params):
        pictures = list(pictures)
        if not pictures:
            raise ValueError("no pictures")
        y0 = pictures[0][0]
        h, w = int(y0.shape[0]), int(y0.shape[1])
        chroma = pictures[0][1] is not None
        p = gpu_params(w, h, chroma, **params)
        device = hasattr(y0, "is_cuda") and y0.is_cuda
        keep = []
        planes = (_lib.Planes * len(pictures))()
        for i, (y, cb, cr) in enumerate(pictures):
            q = planes[i]
            q.height, q.width = int(y.shape[0]), int(y.shape[1])
            q.chroma = 1 if cb is not None else 0
            q.bit_depth = 8
            arrs = [y, cb, cr] if cb is not None else [y]
            if device:
                arrs = [a.contiguous() for a in arrs]
                ptrs, strides = [a.data_ptr() for a in arrs], [a.stride(0) for a in arrs]
            else:
                arrs = [np.ascontiguousarray(a, dtype=np.uint8) for a in arrs]
                ptrs, strides = [a.ctypes.data for a in arrs], [a.strides[0] for a in arrs]
            keep += arrs
            q.y, q.y_stride = ptrs[0], strides[0]
            if cb is not None:
                q.cb, q.cr, q.c_stride = ptrs[1], ptrs[2], strides[1]
        if device:
            import torch
            stream = torch.cuda.current_stream(y0.device).cuda_stream
            _lib.check(self._l.b200_gpu_encode_intra_device(self._h, C.byref(p), len(pictures), planes, stream))
        else:
            _lib.check(self._l.b200_gpu_encode_intra_host(self._h, C.byref(p), len(pictures), planes))
        self._shape = (w, h, chroma)
        out = []
        for i in range(len(pictures)):
            d, n = C.POINTER(C.c_uint8)(), C.c_size_t()
            _lib.check(self._l.b200_gpu_encoder_output(self._h, i, C.byref(d), C.byref(n)))
            out.append(C.string_at(d, n.value))
        return out

    def encode_rgb_grid(self, rgb, tile_w, tile_h, alpha=None, chroma_downsampling=2, only_use_preferred=False, **params):
        """An 8-bit RGB picture -> the access units of a HEIC grid of tile_w x tile_h tiles in one call
        (b200_gpu_encode_rgb_grid_host for numpy input, _device for CUDA tensors, on the tensor's current stream).

        rgb: [H, W, 3|4] uint8 (RGB / RGBA), or a tuple (R, G, B) of [H, W] uint8 planes with the optional alpha plane in
        `alpha`.  params: b200_hevc_enc_params fields as for encode(); colour_primaries / matrix_coefficients / full_range are
        the conversion target as well.  Returns dict(tiles=[bytes] in raster order, alpha=[bytes] or None, cols, rows, width,
        height, pipeline (B200_YCC_PIPE_* mask), colour_ms, upload_ms)."""
        d, p, opt, device = _grid_args(rgb, tile_w, tile_h, alpha, chroma_downsampling, only_use_preferred, None, None, None, params)
        info = GridEncodeInfo()
        if device:
            import torch
            first = rgb[0] if isinstance(rgb, (tuple, list)) else rgb
            with torch.cuda.device(first.device):
                stream = torch.cuda.current_stream(first.device).cuda_stream
                _lib.check(self._l.b200_gpu_encode_rgb_grid_device(self._h, C.byref(d), tile_w, tile_h, C.byref(p), C.byref(opt), stream,
                                                                   C.byref(info)))
        else:
            _lib.check(self._l.b200_gpu_encode_rgb_grid_host(self._h, C.byref(d), tile_w, tile_h, C.byref(p), C.byref(opt), C.byref(info)))
        self._shape = (tile_w, tile_h, not info.has_alpha)       # recon(): the last batch coded (the alpha tiles when present)
        n = info.cols * info.rows
        out = []
        for i in range(n * (2 if info.has_alpha else 1)):
            dp, sz = C.POINTER(C.c_uint8)(), C.c_size_t()
            _lib.check(self._l.b200_gpu_encoder_output(self._h, i, C.byref(dp), C.byref(sz)))
            out.append(C.string_at(dp, sz.value))
        return dict(tiles=out[:n], alpha=out[n:] if info.has_alpha else None, cols=info.cols, rows=info.rows, width=info.width,
                    height=info.height, pipeline=info.pipeline, colour_ms=info.colour_ms, upload_ms=info.upload_ms)

    def recon(self, i):
        """Picture i of the last call as reconstructed before in-loop filtering: [y, cb, cr] (uint8; [y] for 4:0:0)."""
        w, h, chroma = self._shape
        y = np.empty((h, w), np.uint8)
        cb = np.empty(((h + 1) // 2, (w + 1) // 2), np.uint8) if chroma else None
        cr = np.empty_like(cb) if chroma else None
        _lib.check(self._l.b200_gpu_encoder_read_recon(self._h, i, y.ctypes.data, cb.ctypes.data if chroma else None,
                                                       cr.ctypes.data if chroma else None, w, (w + 1) // 2 if chroma else 0))
        return [y, cb, cr] if chroma else [y]

    def stats(self) -> GpuEncodeStats:
        s = GpuEncodeStats()
        _lib.check(self._l.b200_gpu_encoder_get_stats(self._h, C.byref(s)))
        return s

    def e1_warps_per_sm(self, speed=0) -> int:
        """Resident analysis (E1) warps per SM of the current device at this speed."""
        n = C.c_int()
        _lib.check(self._l.b200_gpu_encoder_e1_warps_per_sm(speed, C.byref(n)))
        return n.value


def synthetic_image(seed: int, width: int, height: int, bit_depth: int = 8, chroma=True):
    """Source picture of SURVEY.md 8(d): smooth gradient + 8 random-oriented sinusoid gratings + 1/16-amplitude noise,
    all driven by the 32-bit LCG s = s*1664525 + 1013904223 seeded with `seed`."""
    s = seed & 0xFFFFFFFF

    def nxt():
        nonlocal s
        s = (s * 1664525 + 1013904223) & 0xFFFFFFFF
        return s >> 8

    maxv = (1 << bit_depth) - 1
    yy, xx = np.mgrid[0:height, 0:width].astype(np.float32)
    planes = []
    # chroma: False / 0 = 4:0:0, True / 1 = 4:2:0, 2 = 4:2:2, 3 = 4:4:4 (chroma_format_idc)
    cfmt = int(chroma)
    for c in range(3 if cfmt else 1):
        subx = 2 if (c and cfmt in (1, 2)) else 1
        suby = 2 if (c and cfmt == 1) else 1
        h, w = (height + suby - 1) // suby, (width + subx - 1) // subx
        X, Y = xx[:h, :w] * subx, yy[:h, :w] * suby
        gx, gy = (nxt() % 200 - 100) / 100.0, (nxt() % 200 - 100) / 100.0
        img = 0.5 + 0.25 * (gx * (X / max(width, 1) - 0.5) + gy * (Y / max(height, 1) - 0.5))
        for _ in range(8):
            ang = (nxt() % 3600) / 3600.0 * np.pi
            freq = 2 * np.pi / (4 + nxt() % 120)
            ph = (nxt() % 1000) / 1000.0 * 2 * np.pi
            amp = (0.02 + (nxt() % 100) / 1500.0) * (0.5 if c else 1.0)
            img = img + amp * np.sin(freq * (np.cos(ang) * X + np.sin(ang) * Y) + ph)
        rs = np.random.RandomState(nxt() & 0x7FFFFFFF)       # noise: bulk generator seeded from the LCG stream
        img = img + (rs.rand(h, w).astype(np.float32) - 0.5) / 16.0
        planes.append(np.clip(np.rint(img * maxv), 0, maxv).astype(np.uint16 if bit_depth > 8 else np.uint8))
    return planes if chroma else [planes[0], None, None]
