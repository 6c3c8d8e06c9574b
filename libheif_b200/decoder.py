"""HEVC intra decoder (host front-end + sm_90a kernels) -- Python mirror of the decoder-plugin call sequence.

Reference interfaces mirrored:
  heif_decoder_plugin::new_decoder2 / push_data2 / decode_next_image2 / free_decoder   libheif/api/libheif/heif_plugin.h:85-169
  as driven by Decoder::decode_single_frame_from_compressed_data                        libheif/codecs/decoder.cc:523-563
  and, for grids, ImageItem_Grid::decode_full_grid_image                                libheif/image-items/grid.cc:250-468
"""
import ctypes as C
from typing import List, Optional, Sequence

import numpy as np

from . import _lib
from ._lib import DecodeStats, ImageInfo
from .color import _BYTES_PER_PIXEL, Geometry, YCbCrImage, convert_colorspace


class Decoder:
    """One decoder context per process/GPU (owns device arenas, pinned staging and the parser thread pool)."""

    def __init__(self, host_threads: int = 0):
        self.l = _lib.lib()
        self.h = C.c_void_p()
        _lib.check(self.l.b200_decoder_create(C.byref(self.h), host_threads))
        self.info = None

    def close(self):
        if self.h:
            self.l.b200_decoder_destroy(self.h)
            self.h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @staticmethod
    def _aus(aus: Sequence[bytes]):
        n = len(aus)
        arr = (C.c_char_p * n)(*aus)
        sizes = (C.c_size_t * n)(*[len(a) for a in aus])
        return arr, sizes

    def decode_grid(self, aus: Sequence[bytes], cols: int = 1, rows: int = 1, canvas=(0, 0), max_image_size_pixels: int = 0, stream=None):
        """push + decode cols*rows access units (row-major tiles) into the device canvas. Returns ImageInfo."""
        assert len(aus) == cols * rows
        arr, sizes = self._aus(aus)
        info = ImageInfo()
        s = C.c_void_p(stream.cuda_stream) if stream is not None else None
        _lib.check(self.l.b200_decoder_decode_grid(self.h, cols, rows, arr, sizes, max_image_size_pixels, canvas[0], canvas[1], C.byref(info), s))
        self.info = info
        return info

    def decode_image(self, au: bytes, **kw):
        return self.decode_grid([au], 1, 1, **kw)

    def planes_host(self):
        """D2H of the canvas planes -> list of numpy arrays (uint8, or uint16 for > 8 bit)."""
        i = self.info
        dt = np.uint8 if i.bit_depth == 8 else np.uint16
        y = np.empty((i.height, i.width), dt)
        if i.chroma == 0:
            _lib.check(self.l.b200_decoder_read_planes(self.h, y.ctypes.data, y.strides[0], None, None, 0, None))
            return [y]
        sx, sy = (1 if i.chroma in (1, 2) else 0), (1 if i.chroma == 1 else 0)      # 4:2:0 / 4:2:2 / 4:4:4
        cb = np.empty(((i.height + sy) >> sy, (i.width + sx) >> sx), dt)
        cr = np.empty_like(cb)
        _lib.check(self.l.b200_decoder_read_planes(self.h, y.ctypes.data, y.strides[0], cb.ctypes.data, cr.ctypes.data, cb.strides[0], None))
        return [y, cb, cr]

    def planes_device(self) -> _lib.Planes:
        p = _lib.Planes()
        _lib.check(self.l.b200_decoder_get_planes(self.h, C.byref(p)))
        return p

    def set_front_end(self, device: bool):
        """True (default): CABAC + syntax on the GPU; False: on the host cores."""
        _lib.check(self.l.b200_decoder_set_front_end(self.h, 1 if device else 0))

    def set_debug_stage(self, stage: int):
        _lib.check(self.l.b200_decoder_set_debug_stage(self.h, stage))

    def debug_tile(self, index: int, coded_w: int, coded_h: int):
        i = self.info
        dt = np.uint8 if i.bit_depth == 8 else np.uint16
        y = np.empty((coded_h, coded_w), dt)
        sx, sy = (1 if i.chroma in (1, 2) else 0), (1 if i.chroma == 1 else 0)
        cb = np.empty((coded_h >> sy, coded_w >> sx), dt)
        cr = np.empty_like(cb)
        mono = i.chroma == 0
        _lib.check(self.l.b200_decoder_debug_read_tile(self.h, index, 0, y.ctypes.data, None if mono else cb.ctypes.data, None if mono else cr.ctypes.data))
        return [y] if mono else [y, cb, cr]

    def rerun_device(self, stream=None):
        """Re-launch reconstruction/deblocking/SAO on the command stream resident in HBM (kernel-only timing)."""
        s = C.c_void_p(stream.cuda_stream) if stream is not None else None
        _lib.check(self.l.b200_decoder_rerun_device(self.h, s))

    def stats(self) -> DecodeStats:
        st = DecodeStats()
        _lib.check(self.l.b200_decoder_get_stats(self.h, C.byref(st)))
        return st

    def to_rgb_device(self, out_chroma: int, geometry: Optional[Geometry] = None, out=None, stream=None, scale=None):
        """Colour post-stage on the canvas, device -> device (torch tensor result).  scale=(w, h): the result scaled to w x h
        with the reference's nearest-neighbour scaler, only the kept pixels converted (b200_color_convert_scaled_device)."""
        import torch
        p = self.planes_device()
        geom = geometry or Geometry(p.width, p.height)
        ow, oh = scale or geom.size
        bpp = _BYTES_PER_PIXEL[out_chroma]
        if out is None:
            out = torch.empty((oh, ow * bpp), dtype=torch.uint8, device="cuda")
        opt = _lib.ColorOptions(out_chroma, 0, 0)
        s = C.c_void_p(stream.cuda_stream) if stream is not None else C.c_void_p(torch.cuda.current_stream().cuda_stream)
        if scale is None:
            _lib.check(self.l.b200_color_convert_device(C.byref(p), C.byref(geom.g), C.byref(opt), out.data_ptr(), None, None,
                                                        out.stride(0), s, None))
        else:
            _lib.check(self.l.b200_color_convert_scaled_device(C.byref(p), C.byref(geom.g), C.byref(opt), int(ow), int(oh), out.data_ptr(),
                                                               None, None, out.stride(0), s, None))
        return out

    def decode_grid_to_rgb_host(self, aus: Sequence[bytes], cols: int, rows: int, out_chroma: int, canvas=(0, 0), geometry: Optional[Geometry] = None,
                                out: Optional[np.ndarray] = None, max_image_size_pixels: int = 0, scale=None):
        """heif_decode_image() equivalent on the fused path: HEVC tiles in host memory -> interleaved RGB in host memory.
        scale=(w, h): heif_decode_image + heif_image_scale_image in one call (b200_decode_grid_to_rgb_scaled_host); `out` is
        then [h, w*bytes_per_pixel] and only the scaled picture is converted and copied."""
        arr, sizes = self._aus(aus)
        info = ImageInfo()
        bpp = _BYTES_PER_PIXEL[out_chroma]
        opt = _lib.ColorOptions(out_chroma, 0, 0)
        if out is None:
            # size is known only after parsing: decode once into a maximal buffer is wasteful, so require the caller
            # to pass `out` for big images; small ones use a probe of tile size * grid
            raise ValueError("pass a preallocated `out` array [H, W*bytes_per_pixel] (uint8)")
        g = C.byref(geometry.g) if geometry is not None else None
        if scale is None:
            _lib.check(self.l.b200_decode_grid_to_rgb_host(self.h, cols, rows, arr, sizes, max_image_size_pixels, canvas[0], canvas[1], g,
                                                           C.byref(opt), out.ctypes.data, out.strides[0], C.byref(info)))
        else:
            _lib.check(self.l.b200_decode_grid_to_rgb_scaled_host(self.h, cols, rows, arr, sizes, max_image_size_pixels, canvas[0], canvas[1], g,
                                                                  C.byref(opt), int(scale[0]), int(scale[1]), out.ctypes.data, out.strides[0],
                                                                  C.byref(info)))
        self.info = info
        return out, info

    def decode_grid_to_rgb_host_async(self, aus: Sequence[bytes], cols: int, rows: int, out_chroma: int, out: np.ndarray, canvas=(0, 0),
                                      geometry: Optional[Geometry] = None, max_image_size_pixels: int = 0):
        """Throughput form (b200_decode_grid_to_rgb_host_async): returns once the work is queued; `out` must be page-locked
        (a pinned torch tensor's numpy view, or memory from b200_host_alloc / b200_host_register).  Call wait() before reading."""
        arr, sizes = self._aus(aus)
        self._keep = (arr, sizes, aus)                     # the access units are read during this call only, the arrays until it returns
        info = ImageInfo()
        opt = _lib.ColorOptions(out_chroma, 0, 0)
        g = C.byref(geometry.g) if geometry is not None else None
        _lib.check(self.l.b200_decode_grid_to_rgb_host_async(self.h, cols, rows, arr, sizes, max_image_size_pixels, canvas[0], canvas[1], g,
                                                             C.byref(opt), out.ctypes.data, out.strides[0], C.byref(info)))
        self.info = info
        return info

    def wait(self):
        _lib.check(self.l.b200_decoder_wait(self.h))
