"""libheif_b200 -- H100-native replacement of libheif's per-tile decode pixel pipeline.

Host-side mirror (Python) of the reference interfaces for this path; all pixel work happens in
libb200heif.so (hand-written sm_90a CUDA behind the C ABI of include/b200_heif.h).
PyTorch is used only for device memory, streams and torch.distributed plumbing.
"""
from ._lib import lib, B200Error, SO_PATH  # noqa: F401
from .color import (Geometry, YCbCrImage, convert_colorspace, convert_colorspace_host, rgb_to_ycbcr, rgb_to_ycbcr_host,  # noqa: F401
                    rgb_to_ycbcr_ex, rgb_to_ycbcr_ex_host, rgb_to_ycbcr_plan, YCC_PIPE_NAMES,
                    CHROMA_420, CHROMA_422, CHROMA_444, CHROMA_MONO, CHROMA_INTERLEAVED_RGB, CHROMA_INTERLEAVED_RGBA,
                    CHROMA_INTERLEAVED_RRGGBB_BE, CHROMA_INTERLEAVED_RRGGBBAA_BE, CHROMA_INTERLEAVED_RRGGBB_LE,
                    CHROMA_INTERLEAVED_RRGGBBAA_LE)
from .decoder import Decoder, ImageInfo, DecodeStats  # noqa: F401,E402
from . import hevc_enc  # noqa: F401,E402
from . import compose  # noqa: F401,E402
from .compose import thumbnail_size  # noqa: F401,E402
