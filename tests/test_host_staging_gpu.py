"""Host <-> device staging of the host entry points (b200_color_convert_host, b200_rgb_to_ycbcr_host, the pageable
destination of b200_decode_grid_to_rgb_host): rows longer than one 32 MiB bounce slot, several bands through both slots,
buffers that grow and shrink between calls, and a second GPU.  Every result equals the device-to-device form or the
colour oracle byte for byte."""
import numpy as np
import pytest

import libheif_b200 as lb
from util import oracle_postprocess, random_ycbcr

pytestmark = pytest.mark.gpu

SLOT = 32 << 20                      # bytes of one bounce slot


def _planes(rng, w, h, bpp, alpha):
    """4:2:0 planes of `bpp` bits (uint8 / uint16 numpy arrays)."""
    dt, hi = (np.uint8, 256) if bpp == 8 else (np.uint16, 1 << bpp)
    cw, ch = (w + 1) // 2, (h + 1) // 2
    return [rng.integers(0, hi, s, dtype=dt) if s else None for s in ((h, w), (ch, cw), (ch, cw), (h, w) if alpha else None)]


def _image(planes, bpp, dev=None):
    import torch

    def cv(p):
        if p is None or dev is None:
            return p
        return torch.from_numpy(p.view(np.int16) if bpp > 8 else p).to(dev)
    y, cb, cr, a = (cv(p) for p in planes)
    return lb.YCbCrImage(y, cb, cr, a, chroma=lb.CHROMA_420, bit_depth=bpp, colour_primaries=9, transfer_characteristics=16,
                         matrix_coefficients=9, full_range=False)


def _check_ycc(host, dev):
    for name, h, d in zip("Y Cb Cr A".split(), (host.y, host.cb, host.cr, host.alpha), (dev.y, dev.cb, dev.cr, dev.alpha)):
        assert (h is None) == (d is None), name
        if h is not None:
            assert np.array_equal(h, d.cpu().numpy()), f"{name} differs"


def test_color_host_rows_longer_than_a_bounce_slot(cuda):
    """4:2:0 10 bit -> RRGGBBAA: every output row is longer than a slot, so each row is a band of its own, alternating slots."""
    w, h = 4194336, 4
    assert w * 8 > SLOT
    planes = _planes(np.random.default_rng(1), w, h, 10, alpha=True)
    host, _ = lb.convert_colorspace_host(_image(planes, 10), lb.CHROMA_INTERLEAVED_RRGGBBAA_LE)
    dev = lb.convert_colorspace(_image(planes, 10, cuda), lb.CHROMA_INTERLEAVED_RRGGBBAA_LE)
    assert np.array_equal(host.view(np.uint8), dev.cpu().numpy().view(np.uint8))


def test_rgb_to_ycbcr_host_rows_longer_than_a_bounce_slot(cuda):
    import torch
    w, h = 8388612, 3
    assert w * 4 > SLOT
    rgba = np.random.default_rng(2).integers(0, 256, (h, w, 4), dtype=np.uint8)
    host = lb.rgb_to_ycbcr_host(rgba, lb.CHROMA_420, matrix_coefficients=6, colour_primaries=1, full_range=False)
    dev = lb.rgb_to_ycbcr(torch.from_numpy(rgba).to(cuda), lb.CHROMA_420, matrix_coefficients=6, colour_primaries=1, full_range=False)
    torch.cuda.synchronize()
    _check_ycc(host, dev)


def test_pageable_decode_in_several_bands(cuda):
    """5 x 5 grid of one 1024 x 1024 tile -> 5120 x 5120 RGB24 (79 MB: two full bounce slots and a partial third) into pageable
    memory equals the same call into page-locked memory."""
    import torch
    y, cb, cr = lb.hevc_enc.synthetic_image(0xB200, 1024, 1024, 8, True)
    tile = lb.hevc_enc.encode_intra(y, cb, cr, log2_ctb_size=5, wpp=1, seed=0xB200, vui_present=1, colour_description_present=1,
                                    colour_primaries=1, transfer_characteristics=13, matrix_coefficients=6, full_range=0)
    tiles = [tile] * 25
    W = H = 5120
    assert 2 * SLOT < H * W * 3 < 3 * SLOT
    d = lb.Decoder(host_threads=8)
    try:
        pageable = np.zeros((H, W * 3), np.uint8)
        d.decode_grid_to_rgb_host(tiles, 5, 5, lb.CHROMA_INTERLEAVED_RGB, out=pageable)
        pinned = torch.zeros((H, W * 3), dtype=torch.uint8, pin_memory=True)
        d.decode_grid_to_rgb_host(tiles, 5, 5, lb.CHROMA_INTERLEAVED_RGB, out=pinned.numpy())
        assert np.array_equal(pageable, pinned.numpy())
    finally:
        d.close()


def test_rgb_to_ycbcr_host_staging_grows_and_shrinks(cuda):
    """small -> large (several bands) -> small: the kept buffers are re-used and grown without changing a result."""
    import torch
    rng = np.random.default_rng(3)
    for w, h, bpp, chroma in ((64, 48, 3, lb.CHROMA_420), (6000, 3001, 4, lb.CHROMA_422), (33, 17, 4, lb.CHROMA_444)):
        rgb = rng.integers(0, 256, (h, w, bpp), dtype=np.uint8)
        host = lb.rgb_to_ycbcr_host(rgb, chroma, matrix_coefficients=1, colour_primaries=1, full_range=True)
        dev = lb.rgb_to_ycbcr(torch.from_numpy(rgb).to(cuda), chroma, matrix_coefficients=1, colour_primaries=1, full_range=True)
        torch.cuda.synchronize()
        _check_ycc(host, dev)


def test_color_host_on_two_gpus(cuda):
    """Each GPU keeps its own staging: device 0, then 1, then 0 again, each equal to the colour oracle."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    y, cb, cr, _ = random_ycbcr(5, 300, 200, 1, 8)
    want, _, _ = oracle_postprocess(y, cb, cr, None, 1, 8, (1, 13, 6, 0), [], 10)
    img = lb.YCbCrImage(y.astype(np.uint8), cb.astype(np.uint8), cr.astype(np.uint8), None, chroma=lb.CHROMA_420, bit_depth=8,
                        colour_primaries=1, transfer_characteristics=13, matrix_coefficients=6, full_range=False)
    for dev in (0, 1, 0):
        with torch.cuda.device(dev):
            out, _ = lb.convert_colorspace_host(img, lb.CHROMA_INTERLEAVED_RGB)
        assert np.array_equal(out.reshape(-1), want), f"device {dev}"
