"""GPU parity: the sm_90a HEVC intra decoder (host front-end + reconstruction / deblocking / SAO kernels, through the
C ABI) vs the C restatement (oracle/hevc_oracle.c, pinned on FFmpeg) -- bit-exact on every plane, every stream,
including the intermediate stages (before deblocking, after deblocking) to localise mismatches."""
import hashlib

import numpy as np
import pytest

import libheif_b200 as lb
from hevc_cases import SYNTH, SYNTH_CPU_EXTRA, all_streams, synth_stream
from oracle import bindings as ob

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", params=["device", "host"])
def dec(cuda, request):
    """Both front-ends must give identical results: CABAC on the GPU (default) and CABAC on the host cores."""
    d = lb.Decoder(host_threads=8)
    d.set_front_end(request.param == "device")
    yield d
    d.close()


@pytest.mark.parametrize("name,au", all_streams(), ids=[s[0] for s in all_streams()])
def test_single_picture_matches_oracle(dec, name, au):
    want, info = ob.restatement_decode(au)
    dec.set_debug_stage(0)
    i = dec.decode_image(au)
    got = dec.planes_host()
    assert (i.width, i.height, i.bit_depth) == (want[0].shape[1], want[0].shape[0], info["bit_depth"])
    assert (i.colour_primaries, i.transfer_characteristics, i.matrix_coefficients, i.full_range) == (info["cp"], info["tc"], info["mc"], info["full_range"])
    for c in range(len(want)):
        assert np.array_equal(got[c], want[c]), f"{name}: plane {c} first diffs {np.argwhere(got[c] != want[c])[:4].tolist()}"


@pytest.mark.parametrize("name", ["ctb32", "ctb64_wpp_random", "main10", "slices_nolf", "rainbow_452x462.au"])
@pytest.mark.parametrize("stage", [1, 2])
def test_intermediate_stages(dec, name, stage):
    au = dict(all_streams())[name]
    want, info = ob.restatement_decode(au, stage)          # cropped to the conformance window
    dec.set_debug_stage(stage)
    try:
        dec.decode_image(au)
        h, w = want[0].shape
        cw, ch = (w + 7) & ~7, (h + 7) & ~7
        got = dec.debug_tile(0, cw, ch)
        for c in range(len(want)):
            hh, ww = want[c].shape
            assert np.array_equal(got[c][:hh, :ww], want[c]), f"stage {stage} plane {c}"
    finally:
        dec.set_debug_stage(0)


def test_grid_of_tiles_matches_per_tile_oracle(dec):
    """3x2 grid of independent tiles pasted into one canvas (ImageItem_Grid semantics) incl. a canvas smaller than the
    tile area (tiles overhanging the right/bottom border are clipped like HeifPixelImage::copy_image_to)."""
    tiles = []
    for k in range(6):
        y, cb, cr = lb.hevc_enc.synthetic_image(0xB200 + k, 128, 64, 8, True)
        tiles.append(lb.hevc_enc.encode_intra(y, cb, cr, log2_ctb_size=5, wpp=k % 2, seed=0xB200 + k))
    ref = [ob.restatement_decode(t)[0] for t in tiles]
    for canvas in [(0, 0), (350, 100)]:
        i = dec.decode_grid(tiles, cols=3, rows=2, canvas=canvas)
        got = dec.planes_host()
        W, H = (384, 128) if canvas == (0, 0) else canvas
        assert (i.width, i.height) == (W, H)
        want = [np.zeros((H, W), np.uint16), np.zeros(((H + 1) // 2, (W + 1) // 2), np.uint16), np.zeros(((H + 1) // 2, (W + 1) // 2), np.uint16)]
        for k in range(6):
            col, row = k % 3, k // 3
            for c in range(3):
                s = 1 if c == 0 else 2
                x0, y0 = col * 128 // s, row * 64 // s
                hh, ww = want[c].shape
                t = ref[k][c][:max(0, hh - y0), :max(0, ww - x0)]
                want[c][y0:y0 + t.shape[0], x0:x0 + t.shape[1]] = t
        for c in range(3):
            assert np.array_equal(got[c], want[c]), f"canvas {canvas} plane {c}"


def test_decode_to_rgb_end_to_end(dec):
    """HEVC tiles (host) -> RGB24 (host) through the fused C-ABI entry; equals restatement planes + colour oracle."""
    from util import oracle_postprocess
    au = synth_stream("big_qp37_vui")                      # VUI 1/13/6 full range -> integer colour path
    planes, info = ob.restatement_decode(au)
    want, ow, oh = oracle_postprocess(planes[0], planes[1], planes[2], None, 1, 8, (info["cp"], info["tc"], info["mc"], info["full_range"]), [], 10)
    out = np.empty((oh, ow * 3), np.uint8)
    dec.decode_grid_to_rgb_host([au], 1, 1, lb.CHROMA_INTERLEAVED_RGB, out=out)
    assert np.array_equal(out.reshape(-1), want)


def test_example_heic_rgb_md5(dec):
    """BASELINE config 1 / SURVEY Appendix C: examples/example.heic primary item -> RGB24 md5 of the reference
    (heif_decode_image with the CPU plugin) = 01672ec0cdf97b977628957cd6533dc2."""
    au = dict(all_streams())["example_primary_1280x854.au"]
    out = np.empty((854, 1280 * 3), np.uint8)
    dec.decode_grid_to_rgb_host([au], 1, 1, lb.CHROMA_INTERLEAVED_RGB, out=out)
    assert hashlib.md5(out.tobytes()).hexdigest() == "01672ec0cdf97b977628957cd6533dc2"


def test_unsupported_and_corrupt_streams_fail_cleanly(dec):
    au = bytearray(synth_stream("ctb32"))
    with pytest.raises(lb.B200Error):
        dec.decode_image(bytes(au[:len(au) // 2]))          # truncated slice data
    with pytest.raises(lb.B200Error):
        dec.decode_image(synth_stream("ctb64"), max_image_size_pixels=1000)   # security limit (decoder_libde265.cc:189-198)
    i = dec.decode_image(synth_stream("ctb32"))            # decoder still usable afterwards
    assert i.width == 128


@pytest.mark.parametrize("overlap", ["0", "1"])
def test_entropy_and_reconstruction_sequential_and_concurrent(cuda, overlap, monkeypatch):
    """K0 (CABAC) and K1 (reconstruction) run back to back for large batches and concurrently -- K1 consuming the command
    stream CTB by CTB while K0 produces it -- for small ones; both orders must give the oracle's planes."""
    monkeypatch.setenv("B200_OVERLAP", overlap)
    d = lb.Decoder(host_threads=4)
    try:
        names = ["ctb32_wpp_deep", "slices_wpp", "main12_wpp", "dependent_slices", "tile_1024_like"]
        for name in names:
            au = synth_stream(name)
            want, _ = ob.restatement_decode(au)
            d.decode_grid([au], 1, 1)
            got = d.planes_host()
            for c in range(len(want)):
                assert np.array_equal(got[c], want[c]), f"{name} plane {c} overlap={overlap}"
    finally:
        d.close()


def test_batch_of_heterogeneous_pictures(dec):
    """One batch of equally sized pictures coded with DIFFERENT parameters (CTB 16 / 32 / 64, QPs, WPP on and off, slices): the
    shape the decoder plugin's submission queue produces when libheif decodes unrelated images from several threads."""
    aus, want = [], []
    for k in range(12):
        y, cb, cr = lb.hevc_enc.synthetic_image(300 + k, 128, 128, 8, True)
        au = lb.hevc_enc.encode_intra(y, cb, cr, bit_depth=8, log2_ctb_size=4 + k % 3, qp=22 + k % 9, wpp=k % 2, seed=0xB200 + k,
                                      slice_ctb_rows=(2 if k % 4 == 3 else 0), transform_skip=k % 2, cu_qp_delta=(k // 2) % 2)
        aus.append(au)
        want.append(ob.restatement_decode(au)[0])
    dec.decode_grid(aus, cols=len(aus), rows=1)
    got = dec.planes_host()
    for k in range(len(aus)):
        for c in range(3):
            w = 128 if c == 0 else 64
            tile = got[c][:, k * w:(k + 1) * w]
            assert np.array_equal(tile, want[k][c]), f"picture {k} plane {c}: first diffs {np.argwhere(tile != want[k][c])[:4].tolist()}"


@pytest.mark.parametrize("tail", ["1"])
def test_tail_overlap_single_pictures(cuda, tail, monkeypatch):
    """Tail overlap (b200_hevc_decode.cu: K0 at full occupancy, the live K1 queued behind it through the start gate), forced
    here on single pictures (B200_TAIL_FORCE; by default only batches of more than one K0 wave take it): oracle planes."""
    monkeypatch.delenv("B200_OVERLAP", raising=False)
    monkeypatch.setenv("B200_TAIL_OVERLAP", tail)
    monkeypatch.setenv("B200_TAIL_FORCE", "1")
    d = lb.Decoder(host_threads=4)
    try:
        for name in ["ctb32_wpp_deep", "slices_wpp", "main12_wpp", "dependent_slices", "tile_1024_like", "ctb64"]:
            au = synth_stream(name)
            want, _ = ob.restatement_decode(au)
            for _ in range(2):
                d.decode_grid([au], 1, 1)
                assert d.stats().front_end == 2
                got = d.planes_host()
                for c in range(len(want)):
                    assert np.array_equal(got[c], want[c]), f"{name} plane {c} tail={tail}"
    finally:
        d.close()


@pytest.mark.parametrize("tail", ["0", "1"])
@pytest.mark.parametrize("tiles_per_chunk", [3, 6, 7])
def test_chunked_pipeline_equals_back_to_back(cuda, tiles_per_chunk, tail, monkeypatch):
    """Large grids headed for page-locked host memory go through K1 / K3 / K4 / K6 in bands of tile rows, the D2H of a band
    overlapping the kernels of the next.  Forced here on a small 3 x 5 grid of different pictures (B200_CHUNKS=1): planes ==
    per-tile oracle, RGB (page-locked and pageable destination, asynchronous form, cropped canvas) == the one-launch pipeline."""
    import torch
    from util import oracle_postprocess
    cols, rows, tw, th = 3, 5, 128, 64
    tiles = []
    for k in range(cols * rows):
        y, cb, cr = lb.hevc_enc.synthetic_image(0xC00 + k, tw, th, 8, True)
        tiles.append(lb.hevc_enc.encode_intra(y, cb, cr, log2_ctb_size=4 + k % 2, wpp=(k % 3 != 0), qp=24 + k % 5, seed=0xB200 + k, slice_ctb_rows=(1 if k == 4 else 0),
                                              vui_present=1, colour_description_present=1, colour_primaries=1, transfer_characteristics=13, matrix_coefficients=6, full_range=k % 2 * 0))
    ref = [ob.restatement_decode(t)[0] for t in tiles]
    W, H = cols * tw, rows * th
    want = [np.zeros((H, W), np.uint16), np.zeros((H // 2, W // 2), np.uint16), np.zeros((H // 2, W // 2), np.uint16)]
    for k in range(cols * rows):
        col, row = k % cols, k // cols
        for c in range(3):
            s = 1 if c == 0 else 2
            want[c][row * th // s:(row + 1) * th // s, col * tw // s:(col + 1) * tw // s] = ref[k][c]
    monkeypatch.setenv("B200_CHUNKS", "0")
    monkeypatch.setenv("B200_TAIL_OVERLAP", "0")
    d = lb.Decoder(host_threads=4)
    try:
        base = np.empty((H, W * 3), np.uint8)
        d.decode_grid_to_rgb_host(tiles, cols, rows, lb.CHROMA_INTERLEAVED_RGB, out=base)
        assert d.stats().front_end != 3
        base_crop = np.empty((H - 30, (W - 50) * 3), np.uint8)
        d.decode_grid_to_rgb_host(tiles, cols, rows, lb.CHROMA_INTERLEAVED_RGB, out=base_crop, canvas=(W - 50, H - 30))
        monkeypatch.setenv("B200_CHUNKS", "1")
        monkeypatch.setenv("B200_CHUNK_TILES", str(tiles_per_chunk))
        monkeypatch.setenv("B200_TAIL_OVERLAP", tail)      # bands with the live K1 of each band behind a full-occupancy K0
        monkeypatch.setenv("B200_TAIL_FORCE", "1")
        d.decode_grid(tiles, cols=cols, rows=rows)
        assert d.stats().front_end == 3
        got = d.planes_host()
        for c in range(3):
            assert np.array_equal(got[c], want[c]), f"plane {c}"
        pageable = np.empty((H, W * 3), np.uint8)
        d.decode_grid_to_rgb_host(tiles, cols, rows, lb.CHROMA_INTERLEAVED_RGB, out=pageable)
        assert np.array_equal(pageable, base)
        pinned = torch.empty((H, W * 3), dtype=torch.uint8, pin_memory=True)
        for _ in range(3):                                  # repeated: buffers, queues and flags are re-armed per call
            pinned.zero_()
            d.decode_grid_to_rgb_host(tiles, cols, rows, lb.CHROMA_INTERLEAVED_RGB, out=pinned.numpy())
            assert np.array_equal(pinned.numpy(), base)
        pinned.zero_()
        for _ in range(3):
            d.decode_grid_to_rgb_host_async(tiles, cols, rows, lb.CHROMA_INTERLEAVED_RGB, out=pinned.numpy())
        d.wait()
        assert np.array_equal(pinned.numpy(), base)
        crop = torch.empty((H - 30, (W - 50) * 3), dtype=torch.uint8, pin_memory=True)
        d.decode_grid_to_rgb_host(tiles, cols, rows, lb.CHROMA_INTERLEAVED_RGB, out=crop.numpy(), canvas=(W - 50, H - 30))
        assert np.array_equal(crop.numpy(), base_crop)
        # a corrupt tile in the middle chunk: an error, not a hang; the decoder stays usable
        bad = list(tiles)
        b = bytearray(bad[7]); b[len(b) // 2:len(b) // 2 + 40] = bytes(40); bad[7] = bytes(b)
        try:
            d.decode_grid_to_rgb_host(bad, cols, rows, lb.CHROMA_INTERLEAVED_RGB, out=pinned.numpy())
        except lb.B200Error:
            pass
        d.decode_grid_to_rgb_host(tiles, cols, rows, lb.CHROMA_INTERLEAVED_RGB, out=pinned.numpy())
        assert np.array_equal(pinned.numpy(), base)
    finally:
        d.close()


CHROMA_FORMAT_STREAMS = [c[0] for c in SYNTH_CPU_EXTRA if c[4] in (2, 3)]


@pytest.mark.parametrize("name", CHROMA_FORMAT_STREAMS)
@pytest.mark.parametrize("stage", [0, 1])
def test_422_and_444_coded_pictures_match_oracle(dec, name, stage):
    """chroma_format_idc 2 / 3: the Cb and Cr planes are reconstructed by luma-like work items from their own commands (two
    square blocks per unit in 4:2:2); deblocking and SAO use the format's chroma grid.  Stage 1 = before the in-loop filters."""
    au = synth_stream(name)
    want, info = ob.restatement_decode(au, stage)           # cropped to the conformance window
    dec.set_debug_stage(stage)
    try:
        i = dec.decode_image(au)
        if stage == 0:
            got = dec.planes_host()
        else:
            h, w = want[0].shape
            got = dec.debug_tile(0, (w + 7) & ~7, (h + 7) & ~7)
    finally:
        dec.set_debug_stage(0)
    assert i.chroma == info["chroma"] and i.bit_depth == info["bit_depth"]
    for c in range(3):
        hh, ww = want[c].shape
        assert np.array_equal(got[c][:hh, :ww], want[c]), f"{name} stage {stage}: plane {c} first diffs {np.argwhere(got[c][:hh, :ww] != want[c])[:4].tolist()}"


@pytest.mark.parametrize("name,out_chroma", [("x_444_basic", lb.CHROMA_INTERLEAVED_RGB), ("x_422_basic", lb.CHROMA_INTERLEAVED_RGB), ("x_444_main10_ctb16_random_tskip", lb.CHROMA_INTERLEAVED_RRGGBB_LE),
                                             ("x_422_main12_ctb64_deep_dqp", lb.CHROMA_INTERLEAVED_RRGGBBAA_BE)])
def test_422_and_444_to_rgb_through_the_fused_entry_point(dec, name, out_chroma):
    from util import oracle_postprocess
    au = synth_stream(name)
    planes, info = ob.restatement_decode(au)
    want, ow, oh = oracle_postprocess(planes[0], planes[1], planes[2], None, info["chroma"], info["bit_depth"], (info["cp"], info["tc"], info["mc"], info["full_range"]), [], out_chroma)
    bpp = {10: 3, 11: 4, 12: 6, 13: 8, 14: 6, 15: 8}[out_chroma]
    out = np.empty((oh, ow * bpp), np.uint8)
    dec.decode_grid_to_rgb_host([au], 1, 1, out_chroma, out=out)
    assert np.array_equal(out.reshape(-1), want)


def test_grid_of_444_tiles(dec):
    tiles, want = [], []
    for k in range(4):
        y, cb, cr = lb.hevc_enc.synthetic_image(0x444 + k, 64, 64, 8, 3)
        au = lb.hevc_enc.encode_intra(y, cb, cr, log2_ctb_size=4 + k % 2, wpp=k % 2, seed=k + 1)
        tiles.append(au); want.append(ob.restatement_decode(au)[0])
    dec.decode_grid(tiles, cols=2, rows=2)
    got = dec.planes_host()
    for k in range(4):
        r, c0 = divmod(k, 2)
        for c in range(3):
            assert np.array_equal(got[c][r * 64:(r + 1) * 64, c0 * 64:(c0 + 1) * 64], want[k][c]), f"tile {k} plane {c}"
