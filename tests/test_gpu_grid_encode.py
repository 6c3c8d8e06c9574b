"""One-call RGB -> HEIC grid encoder on the GPU (b200_gpu_encode_rgb_grid_*, GpuEncoder.encode_rgb_grid): refusals without a
device; every tile byte for byte what the two-step route writes (RGB -> YCbCr of the edge-padded tile, then the GPU encoder);
host and device forms alike; the grid decodes back; and, inside the unmodified reference libheif, the same picture as
heif_context_encode_grid with the "b200-gpu" plugin.

Run as a script (`python tests/test_gpu_grid_encode.py child <file>`) this file is the child process of the last test: it
loads the reference libheif RTLD_GLOBAL and therefore never imports torch."""
import ctypes as C
import functools
import hashlib
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import libheif_b200 as lb  # noqa: E402
from libheif_b200 import _lib  # noqa: E402
from libheif_b200.hevc_enc import GpuEncoder, gpu_params, grid_encode_check, synthetic_image  # noqa: E402


@functools.lru_cache(maxsize=None)
def picture(w, h, nch, seed=0x61D):
    """[h, w, nch] uint8: one synthetic_image luma plane per channel (smooth gradients, gratings and noise)."""
    return np.stack([synthetic_image(seed + c, w, h, 8, False)[0] for c in range(nch)], axis=2)


def source(layout, w, h):
    """(rgb argument of encode_rgb_grid, alpha argument, alpha plane or None) of one input layout."""
    px = picture(w, h, 4 if layout in ("rgba32", "planar_alpha") else 3)
    if layout == "rgb24" or layout == "rgba32":
        return px, None, (px[:, :, 3] if layout == "rgba32" else None)
    planes = tuple(np.ascontiguousarray(px[:, :, c]) for c in range(3))
    a = np.ascontiguousarray(px[:, :, 3]) if layout == "planar_alpha" else None
    return planes, a, a


def nclx_params(mc, full, qp=27):
    cp = 9 if mc == 9 else 1
    return dict(qp=qp, log2_ctb_size=5, vui_present=1, colour_description_present=1, colour_primaries=cp, transfer_characteristics=13,
                matrix_coefficients=mc, full_range=int(full))


def padded_windows(a, w, h, tw, th):
    """The tiles of plane / interleaved picture `a` ([h, w] or [h, w, c]) in raster order, edge-replicated past the picture."""
    cols, rows = -(-w // tw), -(-h // th)
    pad = ((0, rows * th - h), (0, cols * tw - w)) + ((0, 0),) * (a.ndim - 2)
    p = np.pad(a, pad, mode="edge")
    return [np.ascontiguousarray(p[r * th:(r + 1) * th, c * tw:(c + 1) * tw]) for r in range(rows) for c in range(cols)]


def two_step(enc, rgb, alpha_plane, w, h, tw, th, params, convert=None):
    """The route a caller takes without the one-call path: pad and cut the RGB tiles on the host, convert each with
    lb.rgb_to_ycbcr_ex_host (or `convert`), encode the tiles with GpuEncoder.encode; alpha tiles as 4:0:0 pictures."""
    planar = isinstance(rgb, tuple)
    if planar:
        srcs = list(rgb) + ([alpha_plane] if alpha_plane is not None else [])
    else:
        srcs = [rgb]
    wins = [padded_windows(s, w, h, tw, th) for s in srcs]
    pics = []
    for k in range(len(wins[0])):
        t = tuple(wn[k] for wn in wins) if planar else wins[0][k]
        if convert is not None:
            pics.append(convert(t))
        else:
            img, _ = lb.rgb_to_ycbcr_ex_host(t, out_chroma=lb.CHROMA_420, matrix_coefficients=params["matrix_coefficients"],
                                             colour_primaries=params["colour_primaries"], full_range=bool(params["full_range"]))
            pics.append((img.y, img.cb, img.cr))
    tiles = enc.encode(pics, **params)
    if alpha_plane is None:
        return tiles, None
    return tiles, enc.encode([(a, None, None) for a in padded_windows(alpha_plane, w, h, tw, th)], **params)


# ------------------------------------------------------------------------------------------------ CPU: the host-only check
def _check_raw(rgb_image, tw, th, p, opt=None):
    return _lib.lib().b200_gpu_encode_rgb_grid_check(C.byref(rgb_image) if rgb_image is not None else None, tw, th,
                                                     C.byref(p) if p is not None else None, C.byref(opt) if opt is not None else None)


def _refusal(code, fn, *a, **kw):
    with pytest.raises(lb.B200Error) as e:
        fn(*a, **kw)
    assert e.value.code == code, str(e.value)
    return str(e.value)


def test_check_refuses_depth_above_8():
    rrggbb = np.zeros((64, 64, 3), np.uint16)
    assert "bit depth 10" in _refusal(-2, grid_encode_check, rrggbb, 32, 32, input_bit_depth=10, endianness="little")
    planar16 = tuple(np.zeros((64, 64), np.uint16) for _ in range(3))
    assert "bit depth 16" in _refusal(-2, grid_encode_check, planar16, 32, 32, input_bit_depth=16)


@pytest.mark.parametrize("mc", [11, 14])
def test_check_refuses_matrix(mc):
    assert f"matrix_coefficients {mc}" in _refusal(-2, grid_encode_check, picture(64, 64, 3), 32, 32, matrix_coefficients=mc)


def test_check_refuses_average_with_only_use_preferred():
    msg = _refusal(-2, grid_encode_check, picture(64, 64, 3), 32, 32, chroma_downsampling=2, only_use_preferred=True)
    assert "only_use_preferred" in msg
    assert grid_encode_check(picture(64, 64, 3), 32, 32, chroma_downsampling=1, only_use_preferred=True) is None


def _refused_fields():
    from test_hevc_gpu_encoder import REFUSED
    return REFUSED


@pytest.mark.parametrize("field,value", _refused_fields(), ids=[f"{f}={v}" for f, v in _refused_fields()])
def test_check_refuses_encoder_field(field, value):
    msg = _refusal(-2, grid_encode_check, picture(64, 64, 3), 32, 32, **{field: value})
    assert field.split("_")[0] in msg, msg


@pytest.mark.parametrize("tw,th,what", [(127, 128, "odd"), (128, 65, "odd"), (6, 128, "too small"), (128, 4, "too small"),
                                        (16386, 128, "too large"), (128, 16386, "too large")])
def test_check_refuses_tile_size(tw, th, what):
    assert f"tile size {tw}x{th}" in _refusal(-1, grid_encode_check, picture(64, 64, 3), tw, th), what


def test_check_refuses_null_pointers():
    rgb = picture(64, 64, 3)
    d = _lib.RgbImage()
    d.rgb, d.rgb_stride, d.width, d.height, d.chroma, d.bit_depth = rgb.ctypes.data, rgb.strides[0], 64, 64, lb.CHROMA_INTERLEAVED_RGB, 8
    p = gpu_params(32, 32, True)
    assert _check_raw(d, 32, 32, p) == 0
    assert _check_raw(None, 32, 32, p) == -1
    assert _check_raw(d, 32, 32, None) == -1
    d.rgb = None
    assert _check_raw(d, 32, 32, p) == -1
    assert "missing" in _lib.lib().b200_last_error().decode()
    q = _lib.RgbImage()
    r = np.zeros((64, 64), np.uint8)
    q.r, q.g, q.b, q.r_stride, q.g_stride, q.b_stride = r.ctypes.data, r.ctypes.data, None, 64, 64, 64
    q.width, q.height, q.chroma, q.bit_depth = 64, 64, lb.CHROMA_444, 8
    assert _check_raw(q, 32, 32, p) == -1
    l = _lib.lib()
    d.rgb = rgb.ctypes.data                             # a NULL encoder is refused before any CUDA call
    assert l.b200_gpu_encode_rgb_grid_host(None, C.byref(d), 32, 32, C.byref(p), None, None) == -1
    assert l.b200_gpu_encode_rgb_grid_device(None, C.byref(d), 32, 32, C.byref(p), None, None, None) == -1


@pytest.mark.parametrize("layout", ["rgb24", "rgba32", "planar", "planar_alpha"])
def test_check_accepts_8bit_layouts(layout):
    rgb, a, _ = source(layout, 200, 136)
    assert grid_encode_check(rgb, 128, 128, alpha=a, qp=27) is None
    assert grid_encode_check(rgb, 200, 136, alpha=a, qp=27, matrix_coefficients=0) is None


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def enc(cuda):
    e = GpuEncoder()
    yield e
    e.close()


LAYOUTS = ["rgb24", "rgba32", "planar", "planar_alpha"]
SIZES = [(384, 256, 128, 128), (452, 462, 128, 128), (200, 136, 200, 136)]


@pytest.mark.gpu
@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("size", SIZES, ids=[f"{s[0]}x{s[1]}-in-{s[2]}x{s[3]}" for s in SIZES])
def test_tiles_equal_two_step_route(enc, size, layout):
    """Matrices 1, 5, 6, 9 (and 0, the special branch of Op_RGB_to_YCbCr) at limited and full range."""
    w, h, tw, th = size
    rgb, a, aplane = source(layout, w, h)
    for mc in (1, 5, 6, 9, 0):
        for full in (False, True):
            prm = nclx_params(mc, full)
            got = enc.encode_rgb_grid(rgb, tw, th, alpha=a, **prm)
            cols, rows = -(-w // tw), -(-h // th)
            assert (got["cols"], got["rows"], got["width"], got["height"]) == (cols, rows, w, h)
            tiles, atiles = two_step(enc, rgb, aplane, w, h, tw, th, prm)
            assert len(got["tiles"]) == cols * rows
            for k in range(cols * rows):
                assert got["tiles"][k] == tiles[k], f"matrix {mc} full {full}: colour tile {k}"
            assert (got["alpha"] is None) == (aplane is None)
            if aplane is not None:
                for k in range(cols * rows):
                    assert got["alpha"][k] == atiles[k], f"matrix {mc} full {full}: alpha tile {k}"


BIG = [("rgb24", 6, False), ("rgba32", 9, True), ("planar_alpha", 1, False)]


@pytest.mark.gpu
@pytest.mark.parametrize("layout,mc,full", BIG, ids=[f"{b[0]}-mc{b[1]}-{'full' if b[2] else 'limited'}" for b in BIG])
def test_large_grid_equals_two_step_route(enc, layout, mc, full):
    """4096 x 4096 in 512 x 512 tiles: several row bands in the host form."""
    w = h = 4096
    rgb, a, aplane = source(layout, w, h)
    prm = nclx_params(mc, full)
    got = enc.encode_rgb_grid(rgb, 512, 512, alpha=a, **prm)
    tiles, atiles = two_step(enc, rgb, aplane, w, h, 512, 512, prm)
    assert got["tiles"] == tiles
    assert got["alpha"] == atiles


@pytest.mark.gpu
def test_tiles_equal_reference_convert_colorspace(enc):
    """The tile planes from the unmodified reference's convert_colorspace instead of this library's conversion."""
    from oracle import ref_encode
    if ref_encode.lib() is None:
        pytest.skip("oracle/_ref reference build not present")
    w, h, tw, th = 452, 462, 128, 128
    rgb, _, aplane = source("rgba32", w, h)
    prm = nclx_params(6, False)

    def convert(t):
        y, cb, cr, _, _ = ref_encode.ref_rgb_to_ycbcr_ex(t.reshape(th, tw * 4), 11, 8, lb.CHROMA_420, (1, 13, 6, 0))
        return y, cb, cr

    got = enc.encode_rgb_grid(rgb, tw, th, **prm)
    tiles, atiles = two_step(enc, rgb, aplane, w, h, tw, th, prm, convert=convert)
    assert got["tiles"] == tiles
    assert got["alpha"] == atiles


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["rgba32", "planar_alpha"])
def test_device_form_equals_host_form(enc, layout):
    import torch
    w, h = 452, 462
    rgb, a, _ = source(layout, w, h)
    host = enc.encode_rgb_grid(rgb, 128, 128, alpha=a, qp=30)
    again = enc.encode_rgb_grid(rgb, 128, 128, alpha=a, qp=30)
    if isinstance(rgb, tuple):
        drgb, da = tuple(torch.from_numpy(p).cuda() for p in rgb), torch.from_numpy(a).cuda()
    else:
        drgb, da = torch.from_numpy(rgb).cuda(), None
    dev = enc.encode_rgb_grid(drgb, 128, 128, alpha=da, qp=30)
    for k in ("tiles", "alpha", "cols", "rows", "width", "height", "pipeline"):
        assert host[k] == dev[k] == again[k], k
    assert host["upload_ms"] > 0 and dev["upload_ms"] == 0
    st = enc.stats()
    assert st.pictures == 2 * 16 and st.analyse_ms > 0


def psnr(a, b):
    mse = np.mean((a.astype(np.float64) - b.astype(np.float64)) ** 2)
    return 99.0 if mse == 0 else 10 * np.log10(255.0 ** 2 / mse)


@pytest.mark.gpu
def test_grid_decodes_back(enc, tmp_path):
    """452 x 462 in 128 x 128 tiles (overhang on both sides): the access units as a grid file; this library's decoder with the
    overhang clipped, FFmpeg and the C restatement per tile give the same picture, close to the converted source."""
    from oracle import bindings as ob
    from oracle.heic_writer import write_heic
    w, h, tw, th = 452, 462, 128, 128
    rgb, _, aplane = source("rgba32", w, h)
    prm = nclx_params(6, False)
    got = enc.encode_rgb_grid(rgb, tw, th, **prm)
    cols, rows = got["cols"], got["rows"]
    path = write_heic(str(tmp_path / "grid.heic"), got["tiles"], cols, rows, out_w=w, out_h=h, nclx=(1, 13, 6, 0))
    assert os.path.getsize(path) > sum(map(len, got["tiles"])) * 0.9
    dec = lb.Decoder(host_threads=8)
    try:
        for aus, chroma in ((got["tiles"], True), (got["alpha"], False)):
            dec.decode_grid(aus, cols=cols, rows=rows, canvas=(w, h))
            planes = dec.planes_host()
            want = [np.zeros((rows * th, cols * tw), np.uint8)]
            if chroma:
                want += [np.zeros((rows * th // 2, cols * tw // 2), np.uint8) for _ in range(2)]
            for k, au in enumerate(aus):
                rs, _ = ob.restatement_decode(au)
                ff, _, _ = ob.ffmpeg_decode(au)
                r, c = divmod(k, cols)
                for p in range(len(want)):
                    s = 1 if p == 0 else 2
                    assert np.array_equal(ff[p], rs[p]), f"tile {k} plane {p}: FFmpeg != restatement"
                    want[p][r * th // s:(r + 1) * th // s, c * tw // s:(c + 1) * tw // s] = rs[p]
            for p in range(len(want)):
                s = 1 if p == 0 else 2
                assert planes[p].shape == ((h + s - 1) // s, (w + s - 1) // s)
                assert np.array_equal(planes[p], want[p][:planes[p].shape[0], :planes[p].shape[1]]), f"plane {p}"
            if chroma:
                img, _ = lb.rgb_to_ycbcr_ex_host(rgb, out_chroma=lb.CHROMA_420, matrix_coefficients=6, colour_primaries=1, full_range=False)
                assert psnr(planes[0], img.y) > 30
            else:
                assert psnr(planes[0], aplane) > 30
    finally:
        dec.close()


@pytest.mark.gpu
def test_same_picture_as_libheif_encode_grid(enc, tmp_path):
    """384 x 256 RGB24 as six 128 x 128 tiles, two ways: heif_context_encode_grid with the "b200-gpu" plugin in the unmodified
    reference libheif (quality 53 -> QP 27 through the plugin's mapping; the reference converts each tile with its default
    sRGB nclx 1 / 13 / 6 / full), and this call written with write_heic.  Both files decode through the reference with the
    FFmpeg-backed CPU plugin to the same RGB."""
    from oracle import bindings as ob
    from oracle.heic_writer import write_heic
    if not (os.path.exists(os.path.join(ob.REF, "libheif_ref.so")) and os.path.exists(os.path.join(ob.REF, "liboracle_plugin.so")) and ob.avcodec_dir()):
        pytest.skip("oracle/_ref reference build not present")
    got = enc.encode_rgb_grid(picture(384, 256, 3), 128, 128, **nclx_params(6, True))
    ours = write_heic(str(tmp_path / "ours.heic"), got["tiles"], 3, 2, out_w=384, out_h=256, nclx=(1, 13, 6, 1))
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "child", ours], stdout=subprocess.PIPE, stderr=subprocess.PIPE,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("RESULT ")][-1][7:])
    assert res["encoder"] == "b200-gpu", res
    assert res["libheif"]["shape"] == res["ours"]["shape"] == [256, 384 * 3]
    assert res["libheif"]["md5"] == res["ours"]["md5"], res
    assert res["ours"]["psnr"] > 28, res


def _child(ours):
    from oracle import refheif as rh
    h = rh.load()
    b200 = _lib.lib()
    assert b200.b200_plugin_bind_libheif(None) == 0, "plugin could not resolve the libheif C API"
    rh.check(h.heif_register_encoder_plugin(b200.b200_get_gpu_encoder_plugin()), "register GPU encoder plugin")
    rh.register_cpu_decoder()
    ctx = h.heif_context_alloc()
    e = C.c_void_p()
    rh.check(h.heif_context_get_encoder_for_format(ctx, rh.COMPRESSION_HEVC, C.byref(e)), "get_encoder_for_format")
    name = h.heif_encoder_get_name(e).decode()
    h.heif_encoder_release(e)
    h.heif_context_free(ctx)
    px = picture(384, 256, 3)
    images = []
    for t in padded_windows(px, 384, 256, 128, 128):
        img = C.c_void_p()
        rh.check(h.heif_image_create(128, 128, rh.COLORSPACE_RGB, rh.CHROMA_INTERLEAVED_RGB, C.byref(img)))
        rh.check(h.heif_image_add_plane(img, rh.CHANNEL_INTERLEAVED, 128, 128, 8))
        st = C.c_int()
        p = h.heif_image_get_plane(img, rh.CHANNEL_INTERLEAVED, C.byref(st))
        np.ctypeslib.as_array(p, shape=(128, st.value))[:, :128 * 3] = t.reshape(128, 128 * 3)
        images.append(img)
    theirs = os.path.join(tempfile.mkdtemp(), "libheif.heic")
    rh.encode_file(theirs, images, columns=3, rows=2, quality=53, params={"log2-ctb-size": 5})
    res = {"encoder": "b200-gpu" if "GPU" in name else name}
    for k, f in (("libheif", theirs), ("ours", ours)):
        out = rh.decode_file(f, chroma=rh.CHROMA_INTERLEAVED_RGB, decoder_id="b200-oracle")
        mse = np.mean((out.reshape(256, 384, 3).astype(np.float64) - px) ** 2)
        res[k] = dict(shape=list(out.shape), md5=hashlib.md5(out.tobytes()).hexdigest(), psnr=float(10 * np.log10(255.0 ** 2 / max(mse, 1e-12))))
    print("RESULT " + json.dumps(res))


if __name__ == "__main__" and len(sys.argv) == 3 and sys.argv[1] == "child":
    _child(sys.argv[2])
