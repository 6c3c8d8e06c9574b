"""GPU HEVC intra encoder (b200_gpu_encoder_*): streams decoded identically by FFmpeg, the C restatement and this library's
decoder; reconstruction equal to what a decoder holds before deblocking; deterministic bytes, alone or in a batch;
compression against the host encoder with the same tool set; parameter refusals without a device."""
import ctypes as C

import numpy as np
import pytest

import libheif_b200 as lb
from libheif_b200 import _lib
from libheif_b200.hevc_enc import GpuEncoder, gpu_params, substream_capacity, synthetic_image
from oracle import bindings as ob


def lcg_noise(seed, w, h, chroma=True):
    s = seed & 0xFFFFFFFF
    out = []
    for c in range(3 if chroma else 1):
        hh, ww = (h, w) if c == 0 else ((h + 1) // 2, (w + 1) // 2)
        v = np.empty(hh * ww, np.uint8)
        for i in range(v.size):
            s = (s * 1664525 + 1013904223) & 0xFFFFFFFF
            v[i] = s >> 24
        out.append(v.reshape(hh, ww))
    return out if chroma else [out[0], None, None]


def flat(w, h, chroma=True):
    y = np.full((h, w), 97, np.uint8)
    return [y, np.full(((h + 1) // 2, (w + 1) // 2), 140, np.uint8), np.full(((h + 1) // 2, (w + 1) // 2), 110, np.uint8)] if chroma else [y, None, None]


def source(kind, w, h, chroma, seed=0xB200):
    if kind == "synthetic":
        return synthetic_image(seed, w, h, 8, chroma)
    if kind == "flat":
        return flat(w, h, chroma)
    return lcg_noise(seed, w, h, chroma)


def psnr(a, b):
    mse = np.mean((a.astype(np.float64) - b.astype(np.float64)) ** 2)
    return 99.0 if mse == 0 else 10 * np.log10(255.0 ** 2 / mse)


# ------------------------------------------------------------------------------------------------ CPU: refusals, bound
def _call_device(p, n, planes):
    # b200_gpu_encode_check: the argument check the encode calls run before touching CUDA, without encoding
    return _lib.lib().b200_gpu_encode_check(C.byref(p) if p is not None else None, n, planes)


def _planes(n, w=64, h=64, chroma=1):
    arr = (_lib.Planes * n)()
    for q in arr:
        q.y, q.cb, q.cr = 0x1000, 0x2000, 0x3000        # only checked for NULL
        q.y_stride, q.c_stride, q.width, q.height, q.chroma, q.bit_depth = w, (w + 1) // 2, w, h, chroma, 8
    return arr


REFUSED = [("sao", 1), ("sign_data_hiding", 1), ("transform_skip", 1), ("cu_qp_delta", 1), ("scaling_lists", 1), ("pcm", 1),
           ("transquant_bypass", 1), ("tile_cols", 2), ("tile_rows", 2), ("slice_ctb_rows", 1), ("dependent_slice_segments", 1),
           ("bit_depth", 10), ("chroma_format_idc", 2), ("chroma_format_idc", 3), ("wpp", 0), ("log2_ctb_size", 4)]


@pytest.mark.parametrize("field,value", REFUSED, ids=[f"{f}={v}" for f, v in REFUSED])
def test_refused_field(field, value):
    p = gpu_params(64, 64, True, **{field: value})
    rc = _call_device(p, 1, _planes(1))
    assert rc == -2, rc                                     # B200_E_UNSUPPORTED
    msg = _lib.lib().b200_last_error().decode()
    assert field.split("_")[0] in msg, msg


def test_invalid_arguments():
    p = gpu_params(64, 64, True)
    assert _call_device(p, 0, _planes(1)) == -1             # n <= 0
    assert _call_device(p, -3, _planes(1)) == -1
    assert _call_device(None, 1, _planes(1)) == -1
    assert _call_device(p, 1, None) == -1
    mixed = _planes(3)
    mixed[2].width = 72
    assert _call_device(p, 3, mixed) == -1                  # mixed sizes in one batch
    nulls = _planes(2)
    nulls[1].cb = None
    assert _call_device(p, 2, nulls) == -1                  # NULL chroma plane
    nulls = _planes(1)
    nulls[0].y = None
    assert _call_device(p, 1, nulls) == -1
    assert _call_device(gpu_params(64, 64, True, qp=52), 1, _planes(1)) == -1
    assert _call_device(gpu_params(4, 64, True), 1, _planes(1, w=4)) == -1
    assert _call_device(p, 3, _planes(3)) == 0              # the same arguments, valid
    assert _call_device(gpu_params(64, 64, False), 1, _planes(1, chroma=0)) == 0


def _worst_bits_per_8x8_cu(chroma):
    """Independent worst case of one 8x8 CU coded as NxN (the densest syntax), from the binarisations of 7.3.8 / 9.3.3:
    a context-coded bin costs at most 6 output bits (rangeTabLps >= 6 -> 6 renormalisation shifts), a bypass bin 1."""
    ctx_bits = 6
    # coeff_abs_level_remaining of the largest level (32767, base level 1): prefix / suffix of 9.3.3.11 with rice 0
    rem, k = 32766, 0
    q = (rem >> k) - 2
    kk = q.bit_length() - 1
    rem_bits = (kk + 3 + 1) + (kk + k)
    per_coef = 3 * ctx_bits + 1 + rem_bits                  # sig, gt1, gt2, sign, remaining
    tbs = 4 + (2 if chroma else 0)                          # four 4x4 luma TBs, one 4x4 Cb and Cr
    per_tb = (2 * 3 * ctx_bits + 2 * 0) + ctx_bits + ctx_bits   # last x / y prefixes (cMax 3), cbf, csbf
    cu = ctx_bits * (1 + 1 + 4 + 1 + 2) + 4 * 5            # split, part mode, 4 prev_intra flags, chroma mode, 2 cbf_cb/cr; 4 x 5 rem bits
    return tbs * (16 * per_coef + per_tb) + cu


@pytest.mark.parametrize("log2ctb", [5, 6])
@pytest.mark.parametrize("chroma", [True, False])
def test_substream_capacity_covers_worst_case(log2ctb, chroma):
    ctb = 1 << log2ctb
    for width in (8, 136, 1024, 16384):
        wctb = (((width + 7) & ~7) + ctb - 1) // ctb
        cus = wctb * (ctb // 8) ** 2
        worst = cus * _worst_bits_per_8x8_cu(chroma) + wctb * 8 + 16     # + end_of_slice_segment_flag per CTB, row end
        assert substream_capacity(width, log2ctb, chroma) * 8 >= worst


# ------------------------------------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def enc(cuda):
    e = GpuEncoder()
    yield e
    e.close()


@pytest.fixture(scope="module", params=["device", "host"])
def dec(cuda, request):
    d = lb.Decoder(host_threads=8)
    d.set_front_end(request.param == "device")
    yield d
    d.close()


CONF = [
    # (w, h, chroma, log2ctb, qp, source, extra)
    (8, 8, True, 5, 22, "synthetic", {}),
    (64, 64, True, 5, 0, "synthetic", {}),
    (64, 64, False, 6, 37, "noise", {}),
    (136, 72, True, 6, 22, "synthetic", dict(deblocking_disabled=1)),
    (136, 72, False, 5, 51, "synthetic", {}),
    (452, 462, True, 5, 37, "synthetic", dict(beta_offset_div2=3, tc_offset_div2=-2)),
    (452, 462, True, 6, 22, "flat", {}),
    (136, 72, True, 5, 22, "noise", dict(cb_qp_offset=4, cr_qp_offset=-3, slice_chroma_qp_offsets=1, slice_cb_qp_offset=-2, slice_cr_qp_offset=2)),
    (64, 64, True, 5, 27, "synthetic", dict(slice_deblocking_override=1, slice_beta_offset_div2=-3, slice_tc_offset_div2=4)),
    (64, 64, True, 6, 27, "synthetic", dict(max_transform_hierarchy_depth_intra=3, strong_intra_smoothing=0)),
    (1024, 1024, True, 5, 51, "synthetic", {}),
    (1024, 1024, False, 6, 22, "synthetic", {}),
]


@pytest.mark.gpu
@pytest.mark.parametrize("case", CONF, ids=[f"{c[0]}x{c[1]}-{'420' if c[2] else '400'}-ctb{1 << c[3]}-qp{c[4]}-{c[5]}-{i}" for i, c in enumerate(CONF)])
def test_conformance(enc, dec, case):
    w, h, chroma, log2ctb, qp, kind, extra = case
    y, cb, cr = source(kind, w, h, chroma)
    au = enc.encode([(y, cb, cr)], log2_ctb_size=log2ctb, qp=qp, **extra)[0]
    ff, _, _ = ob.ffmpeg_decode(au)
    rs, _ = ob.restatement_decode(au)
    dec.set_debug_stage(0)
    dec.decode_image(au)
    got = dec.planes_host()
    for c in range(len(rs)):
        assert np.array_equal(ff[c], rs[c]), f"plane {c}: FFmpeg != restatement"
        assert np.array_equal(got[c], rs[c]), f"plane {c}: decoder != restatement"
    # reconstruction = every decoder's picture before deblocking
    rec = enc.recon(0)
    s1, _ = ob.restatement_decode(au, 1)
    dec.set_debug_stage(1)
    try:
        dec.decode_image(au)
        dbg = dec.debug_tile(0, (w + 7) & ~7, (h + 7) & ~7)
    finally:
        dec.set_debug_stage(0)
    for c in range(len(s1)):
        hh, ww = s1[c].shape
        assert np.array_equal(rec[c], s1[c]), f"plane {c}: recon != restatement stage 1"
        assert np.array_equal(dbg[c][:hh, :ww], s1[c]), f"plane {c}: decoder stage 1 != restatement stage 1"
    if kind == "flat":
        assert psnr(rs[0], y) > 60


@pytest.mark.gpu
def test_device_planes_match_host_planes(enc):
    import torch
    pics = [synthetic_image(0xB200 + k, 200, 136, 8, True) for k in range(3)]
    host = enc.encode(pics, qp=27)
    dev = enc.encode([tuple(torch.from_numpy(a).cuda() for a in p) for p in pics], qp=27)
    assert host == dev


@pytest.mark.gpu
def test_deterministic_and_batch_independent(enc):
    tiles = [synthetic_image(0xB200 + k, 256, 256, 8, True) for k in range(16)]
    a = enc.encode(tiles, qp=27)
    b = enc.encode(tiles, qp=27)
    assert a == b
    for k in range(16):
        assert enc.encode([tiles[k]], qp=27)[0] == a[k], f"tile {k}: batch != alone"


@pytest.mark.gpu
def test_grid_decode(enc, dec):
    tiles = [synthetic_image(0xC000 + k, 256, 256, 8, True) for k in range(16)]
    aus = enc.encode(tiles, qp=30)
    dec.set_debug_stage(0)
    dec.decode_grid(aus, cols=4, rows=4)
    got = dec.planes_host()
    for k, au in enumerate(aus):
        rs, _ = ob.restatement_decode(au)
        col, row = k % 4, k // 4
        for c in range(3):
            s = 1 if c == 0 else 2
            t = got[c][row * 256 // s:(row + 1) * 256 // s, col * 256 // s:(col + 1) * 256 // s]
            assert np.array_equal(t, rs[c]), f"tile {k} plane {c}"


@pytest.mark.gpu
def test_worst_case_noise_qp0(enc, dec):
    """LCG noise at QP 0 with CTB 64: the largest levels and sub-streams (escape codes, the sub-stream bound)."""
    y, cb, cr = lcg_noise(0xB200, 256, 128)
    au = enc.encode([(y, cb, cr)], qp=0, log2_ctb_size=6)[0]
    ff, _, _ = ob.ffmpeg_decode(au)
    rs, _ = ob.restatement_decode(au)
    dec.set_debug_stage(0)
    dec.decode_image(au)
    got = dec.planes_host()
    s1, _ = ob.restatement_decode(au, 1)
    rec = enc.recon(0)
    for c in range(3):
        assert np.array_equal(ff[c], rs[c]) and np.array_equal(got[c], rs[c]), f"plane {c}: decoders disagree"
        assert np.array_equal(rec[c], s1[c]), f"plane {c}: recon != restatement stage 1"
    assert psnr(rs[0], y) > 45
    assert len(au) * 8 / (256 * 128 * 1.5) > 4                # a dense stream: bits per sample


@pytest.mark.gpu
def test_quality_against_host_encoder(enc):
    """Same tool set (no SAO, sign hiding or cu_qp_delta): at every QP the GPU streams are no larger in total and their
    mean luma PSNR is at most 0.1 dB lower."""
    tiles = [synthetic_image(0xB200 + k, 256, 256, 8, True) for k in range(8)]
    for qp in (22, 27, 32, 37):
        g = enc.encode(tiles, qp=qp, log2_ctb_size=5)
        h = [lb.hevc_enc.encode_intra(*t, qp=qp, log2_ctb_size=5, sao=0, sign_data_hiding=0, cu_qp_delta=0, wpp=1, seed=0xB200 + k)
             for k, t in enumerate(tiles)]
        gp = np.mean([psnr(ob.ffmpeg_decode(a)[0][0], t[0]) for a, t in zip(g, tiles)])
        hp = np.mean([psnr(ob.ffmpeg_decode(a)[0][0], t[0]) for a, t in zip(h, tiles)])
        gb, hb = sum(map(len, g)), sum(map(len, h))
        print(f"qp {qp}: GPU {gb} bytes {gp:.3f} dB, host {hb} bytes {hp:.3f} dB")
        assert gb <= hb and gp >= hp - 0.1, (qp, gb, hb, gp, hp)


# ------------------------------------------------------------------------------------------------ through libheif
@pytest.mark.gpu
def test_gpu_encoder_plugin_through_reference_libheif(cuda):
    """The "b200-gpu" heif_encoder_plugin inside the unmodified reference libheif (child process, tests/gpu_plugin_child.py):
    heif_context_encode_image of RGB (the reference's colour conversion) and RGBA (alpha through the same plugin as 4:0:0),
    heif_context_encode_grid of a 3x2 grid; every file decodes with the FFmpeg-backed CPU plugin to the same picture as with
    this library's decoder plugin, with the right sizes and alpha, and close to the source."""
    import json
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if not (os.path.exists(os.path.join(ob.REF, "libheif_ref.so")) and os.path.exists(os.path.join(ob.REF, "liboracle_plugin.so")) and ob.avcodec_dir()):
        pytest.skip("oracle/_ref reference build not present")
    r = subprocess.run([sys.executable, os.path.join(root, "tests", "gpu_plugin_child.py")], stdout=subprocess.PIPE, stderr=subprocess.PIPE,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads([l for l in r.stdout.splitlines() if l.startswith("RESULT ")][-1][7:])
    assert res["encoder_ids"][0] == "b200-gpu", res["encoder_ids"]           # chosen by priority (60 > 50)
    assert res["rgb"]["shape"] == [136, 600] and not res["rgb"]["has_alpha"]
    assert res["rgba"]["shape"] == [136, 800] and res["rgba"]["has_alpha"]
    assert res["grid"]["shape"] == [256, 1152]
    for k in ("rgb", "rgba", "grid"):
        assert res[k]["md5_cpu"] == res[k]["md5_gpu_decoder"], k
        assert res[k]["psnr"] > 28, (k, res[k]["psnr"])       # sanity floor: QP 19 plus the RGB <-> YCbCr round trip
    assert res["rgba"]["alpha_psnr"] > 28
    assert res["bit_depth_refused"], res
