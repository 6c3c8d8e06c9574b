"""Mode-decision speeds of the GPU HEVC encoder (b200_hevc_enc_params::speed): the argument checks and the plugin parameter
without a device; on the GPU, speed 0 (the default) writes the bytes recorded in tests/golden/gpu_encoder_md5.json, speeds 1
and 2 write conforming streams whose reconstruction every decoder reproduces, batches do not change bytes, the work
counters follow the quadtree, compression stays within stated bounds of speed 0, the one-call grid path matches the two-step
route, and the "b200-gpu" plugin's "speed" parameter works inside the unmodified reference libheif."""
import ctypes as C
import hashlib
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import libheif_b200 as lb
from libheif_b200 import _lib
from libheif_b200.hevc_enc import GpuEncoder, default_params, gpu_params, grid_encode_check, synthetic_image
from oracle import bindings as ob
from test_hevc_gpu_encoder import CONF, _call_device, _planes, lcg_noise, psnr, source

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "gpu_encoder_md5.json")
SPEEDS = [0, 1, 2]


# ------------------------------------------------------------------------------------------------ CPU
def test_default_speed_is_0():
    assert default_params().speed == 0
    assert gpu_params(64, 64, True).speed == 0


@pytest.mark.parametrize("speed", SPEEDS)
def test_check_accepts_speed(speed):
    assert _call_device(gpu_params(64, 64, True, speed=speed), 1, _planes(1)) == 0
    assert _call_device(gpu_params(64, 64, False, speed=speed), 2, _planes(2, chroma=0)) == 0
    rgb = np.zeros((64, 96, 3), np.uint8)
    assert grid_encode_check(rgb, 32, 32, speed=speed) is None


@pytest.mark.parametrize("speed", [-1, 3])
def test_check_refuses_speed(speed):
    assert _call_device(gpu_params(64, 64, True, speed=speed), 1, _planes(1)) == -1        # B200_E_INVALID
    assert "speed" in _lib.lib().b200_last_error().decode()
    with pytest.raises(lb.B200Error) as e:
        grid_encode_check(np.zeros((64, 96, 3), np.uint8), 32, 32, speed=speed)
    assert e.value.code == -1 and "speed" in str(e.value), str(e.value)


def _plugin_params(getter):
    class Integer(C.Structure):
        _fields_ = [("default_value", C.c_int), ("have_minmax", C.c_uint8), ("minimum", C.c_int), ("maximum", C.c_int),
                    ("valid_values", C.c_void_p), ("num_valid_values", C.c_int)]

    class Param(C.Structure):         # b200h_encoder_parameter == heif_encoder_parameter (heif_plugin.h)
        _fields_ = [("version", C.c_int), ("name", C.c_char_p), ("type", C.c_int), ("integer", Integer), ("has_default", C.c_int)]

    words = (C.c_void_p * 33).from_address(getattr(_lib.lib(), getter)())        # b200h_encoder_plugin as pointer-sized words (x86-64 layout)
    lst = C.CFUNCTYPE(C.POINTER(C.POINTER(Param)), C.c_void_p)(words[15])(None)
    out = []
    for i in range(16):
        if not lst[i]:
            break
        q = lst[i].contents
        out.append((q.name.decode(), q.version, q.has_default, q.integer.default_value, q.integer.minimum, q.integer.maximum))
    return out


def test_plugin_speed_parameter():
    gpu = _plugin_params("b200_get_gpu_encoder_plugin")
    assert ("speed", 2, 1, 0, 0, 2) in gpu, gpu
    assert "speed" not in [p[0] for p in _plugin_params("b200_get_encoder_plugin")]


def e1_resources():
    """{speed: (registers, stack bytes, static shared memory bytes, spill store + load bytes)} of E1 from the -Xptxas -v log
    that the build keeps beside its objects."""
    log = os.path.join(ROOT, "libheif_b200", "build", "b200_hevc_gpu_enc.cu.ptxas.txt")
    if not os.path.exists(log):
        pytest.skip("no ptxas log of b200_hevc_gpu_enc.cu (library built elsewhere)")
    out = {}
    for chunk in open(log).read().split("Compiling entry function")[1:]:
        m = re.match(r" '_ZN4b2004genc9e1_kernelILi(\d)E", chunk)
        if m:
            st = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", chunk)
            use = re.search(r"Used (\d+) registers.*?(\d+) bytes smem", chunk)
            out[int(m.group(1))] = (int(use.group(1)), int(st.group(1)), int(use.group(2)), int(st.group(2)) + int(st.group(3)))
    return out


def test_e1_resources():
    """Speed 0 keeps the resources of the encoder before speeds existed; no instantiation spills; speed 2 has no luma save
    buffers."""
    res = e1_resources()
    assert set(res) == set(SPEEDS), res
    assert res[0] == (186, 432, 33460, 0), res[0]
    assert all(r[3] == 0 for r in res.values()), res
    assert res[0][2] - res[2][2] >= 4 * 4096 - 64, res[2]                # the four 4 KB luma save buffers are gone


def quadtree_work(w, h, log2ctb):
    """(PU searches, eval_cu calls) of one picture's decision pass: CTB down to 8x8 with NxN at 8x8, implied splits where a CU
    crosses the (8-aligned) coded picture's border; a 64x64 CU is one search (on its first 32x32 block)."""
    W, H = (w + 7) & ~7, (h + 7) & ~7
    n = [0, 0]

    def decide(x0, y0, L):
        s = 1 << L
        if x0 + s > W or y0 + s > H:
            for k in range(4):
                x1, y1 = x0 + (k & 1) * s // 2, y0 + (k >> 1) * s // 2
                if x1 < W and y1 < H:
                    decide(x1, y1, L - 1)
            return
        n[0] += 1
        n[1] += 1
        if L == 3:
            n[0] += 4
            n[1] += 1
        else:
            for k in range(4):
                decide(x0 + (k & 1) * s // 2, y0 + (k >> 1) * s // 2, L - 1)

    c = 1 << log2ctb
    for y in range(0, H, c):
        for x in range(0, W, c):
            decide(x, y, log2ctb)
    return n[0], n[1]


def test_quadtree_work_interior_ctb():
    assert quadtree_work(32, 32, 5) == (85, 37)
    assert quadtree_work(64, 64, 6) == (1 + 4 * 85, 1 + 4 * 37)


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


def golden_cases():
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import make_gpu_encoder_md5 as m
    return m.cases(), m.encode


@pytest.mark.gpu
def test_speed0_is_the_recorded_encoder(enc):
    """Default parameters == speed=0 == the md5 recorded before speeds existed; the counters at speed 0 are the full
    search over the quadtree."""
    with open(GOLDEN) as f:
        want = json.load(f)
    cases, encode = golden_cases()
    assert len(cases) == len(want) >= 6
    for cid, case in cases:
        a = encode(enc, case)
        st = enc.stats()
        b = encode(enc, case, speed=0)
        assert hashlib.md5(a).hexdigest() == want[cid], cid
        assert a == b, cid
        pus, cus = quadtree_work(case[0], case[1], case[3])
        assert (st.mode_evaluations, st.cu_evaluations) == (35 * pus, cus), cid


CONF_IDS = [f"{c[0]}x{c[1]}-{'420' if c[2] else '400'}-ctb{1 << c[3]}-qp{c[4]}-{c[5]}-{i}" for i, c in enumerate(CONF)]


def _decoders_agree(enc, dec, au, w, h, n):
    ff, _, _ = ob.ffmpeg_decode(au)
    rs, _ = ob.restatement_decode(au)
    dec.set_debug_stage(0)
    dec.decode_image(au)
    got = dec.planes_host()
    for c in range(n):
        assert np.array_equal(ff[c], rs[c]), f"plane {c}: FFmpeg != restatement"
        assert np.array_equal(got[c], rs[c]), f"plane {c}: decoder != restatement"
    rec = enc.recon(0)
    s1, _ = ob.restatement_decode(au, 1)
    dec.set_debug_stage(1)
    try:
        dec.decode_image(au)
        dbg = dec.debug_tile(0, (w + 7) & ~7, (h + 7) & ~7)
    finally:
        dec.set_debug_stage(0)
    for c in range(n):
        hh, ww = s1[c].shape
        assert np.array_equal(rec[c], s1[c]), f"plane {c}: recon != restatement stage 1"
        assert np.array_equal(dbg[c][:hh, :ww], s1[c]), f"plane {c}: decoder stage 1 != restatement stage 1"
    return rs


@pytest.mark.gpu
@pytest.mark.parametrize("speed", [1, 2])
@pytest.mark.parametrize("case", CONF, ids=CONF_IDS)
def test_conformance(enc, dec, case, speed):
    w, h, chroma, log2ctb, qp, kind, extra = case
    y, cb, cr = source(kind, w, h, chroma)
    au = enc.encode([(y, cb, cr)], log2_ctb_size=log2ctb, qp=qp, speed=speed, **extra)[0]
    rs = _decoders_agree(enc, dec, au, w, h, 3 if chroma else 1)
    if kind == "flat":
        assert psnr(rs[0], y) > 60


@pytest.mark.gpu
@pytest.mark.parametrize("speed", [1, 2])
def test_worst_case_noise_qp0(enc, dec, speed):
    """LCG noise at QP 0 with CTB 64: the densest sub-streams stay inside the worst-case buffer."""
    y, cb, cr = lcg_noise(0xB200, 256, 128)
    au = enc.encode([(y, cb, cr)], qp=0, log2_ctb_size=6, speed=speed)[0]
    rs = _decoders_agree(enc, dec, au, 256, 128, 3)
    assert psnr(rs[0], y) > 45
    assert len(au) * 8 / (256 * 128 * 1.5) > 4


@pytest.mark.gpu
@pytest.mark.parametrize("speed", SPEEDS)
def test_deterministic_and_batch_independent(enc, speed):
    tiles = [synthetic_image(0xB200 + k, 256, 256, 8, True) for k in range(16)]
    a = enc.encode(tiles, qp=27, speed=speed)
    assert enc.encode(tiles, qp=27, speed=speed) == a
    for k in range(16):
        assert enc.encode([tiles[k]], qp=27, speed=speed)[0] == a[k], f"tile {k}: batch != alone"


@pytest.mark.gpu
@pytest.mark.parametrize("case", [CONF[i] for i in (0, 2, 5, 6, 10, 11)], ids=[CONF_IDS[i] for i in (0, 2, 5, 6, 10, 11)])
def test_work_counters(enc, case):
    """Speeds 1 and 2 walk the same quadtree (same eval_cu count) and evaluate at most 18 of the 35 modes per PU search."""
    w, h, chroma, log2ctb, qp, kind, extra = case
    pics = [tuple(source(kind, w, h, chroma, seed=0xB200 + k)) for k in range(3)]
    pus, cus = quadtree_work(w, h, log2ctb)
    enc.encode(pics, log2_ctb_size=log2ctb, qp=qp, **extra)
    s0 = enc.stats()
    assert (s0.mode_evaluations, s0.cu_evaluations) == (3 * 35 * pus, 3 * cus)
    for speed in (1, 2):
        enc.encode(pics, log2_ctb_size=log2ctb, qp=qp, speed=speed, **extra)
        st = enc.stats()
        assert st.cu_evaluations == s0.cu_evaluations, speed
        assert st.mode_evaluations * 35 <= s0.mode_evaluations * 18, (speed, st.mode_evaluations, s0.mode_evaluations)
        assert st.mode_evaluations >= 3 * 11 * pus, speed                  # round 1 alone has 11 fixed modes


@pytest.mark.gpu
def test_quality_against_speed0(enc):
    """8 synthetic 256x256 tiles at QP 22 / 27 / 32 / 37 against speed 0 at the same QP: speed 1 at most 3 % more bytes in
    total and a mean luma PSNR at most 0.1 dB lower; speed 2 at most 8 % more bytes and 0.3 dB lower."""
    tiles = [synthetic_image(0xB200 + k, 256, 256, 8, True) for k in range(8)]
    bounds = {1: (1.03, 0.1), 2: (1.08, 0.3)}
    for qp in (22, 27, 32, 37):
        got = {}
        for speed in SPEEDS:
            aus = enc.encode(tiles, qp=qp, log2_ctb_size=5, speed=speed)
            got[speed] = (sum(map(len, aus)), float(np.mean([psnr(ob.ffmpeg_decode(a)[0][0], t[0]) for a, t in zip(aus, tiles)])))
        print(f"qp {qp}: " + ", ".join(f"speed {s} {b} bytes {p:.3f} dB" for s, (b, p) in got.items()))
        b0, p0 = got[0]
        for speed, (rb, dp) in bounds.items():
            b, p = got[speed]
            assert b <= rb * b0 and p >= p0 - dp, (qp, speed, b, b0, p, p0)


@pytest.mark.gpu
@pytest.mark.parametrize("layout", ["rgb24", "planar_alpha"])
def test_grid_speed2_equals_two_step_route(enc, layout):
    from test_gpu_grid_encode import nclx_params, source as grid_source, two_step
    w, h, tw, th = 452, 462, 128, 128
    rgb, a, aplane = grid_source(layout, w, h)
    prm = dict(nclx_params(6, False), speed=2)
    got = enc.encode_rgb_grid(rgb, tw, th, alpha=a, **prm)
    tiles, atiles = two_step(enc, rgb, aplane, w, h, tw, th, prm)
    assert got["tiles"] == tiles
    assert (got["alpha"] is None) == (aplane is None)
    if aplane is not None:
        assert got["alpha"] == atiles
    assert got["tiles"] != two_step(enc, rgb, None, w, h, tw, th, nclx_params(6, False))[0]     # speed reached the kernels


@pytest.mark.gpu
def test_grid_stats_sum_both_batches(enc):
    from test_gpu_grid_encode import source as grid_source
    rgb, a, _ = grid_source("planar_alpha", 256, 128)
    enc.encode_rgb_grid(rgb, 128, 128, alpha=a, qp=27, speed=2)
    st = enc.stats()
    pus, cus = quadtree_work(128, 128, 5)
    assert st.cu_evaluations == 2 * 2 * cus                                 # 2 colour + 2 alpha tiles
    assert 2 * 2 * 11 * pus <= st.mode_evaluations <= 2 * 2 * 18 * pus


@pytest.mark.gpu
def test_speed2_fits_more_e1_warps(enc):
    w = {s: enc.e1_warps_per_sm(s) for s in SPEEDS}
    assert w[0] == w[1] == 6, w
    assert w[2] > 6, w


@pytest.mark.gpu
def test_speed_through_reference_libheif(cuda):
    """"b200-gpu" with speed=2 inside the unmodified reference libheif (child process, tests/gpu_speed_plugin_child.py): RGB,
    RGBA and a 3x2 grid decode to the same picture with the FFmpeg-backed CPU plugin and this library's decoder plugin,
    close to the source; speed=0 writes the file the default writes; a speed-2 sequence is the same at sequence-batch 1
    and 0."""
    if not (os.path.exists(os.path.join(ob.REF, "libheif_ref.so")) and os.path.exists(os.path.join(ob.REF, "liboracle_plugin.so")) and ob.avcodec_dir()):
        pytest.skip("oracle/_ref reference build not present")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "gpu_speed_plugin_child.py")], stdout=subprocess.PIPE, stderr=subprocess.PIPE,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    res = json.loads([l for l in r.stdout.splitlines() if l.startswith("RESULT ")][-1][7:])
    assert res["rgb"]["shape"] == [136, 600] and res["rgba"]["shape"] == [136, 800] and res["grid"]["shape"] == [256, 1152], res
    for k in ("rgb", "rgba", "grid"):
        assert res[k]["same_decoders"], k
        assert res[k]["psnr"] > 28, (k, res[k]["psnr"])
    d = res["default"]
    assert d["speed0"] == d["unset"], d
    assert d["speed2"] != d["unset"], d
    assert res["sequence"]["1"] == res["sequence"]["0"], res["sequence"]


@pytest.mark.gpu
def test_speed2_decides_from_the_source(enc):
    """Open loop: speed 2's decisions depend on the source and lambda alone.  QP pairs with the same lambda (0 / 1, 2 / 3,
    4 / 5) reconstruct differently but must give the same decisions; mode_evaluations (which follows the chosen modes through
    the MPM candidates of later PUs) fingerprints them.  Closed loop (speed 1) sees the different reconstructions."""
    pics = [tuple(lcg_noise(0x5EED + k, 128, 128)) for k in range(2)] + [tuple(synthetic_image(0x5EED, 128, 128, 8, True))]
    closed_differs = False
    for qa, qb in ((0, 1), (2, 3), (4, 5)):
        ev = {}
        for speed in (1, 2):
            for qp in (qa, qb):
                enc.encode(pics, qp=qp, speed=speed)
                ev[speed, qp] = enc.stats().mode_evaluations
        assert ev[2, qa] == ev[2, qb], (qa, qb, ev)
        closed_differs |= ev[1, qa] != ev[1, qb]
    assert closed_differs
