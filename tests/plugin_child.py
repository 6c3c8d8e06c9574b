"""Child process of tests/test_plugin*.py (never imports torch: libheif_ref.so is loaded RTLD_GLOBAL here).
usage: plugin_child.py encode-cpu | roundtrip-gpu"""
import ctypes as C
import hashlib
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
from oracle import bindings as ob  # noqa: E402
from oracle import refheif as rh  # noqa: E402
from libheif_b200 import _lib  # noqa: E402

mode = sys.argv[1]
if mode == "plugin-path-gpu":
    # LIBHEIF_PLUGIN_PATH loading (libheif/plugins_unix.cc:33-119, init.cc:124-133): libheif dlopen()s every *.so of the directory and
    # registers the table behind its `plugin_info` symbol -- nothing here calls heif_register_decoder_plugin
    plugdir = tempfile.mkdtemp()
    os.symlink(os.path.join(ROOT, "libheif_b200", "libb200heif.so"), os.path.join(plugdir, "libb200heif.so"))
    os.environ["LIBHEIF_PLUGIN_PATH"] = plugdir
h = rh.load()
b200 = _lib.lib()
assert b200.b200_plugin_bind_libheif(None) == 0, "plugin could not resolve the libheif C API"
rh.check(h.heif_register_encoder_plugin(b200.b200_get_encoder_plugin()), "register encoder plugin")
rh.register_cpu_decoder()

sys.path.insert(0, os.path.join(ROOT, "tests"))
from libheif_b200.hevc_enc import synthetic_image  # noqa: E402  (pure numpy helper)

res = {}
tmp = tempfile.mkdtemp()
nclx = (1, 13, 6, 1)
# single image, odd size -> conformance window + (possibly) clap written by libheif
y, cb, cr = synthetic_image(1, 200, 136, 8, True)
img = rh.make_ycbcr_image(y, cb, cr, 8, nclx)
rh.encode_file(os.path.join(tmp, "single.heic"), [img], quality=70)
cpu_single = rh.decode_file(os.path.join(tmp, "single.heic"), decoder_id="b200-oracle")
res["single_shape"] = list(cpu_single.shape)
ref_y = np.repeat(y[:, :, None], 3, 2)
res["single_psnr_luma_vs_green"] = float(10 * np.log10(255 ** 2 / max(1e-9, np.mean((cpu_single.reshape(136, 200, 3)[:, :, 1].astype(float) - y.astype(float)) ** 2))))
# 3x2 grid of 128x128 tiles through heif_context_encode_grid (same encoder instance for every tile, grid.cc:886-906)
tiles = []
for k in range(6):
    ty, tcb, tcr = synthetic_image(100 + k, 128, 128, 8, True)
    tiles.append(rh.make_ycbcr_image(ty, tcb, tcr, 8, nclx))
rh.encode_file(os.path.join(tmp, "grid.heic"), tiles, columns=3, rows=2, quality=60, params={"log2-ctb-size": 5})
cpu_grid = rh.decode_file(os.path.join(tmp, "grid.heic"), decoder_id="b200-oracle", threads=4)
res["grid_shape"] = list(cpu_grid.shape)
res["grid_md5_cpu"] = hashlib.md5(cpu_grid.tobytes()).hexdigest()
res["single_md5_cpu"] = hashlib.md5(cpu_single.tobytes()).hexdigest()
# oracle/heic_writer.py: the same tiles wrapped by our own ISOBMFF writer must decode to the same picture as the file the
# reference's writer produced (same encoder parameters -> byte-identical access units)
from oracle import heic_writer as hw  # noqa: E402
from libheif_b200 import hevc_enc  # noqa: E402
aus = []
for k in range(6):
    ty, tcb, tcr = synthetic_image(100 + k, 128, 128, 8, True)
    aus.append(hevc_enc.encode_intra(ty, tcb, tcr, bit_depth=8, log2_ctb_size=5, qp=51 - (60 * 45 + 50) // 100, wpp=1, seed=0xB200, vui_present=1,
                                     colour_description_present=1, colour_primaries=1, transfer_characteristics=13, matrix_coefficients=6, full_range=1))
hw.write_heic(os.path.join(tmp, "grid_own.heic"), aus, cols=3, rows=2)
own = rh.decode_file(os.path.join(tmp, "grid_own.heic"), decoder_id="b200-oracle", threads=4)
res["grid_md5_own_writer"] = hashlib.md5(own.tobytes()).hexdigest()
hw.write_heic(os.path.join(tmp, "single_own.heic"), aus[:1])
res["single_own_shape"] = list(rh.decode_file(os.path.join(tmp, "single_own.heic"), decoder_id="b200-oracle").shape)
if mode == "plugin-path-gpu":
    h.heif_init.restype = rh.Err
    h.heif_init.argtypes = [C.c_void_p]
    rh.check(h.heif_init(None), "heif_init")
    for name in ("single", "grid"):
        a = rh.decode_file(os.path.join(tmp, name + ".heic"), decoder_id="b200", threads=8)
        res[name + "_md5_gpu"] = hashlib.md5(a.tobytes()).hexdigest()
    # concurrency: an 8x8 grid decoded from 64 libheif threads, one plugin instance per tile, all in flight at once
    # (the shape of the reference's tests/test-race.go); the submission queue must batch them and stay bit-exact
    aus64 = []
    for k in range(64):
        ty, tcb, tcr = synthetic_image(300 + k, 128, 128, 8, True)
        aus64.append(hevc_enc.encode_intra(ty, tcb, tcr, bit_depth=8, log2_ctb_size=5 + k % 2, qp=22 + k % 9, wpp=(k // 2) % 2, seed=0xB200 + k, vui_present=1,     # (CTB 16 is left out: FFmpeg's chroma SAO deviates there, DESIGN.md 3)
                                           colour_description_present=1, colour_primaries=1, transfer_characteristics=13, matrix_coefficients=6, full_range=1))
    # (tiles of one grid share the parameter sets in a real file; here every tile gets its own hvcC-less item through separate files)
    same = [hevc_enc.encode_intra(*synthetic_image(400 + k, 128, 128, 8, True), bit_depth=8, log2_ctb_size=5, qp=26, wpp=1, seed=0xB200, vui_present=1,
                                  colour_description_present=1, colour_primaries=1, transfer_characteristics=13, matrix_coefficients=6, full_range=1) for k in range(64)]
    hw.write_heic(os.path.join(tmp, "grid64.heic"), same, cols=8, rows=8)
    cpu64 = rh.decode_file(os.path.join(tmp, "grid64.heic"), decoder_id="b200-oracle", threads=8)
    res["grid64_md5_cpu"] = hashlib.md5(cpu64.tobytes()).hexdigest()
    for rep in range(3):
        g64 = rh.decode_file(os.path.join(tmp, "grid64.heic"), decoder_id="b200", threads=64)
        res[f"grid64_md5_gpu_{rep}"] = hashlib.md5(g64.tobytes()).hexdigest()
    st = (C.c_uint64 * 3)()
    b200.b200_plugin_queue_stats(st)
    res["queue_batches"], res["queue_pictures"], res["queue_max_batch"] = int(st[0]), int(st[1]), int(st[2])
    # different pictures in flight at once (mixed CTB sizes / QPs / WPP): single-image files decoded from 16 Python threads
    import threading
    files = []
    for k, a in enumerate(aus64[:16]):
        f = os.path.join(tmp, f"one{k}.heic"); hw.write_heic(f, [a]); files.append(f)
    want = [hashlib.md5(rh.decode_file(f, decoder_id="b200-oracle").tobytes()).hexdigest() for f in files]
    got = [None] * len(files)
    def work(i):
        try:
            got[i] = hashlib.md5(rh.decode_file(files[i], decoder_id="b200").tobytes()).hexdigest()
        except Exception as e:  # noqa: BLE001
            got[i] = "ERR " + str(e)[:200]
    th = [threading.Thread(target=work, args=(i,)) for i in range(len(files))]
    [t.start() for t in th]; [t.join() for t in th]
    # 4:2:2 and 4:4:4 coded pictures through heif_decode_image (the plugin returns heif_chroma_422 / _444 planes; the reference converts them)
    cf_ok, cf_bad = True, []
    for cf, bd, outc in ((2, 8, rh.CHROMA_INTERLEAVED_RGB), (3, 8, rh.CHROMA_INTERLEAVED_RGB), (2, 10, 14), (3, 12, 14)):
        py, pcb, pcr = synthetic_image(500 + cf + bd, 160, 96, bd, cf)
        a = hevc_enc.encode_intra(py, pcb, pcr, bit_depth=bd, log2_ctb_size=5, qp=24, wpp=1, vui_present=1, colour_description_present=1, colour_primaries=1,
                                  transfer_characteristics=13, matrix_coefficients=6, full_range=bd == 8)
        f = os.path.join(tmp, f"cf{cf}_{bd}.heic"); hw.write_heic(f, [a])
        w_ = hashlib.md5(rh.decode_file(f, chroma=outc, decoder_id="b200-oracle").tobytes()).hexdigest()
        g_ = hashlib.md5(rh.decode_file(f, chroma=outc, decoder_id="b200").tobytes()).hexdigest()
        if w_ != g_:
            cf_ok = False; cf_bad.append((cf, bd))
    res["chroma_formats_ok"] = cf_ok
    res["chroma_formats_bad"] = cf_bad
    res["mixed_ok"] = got == want
    res["mixed_bad"] = [(i, got[i][:120]) for i in range(len(files)) if got[i] != want[i]]
if mode == "roundtrip-gpu":
    rh.check(h.heif_register_decoder_plugin(b200.b200_get_decoder_plugin()), "register decoder plugin")
    for name in ("single", "grid"):
        a = rh.decode_file(os.path.join(tmp, name + ".heic"), decoder_id="b200", threads=8)      # explicit selection (decoder.cc:330-338)
        res[name + "_md5_gpu"] = hashlib.md5(a.tobytes()).hexdigest()
        bdef = rh.decode_file(os.path.join(tmp, name + ".heic"), threads=8)                        # priority selection: 200 > 500? (oracle reports 500)
        res[name + "_md5_default"] = hashlib.md5(bdef.tobytes()).hexdigest()
if mode == "roundtrip-gpu":
    # the call sequence of a sequence track (sequences/track_visual.cc:212-275) straight on the plugin table: one instance, one
    # push_data2 per sample with its user_data (parameter sets only in the first), pictures come back in order with the
    # user_data they were pushed with
    FN = C.CFUNCTYPE
    class DecPlugin(C.Structure):
        _fields_ = [("api", C.c_int), ("name", C.c_void_p), ("init", C.c_void_p), ("deinit", C.c_void_p), ("supports", C.c_void_p),
                    ("new_decoder", C.c_void_p), ("free_decoder", FN(None, C.c_void_p)), ("push_data", C.c_void_p), ("decode_image", C.c_void_p),
                    ("set_strict", C.c_void_p), ("id_name", C.c_char_p), ("decode_next", C.c_void_p), ("min_version", C.c_uint32), ("supports2", C.c_void_p),
                    ("new_decoder2", FN(rh.Err, C.POINTER(C.c_void_p), C.c_void_p)), ("push_data2", FN(rh.Err, C.c_void_p, C.c_char_p, C.c_size_t, C.c_size_t)),
                    ("flush_data", FN(rh.Err, C.c_void_p)), ("decode_next2", FN(rh.Err, C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), C.c_void_p))]
    tab = C.cast(b200.b200_get_decoder_plugin(), C.POINTER(DecPlugin)).contents
    frames = []
    for k in range(3):
        fy, fcb, fcr = synthetic_image(500 + k, 96, 64, 8, True)
        frames.append(hevc_enc.encode_intra(fy, fcb, fcr, bit_depth=8, log2_ctb_size=4, qp=25 + k, wpp=1, seed=0xB200))
    inst = C.c_void_p()
    rh.check(tab.new_decoder2(C.byref(inst), None), "new_decoder2")
    for k, au in enumerate(frames):
        nals = hw.split_nals(au)
        keep = nals if k == 0 else [x for x in nals if ((x[0] >> 1) & 0x3f) < 32]       # later samples carry no parameter sets
        data = b"".join(len(x).to_bytes(4, "big") + x for x in keep)
        rh.check(tab.push_data2(inst, data, len(data), 1000 + k), "push_data2")
    rh.check(tab.flush_data(inst), "flush_data")
    seq_ok, users = True, []
    for k in range(3):
        img, user = C.c_void_p(), C.c_size_t()
        rh.check(tab.decode_next2(inst, C.byref(img), C.byref(user), None), "decode_next_image2")
        users.append(int(user.value))
        st = C.c_int()
        ptr = h.heif_image_get_plane_readonly(img, rh.CHANNEL_Y, C.byref(st))
        got_y = np.ctypeslib.as_array(ptr, shape=(64, st.value))[:, :96]
        want_y = ob.ffmpeg_decode(frames[k], 1)[0][0]
        seq_ok = seq_ok and np.array_equal(got_y.astype(np.uint16), np.asarray(want_y).astype(np.uint16))
        h.heif_image_release(img)
    img, user = C.c_void_p(), C.c_size_t()
    rh.check(tab.decode_next2(inst, C.byref(img), C.byref(user), None), "decode_next_image2 (drained)")
    res["sequence_users"] = users; res["sequence_planes_ok"] = bool(seq_ok); res["sequence_drained"] = img.value is None
    tab.free_decoder(inst)
print("RESULT " + json.dumps(res))
