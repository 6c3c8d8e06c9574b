"""Child process of tests/test_sequences_gpu.py (never imports torch: libheif_ref.so is loaded RTLD_GLOBAL here).
Image sequences through the unmodified reference libheif with this library's plugins: heif_track_encode_sequence_image with
the "b200" (host) or "b200-gpu" encoder table; the raw samples read with heif_track_get_next_raw_sequence_sample and decoded
by FFmpeg behind the track's hvcC parameter sets; the track decoded with heif_track_decode_next_image through this library's
decoder plugin.

    python tests/seq_plugin_child.py cpu            # "b200" table only, no device
    python tests/seq_plugin_child.py gpu <batch> [seq37]   # "b200-gpu" table at sequence-batch <batch>, and the decoder plugin
    python tests/seq_plugin_child.py memlimit       # the decoder plugin's read-ahead under a low max_total_memory
"""
import ctypes as C
import hashlib
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
from oracle import bindings as ob  # noqa: E402
from oracle import refheif as rh  # noqa: E402
import refheif_seq as rs  # noqa: E402
from libheif_b200 import _lib  # noqa: E402
from libheif_b200.hevc_enc import encode_intra, synthetic_image  # noqa: E402  (host encoder, numpy helper)

mode = sys.argv[1]
h = rs.load()
b200 = _lib.lib()
assert b200.b200_plugin_bind_libheif(None) == 0, "plugin could not resolve the libheif C API"
if mode in ("cpu", "memlimit"):
    rh.check(h.heif_register_encoder_plugin(b200.b200_get_encoder_plugin()), "register host encoder plugin")
else:
    rh.check(h.heif_register_encoder_plugin(b200.b200_get_gpu_encoder_plugin()), "register GPU encoder plugin")
if mode != "cpu":
    rh.check(h.heif_register_decoder_plugin(b200.b200_get_decoder_plugin()), "register decoder plugin")
rh.register_cpu_decoder()

QUALITY = 70
QP = 51 - (QUALITY * 45 + 50) // 100           # the plugins' quality -> QP mapping
tmp = tempfile.mkdtemp()
res = {}


def md5(b):
    return hashlib.md5(b).hexdigest()


def psnr(a, b):
    mse = np.mean((a.astype(np.float64) - b.astype(np.float64)) ** 2)
    return 99.0 if mse == 0 else float(10 * np.log10(255.0 ** 2 / mse))


def release(imgs):
    for i in imgs:
        h.heif_image_release(i)


def ycc_frames(n, w, hh, seed, chroma=True):
    return [synthetic_image(seed + k, w, hh, 8, chroma) for k in range(n)]


def rgb_frames(n, w, hh, seed, alpha=False):
    out = []
    for k in range(n):
        pl = [synthetic_image(seed + 7 * k + c, w, hh, 8, False)[0] for c in range(4 if alpha else 3)]
        out.append(np.stack(pl, axis=2))
    return out


def frames_digest(calls, keys):
    """md5 over the planes of every decoded frame (calls: refheif_seq.decode_track output) and the per-call status."""
    m = hashlib.md5()
    for c in calls:
        if c[0] != "ok":
            m.update(b"error")
            continue
        for k in keys:
            if k in c[1]:
                m.update(c[1][k].tobytes())
    return m.hexdigest()


def sample_report(path):
    samples = rs.raw_samples(path)
    return dict(count=len(samples), durations=[d for _, d in samples], sync=rs.sync_samples(path), tracks=rs.track_info(path)), samples


def ffmpeg_track(path, index=0):
    """FFmpeg's decode of every raw sample of a track, each behind the parameter sets of the track's hvcC: [[y, cb, cr]] (uint8;
    [y] for 4:0:0).  (The FFmpeg-backed oracle plugin decodes each push on its own, so it cannot follow a track whose later
    samples carry no parameter sets.)"""
    tid = rs.track_info(path)[index]["id"]
    ps = rs.parameter_sets(path)[index]
    out = []
    for sample, _ in rs.raw_samples(path, tid):
        pl, _, _ = ob.ffmpeg_decode(ps + sample)
        out.append([p.astype(np.uint8) for p in pl])
    return out


class DecPlugin(C.Structure):                 # b200h_decoder_plugin (heif_decoder_plugin, v5 members)
    FN = C.CFUNCTYPE
    _fields_ = [("api", C.c_int), ("name", C.c_void_p), ("init", C.c_void_p), ("deinit", C.c_void_p), ("supports", C.c_void_p),
                ("new_decoder", C.c_void_p), ("free_decoder", FN(None, C.c_void_p)), ("push_data", C.c_void_p), ("decode_image", C.c_void_p),
                ("set_strict", C.c_void_p), ("id_name", C.c_char_p), ("decode_next", C.c_void_p), ("min_version", C.c_uint32), ("supports2", C.c_void_p),
                ("new_decoder2", FN(rh.Err, C.POINTER(C.c_void_p), C.c_void_p)), ("push_data2", FN(rh.Err, C.c_void_p, C.c_char_p, C.c_size_t, C.c_size_t)),
                ("flush_data", FN(rh.Err, C.c_void_p)), ("decode_next2", FN(rh.Err, C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), C.c_void_p))]


def plugin_track(path, index=0):
    """This library's decoder plugin driven the way Track_Visual drives it (sequences/track_visual.cc:200-282): one instance,
    the hvcC parameter sets in front of the first sample, one push_data2 per sample with its index as user_data, and
    decode_next_image2 after every push; flush_data after the last.  No libheif colour handling in between, so the planes
    compare with FFmpeg's directly.  Returns ([[y, cb, cr]] in the order handed back, [user_data])."""
    tab = C.cast(b200.b200_get_decoder_plugin(), C.POINTER(DecPlugin)).contents
    tid = rs.track_info(path)[index]["id"]
    ps = rs.parameter_sets(path)[index]
    inst = C.c_void_p()
    rh.check(tab.new_decoder2(C.byref(inst), None), "new_decoder2")
    frames, users = [], []

    def drain():
        while True:
            img, user = C.c_void_p(), C.c_size_t()
            rh.check(tab.decode_next2(inst, C.byref(img), C.byref(user), None), "decode_next_image2")
            if not img.value:
                return
            pl = rs._planes(img.value)
            frames.append([pl[n] for n in ("y", "cb", "cr") if n in pl])
            users.append(int(user.value))
            h.heif_image_release(img)
    for k, (sample, _) in enumerate(rs.raw_samples(path, tid)):
        data = (ps + sample) if k == 0 else sample
        rh.check(tab.push_data2(inst, data, len(data), k), "push_data2")
        drain()
    rh.check(tab.flush_data(inst), "flush_data")
    drain()
    tab.free_decoder(inst)
    return frames, users


def same_planes(a, b):
    return [bool(len(x) == len(y) and all(np.array_equal(p, q) for p, q in zip(x, y))) for x, y in zip(a, b)] + [False] * abs(len(a) - len(b))


def equal_frames(calls, want, names=("y", "cb", "cr")):
    """Per frame: decode_track call k returned a picture whose planes equal want[k]."""
    return [bool(k < len(calls) and calls[k][0] == "ok" and all(np.array_equal(calls[k][1][n], w[c]) for c, n in enumerate(names) if c < len(w)))
            for k, w in enumerate(want)]


def encode_error(fn):
    try:
        fn()
        return None
    except rs.SequenceError as e:
        return dict(code=e.code, sub=e.sub, msg=str(e)[:300])
    except RuntimeError as e:
        return dict(code=-1, sub=-1, msg=str(e)[:300])


if mode == "cpu":
    # 9 RGB frames, 200x136, timescale 30000, durations 1001 + k: the track structure and the decoded pictures
    W, H, N = 200, 136, 9
    rgbs = rgb_frames(N, W, H, 0x5E0)
    f = os.path.join(tmp, "rgb.heif")
    imgs = [rh.rgb_image(x) for x in rgbs]
    rs.write_sequence(f, imgs, quality=QUALITY, timescale=30000, durations=[1001 + k for k in range(N)])
    release(imgs)
    res["rgb"], _ = sample_report(f)
    res["rgb"]["ffmpeg_sizes"] = [list(fr[0].shape) for fr in ffmpeg_track(f)]

    # 9 YCbCr 4:2:0 frames: every sample's slice NAL is the one the host encoder's still path codes for that picture, and
    # every decoded frame equals FFmpeg's decode of that still
    srcs = ycc_frames(N, W, H, 0x5F0)
    f = os.path.join(tmp, "ycc.heif")
    imgs = [rh.make_ycbcr_image(*s) for s in srcs]
    rs.write_sequence(f, imgs, quality=QUALITY, timescale=1000, durations=[40] * N)
    release(imgs)
    res["ycc"], samples = sample_report(f)
    frames = ffmpeg_track(f)
    same_bytes, same_pixels = [], []
    for k, s in enumerate(srcs):
        still = encode_intra(*s, bit_depth=8, log2_ctb_size=5, wpp=1, qp=QP, seed=0xB200)
        same_bytes.append(k < len(samples) and rs.slice_nals(samples[k][0]) == rs.slice_nals(still))
        want, _, _ = ob.ffmpeg_decode(still)
        same_pixels.append(bool(k < len(frames) and all(np.array_equal(frames[k][c], want[c].astype(np.uint8)) for c in range(3))))
    res["ycc"]["slices_equal_still"] = same_bytes
    res["ycc"]["frames_equal_ffmpeg_still"] = same_pixels

    # a frame whose size differs from the first frame's is refused
    a, b = ycc_frames(1, 64, 64, 1)[0], ycc_frames(1, 96, 64, 2)[0]
    imgs = [rh.make_ycbcr_image(*a), rh.make_ycbcr_image(*b)]
    res["size_change"] = encode_error(lambda: rs.write_sequence(os.path.join(tmp, "sz.heif"), imgs, quality=QUALITY))
    release(imgs)
elif mode == "memlimit":
    # 37 frames of 512 x 512 decoded with the context's max_total_memory at 8 MiB: 32 decoded frames at once would need 12 MiB
    src = ycc_frames(37, 512, 512, 0xA00)
    f = os.path.join(tmp, "mem.heif")
    imgs = [rh.make_ycbcr_image(*x) for x in src]
    rs.write_sequence(f, imgs, quality=QUALITY, timescale=1000, durations=[40] * 37)
    release(imgs)
    q0 = (C.c_uint64 * 3)()
    b200.b200_plugin_queue_stats(q0)
    got = rs.decode_track(f, decoder_id="b200", max_total_memory=8 << 20)
    q1 = (C.c_uint64 * 3)()
    b200.b200_plugin_queue_stats(q1)
    res["memlimit"] = dict(status=[c[0] for c in got], errors=[c[2] for c in got if c[0] == "error"][:3], md5=frames_digest(got, ("y", "cb", "cr")),
                           batches=int(q1[0] - q0[0]), max_batch=int(q1[2]))
else:
    batch = int(sys.argv[2])
    params = {"sequence-batch": batch}
    DUR37 = [40 + 3 * (k % 7) for k in range(37)]
    enc_stats0 = (C.c_uint64 * 3)()
    b200.b200_plugin_encoder_stats(enc_stats0)

    # 37 YCbCr 4:2:0 frames (not a multiple of any batch): the slice NAL of every sample is GpuEncoder.encode of that frame
    # alone (the host entry point, b200_gpu_encode_intra_host, with the plugin's parameters)
    from libheif_b200.hevc_enc import GpuEncoder
    W, H, N = 256, 200, 37
    srcs = ycc_frames(N, W, H, 0x600)
    f = os.path.join(tmp, "seq37.heif")
    imgs = [rh.make_ycbcr_image(*s) for s in srcs]
    # durations vary, so that a sample written under another frame's number would carry the wrong one
    rs.write_sequence(f, imgs, quality=QUALITY, params=params, timescale=1000, durations=DUR37)
    release(imgs)
    res["seq37"], samples = sample_report(f)
    res["seq37"]["file_md5"] = md5(open(f, "rb").read())
    ge = GpuEncoder()
    res["seq37"]["slices_equal_alone"] = [k < len(samples) and rs.slice_nals(samples[k][0]) == rs.slice_nals(ge.encode([s], qp=QP, log2_ctb_size=5)[0])
                                          for k, s in enumerate(srcs)]
    ge.close()
    enc_stats1 = (C.c_uint64 * 3)()
    b200.b200_plugin_encoder_stats(enc_stats1)
    res["seq37"]["encoder_calls"] = int(enc_stats1[0] - enc_stats0[0])
    res["seq37"]["encoder_max_batch"] = int(enc_stats1[2])

    # both decoders, the read-ahead's batches, and the source
    q0 = (C.c_uint64 * 3)()
    b200.b200_plugin_queue_stats(q0)
    gpu = rs.decode_track(f, decoder_id="b200")
    q1 = (C.c_uint64 * 3)()
    b200.b200_plugin_queue_stats(q1)
    cpu = ffmpeg_track(f)
    direct, users = plugin_track(f)
    oracle0 = rs.decode_track(f, decoder_id="b200-oracle", max_calls=1)       # the oracle plugin decodes the first sample only
    res["seq37"]["decoded_gpu"] = [c[0] for c in gpu]
    res["seq37"]["ffmpeg_frames"] = len(cpu)
    res["seq37"]["plugin_equal_ffmpeg"] = same_planes(direct, cpu)
    res["seq37"]["plugin_users"] = users
    res["seq37"]["first_equal_oracle_plugin"] = equal_frames(gpu[:1], [[oracle0[0][1][n] for n in ("y", "cb", "cr")]])[0]
    res["seq37"]["md5_gpu_decoder"] = frames_digest(gpu, ("y", "cb", "cr"))
    res["seq37"]["psnr_y_ffmpeg"] = [psnr(fr[0], srcs[k][0]) for k, fr in enumerate(cpu)]
    res["seq37"]["psnr_y"] = [psnr(c[1]["y"], srcs[k][0]) if c[0] == "ok" else 0.0 for k, c in enumerate(gpu)]
    res["seq37"]["queue_batches"] = int(q1[0] - q0[0])
    res["seq37"]["queue_pictures"] = int(q1[1] - q0[1])
    res["seq37"]["queue_max_batch"] = int(q1[2])
    if sys.argv[3:] == ["seq37"]:                   # only the 37-frame sequence
        print("RESULT " + json.dumps(res))
        sys.exit(0)

    # an encoder reused after a refused frame: the frames it had staged for the abandoned track do not reach the next one
    enc = rs.new_encoder(QUALITY, params)
    a = ycc_frames(2, 64, 64, 0x900) + ycc_frames(1, 96, 64, 0x910)
    imgs = [rh.make_ycbcr_image(*x) for x in a]
    refused = encode_error(lambda: rs.write_sequence(os.path.join(tmp, "abandoned.heif"), imgs, quality=QUALITY, params=params, encoder=enc))
    release(imgs)
    b = ycc_frames(3, 96, 64, 0x920)
    imgs = [rh.make_ycbcr_image(*x) for x in b]
    f6 = os.path.join(tmp, "reuse.heif")
    rs.write_sequence(f6, imgs, quality=QUALITY, params=params, encoder=enc, durations=[10, 20, 30])
    release(imgs)
    h.heif_encoder_release(enc)
    smp = rs.raw_samples(f6)
    ge = GpuEncoder()
    res["reuse"] = dict(refused=refused is not None, count=len(smp), durations=[d for _, d in smp],
                        slices_equal_alone=[k < len(smp) and rs.slice_nals(smp[k][0]) == rs.slice_nals(ge.encode([x], qp=QP, log2_ctb_size=5)[0]) for k, x in enumerate(b)])
    ge.close()

    # two repetitions of the track: 74 frames, the second pass equal to the first
    f2 = os.path.join(tmp, "rep.heif")
    imgs = [rh.make_ycbcr_image(*s) for s in srcs]
    rs.write_sequence(f2, imgs, quality=QUALITY, params=params, timescale=1000, durations=DUR37, repetitions=2)
    release(imgs)
    rep = rs.decode_track(f2, decoder_id="b200")
    res["repeat"] = dict(decoded=[c[0] for c in rep], md5_first=frames_digest(rep[:N], ("y", "cb", "cr")), md5_second=frames_digest(rep[N:], ("y", "cb", "cr")),
                         md5_once=frames_digest(gpu, ("y", "cb", "cr")))

    # RGBA: an alpha auxiliary track coded by its own instance of the table, as 4:0:0
    W2, H2, N2 = 200, 136, 9
    rgbas = rgb_frames(N2, W2, H2, 0x700, alpha=True)
    f3 = os.path.join(tmp, "rgba.heif")
    imgs = [rh.rgb_image(x) for x in rgbas]
    rs.write_sequence(f3, imgs, quality=QUALITY, params=params, timescale=1000, durations=[40] * N2)
    release(imgs)
    res["rgba"], _ = sample_report(f3)
    rgba = rs.decode_track(f3, rh.COLORSPACE_RGB, rh.CHROMA_INTERLEAVED_RGBA, decoder_id="b200")
    oracle0 = rs.decode_track(f3, rh.COLORSPACE_RGB, rh.CHROMA_INTERLEAVED_RGBA, decoder_id="b200-oracle", max_calls=1)
    res["rgba"]["decoded_gpu"] = [c[0] for c in rgba]
    res["rgba"]["plugin_equal_ffmpeg"] = same_planes(plugin_track(f3, 0)[0], ffmpeg_track(f3, 0))
    res["rgba"]["alpha_plugin_equal_ffmpeg"] = same_planes(plugin_track(f3, 1)[0], ffmpeg_track(f3, 1))
    res["rgba"]["first_equal_oracle_plugin"] = bool(rgba[0][0] == "ok" and np.array_equal(rgba[0][1]["interleaved"], oracle0[0][1]["interleaved"]))
    res["rgba"]["alpha_psnr"] = [psnr(c[1]["interleaved"][:, :, 3], rgbas[k][:, :, 3]) for k, c in enumerate(rgba) if c[0] == "ok"]
    res["rgba"]["rgb_psnr"] = [psnr(c[1]["interleaved"][:, :, :3], rgbas[k][:, :, :3]) for k, c in enumerate(rgba) if c[0] == "ok"]

    # monochrome
    monos = ycc_frames(11, 160, 96, 0x800, chroma=False)
    f4 = os.path.join(tmp, "mono.heif")
    imgs = [rh.make_ycbcr_image(s[0], None, None) for s in monos]
    rs.write_sequence(f4, imgs, quality=QUALITY, params=params, timescale=1000, durations=[40] * 11)
    release(imgs)
    gpu = rs.decode_track(f4, decoder_id="b200")
    cpu = ffmpeg_track(f4)
    res["mono"], _ = sample_report(f4)
    res["mono"]["decoded_gpu"] = [c[0] for c in gpu]
    res["mono"]["has_chroma"] = any("cb" in c[1] for c in gpu if c[0] == "ok")
    res["mono"]["plugin_equal_ffmpeg"] = same_planes(plugin_track(f4)[0], cpu)
    res["mono"]["psnr_y"] = [psnr(c[1]["y"], monos[k][0]) if c[0] == "ok" else 0.0 for k, c in enumerate(gpu)]

    # refusals: a size change mid-sequence, 10-bit frames
    a, b = ycc_frames(1, 64, 64, 1)[0], ycc_frames(1, 96, 64, 2)[0]
    imgs = [rh.make_ycbcr_image(*a), rh.make_ycbcr_image(*a), rh.make_ycbcr_image(*b)]
    res["size_change"] = encode_error(lambda: rs.write_sequence(os.path.join(tmp, "sz.heif"), imgs, quality=QUALITY, params=params))
    release(imgs)
    y10 = synthetic_image(30, 64, 64, 10, True)
    imgs = [rh.make_ycbcr_image(*y10, bit_depth=10) for _ in range(3)]
    res["ten_bit"] = encode_error(lambda: rs.write_sequence(os.path.join(tmp, "ten.heif"), imgs, quality=QUALITY, params=params))
    release(imgs)

    # one corrupt sample in the middle (its slice refers to a PPS id out of range): only that frame's call fails
    f5 = os.path.join(tmp, "corrupt.heif")
    srcs9 = srcs[:9]
    imgs = [rh.make_ycbcr_image(*s) for s in srcs9]
    rs.write_sequence(f5, imgs, quality=QUALITY, params=params, timescale=1000, durations=[40] * 9)
    release(imgs)
    good = rs.decode_track(f5, decoder_id="b200")
    buf = bytearray(open(f5, "rb").read())
    bad_sample = rs.raw_samples(f5)[4][0]
    at = bytes(buf).find(bad_sample)
    assert at >= 0 and bytes(buf).find(bad_sample, at + 1) < 0
    buf[at + 6], buf[at + 7] = 0xC0, 0x7F        # slice header after the 4-byte length and the 2-byte NAL header: pps id 254
    open(f5, "wb").write(bytes(buf))
    got = rs.decode_track(f5, decoder_id="b200", max_calls=9)
    # the same sample with intact headers but its slice data overwritten: it passes the per-sample header check and reaches the
    # GPU in a group with the others
    f7 = os.path.join(tmp, "corrupt_data.heif")
    imgs = [rh.make_ycbcr_image(*s) for s in srcs9]
    rs.write_sequence(f7, imgs, quality=QUALITY, params=params, timescale=1000, durations=[40] * 9)
    release(imgs)
    buf7 = bytearray(open(f7, "rb").read())
    bad7 = rs.raw_samples(f7)[4][0]
    at7 = bytes(buf7).find(bad7)
    for i in range(at7 + 4 + 48, at7 + len(bad7) - 16):
        buf7[i] = 0xFF
    open(f7, "wb").write(bytes(buf7))
    got7 = rs.decode_track(f7, decoder_id="b200", max_calls=9)
    res["corrupt_data"] = dict(status=[c[0] for c in got7], msg=[c[2] for c in got7 if c[0] == "error"],
                               others_equal=[k == 4 or e for k, e in enumerate(equal_frames(got7, [[g[1][n] for n in ("y", "cb", "cr")] for g in good]))])
    res["corrupt"] = dict(status=[c[0] for c in got],
                          others_equal=[k == 4 or e for k, e in enumerate(equal_frames(got, [[g[1][n] for n in ("y", "cb", "cr")] for g in good]))])

    # still image and grid through heif_decode_image, unchanged: this decoder plugin == the CPU plugin
    planes = [synthetic_image(10 + c, 200, 136, 8, False)[0] for c in range(3)]
    fs = os.path.join(tmp, "still.heic")
    img = rh.rgb_image(np.stack(planes, axis=2))
    rh.encode_file(fs, [img], quality=QUALITY)
    release([img])
    tiles = [rh.rgb_image(np.stack([synthetic_image(100 + 3 * k + c, 128, 128, 8, False)[0] for c in range(3)], axis=2)) for k in range(4)]
    fg = os.path.join(tmp, "grid.heic")
    rh.encode_file(fg, tiles, columns=2, rows=2, quality=QUALITY)
    release(tiles)
    res["still"] = dict(md5_cpu=md5(rh.decode_file(fs, decoder_id="b200-oracle").tobytes()), md5_gpu_decoder=md5(rh.decode_file(fs, decoder_id="b200").tobytes()))
    res["grid"] = dict(md5_cpu=md5(rh.decode_file(fg, decoder_id="b200-oracle").tobytes()), md5_gpu_decoder=md5(rh.decode_file(fg, decoder_id="b200", threads=4).tobytes()))
print("RESULT " + json.dumps(res))
