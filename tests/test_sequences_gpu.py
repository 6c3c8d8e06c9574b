"""Image sequences (heif_track_encode_sequence_image / heif_track_decode_next_image) through the unmodified reference libheif
with this library's plugins: all-intra sequence encoding in the "b200" and "b200-gpu" encoder tables, the GPU table's batched
frames, and the decoder plugin's read-ahead.  The reference runs in a child process (tests/seq_plugin_child.py, see
oracle/refheif.py for why)."""
import json
import os
import subprocess
import sys

import pytest

from oracle import bindings as ob

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
have_ref = os.path.exists(os.path.join(ob.REF, "libheif_ref.so")) and os.path.exists(os.path.join(ob.REF, "liboracle_plugin.so")) and ob.avcodec_dir()
needs_ref = pytest.mark.skipif(not have_ref, reason="oracle/_ref reference build not present")


def child(*args, env=None):
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "seq_plugin_child.py"), *args], stdout=subprocess.PIPE, stderr=subprocess.PIPE,
                       text=True, timeout=900, env=env)
    assert r.returncode == 0, r.stderr[-3000:]
    return json.loads([l for l in r.stdout.splitlines() if l.startswith("RESULT ")][-1][7:])


def test_encoder_tables_declare_sequence_members():
    """Both encoder tables are v4 tables with the sequence members set and does_indicate_keyframes = 1; the GPU table lists
    the "sequence-batch" parameter (default 0 = automatic)."""
    import ctypes as C
    from libheif_b200 import _lib
    lib = _lib.lib()

    class Integer(C.Structure):
        _fields_ = [("default_value", C.c_int), ("have_minmax", C.c_uint8), ("minimum", C.c_int), ("maximum", C.c_int),
                    ("valid_values", C.c_void_p), ("num_valid_values", C.c_int)]

    class Param(C.Structure):         # b200h_encoder_parameter == heif_encoder_parameter (heif_plugin.h)
        _fields_ = [("version", C.c_int), ("name", C.c_char_p), ("type", C.c_int), ("integer", Integer), ("has_default", C.c_int)]

    names = {}
    for getter in ("b200_get_encoder_plugin", "b200_get_gpu_encoder_plugin"):
        p = getattr(lib, getter)()
        words = (C.c_void_p * 33).from_address(p)       # b200h_encoder_plugin as pointer-sized words (x86-64 layout)
        assert C.c_int.from_address(p).value == 4
        # the v4 members after minimum_required_libheif_version: start / frame / end / get_compressed_data2, does_indicate_keyframes
        assert all(words[i] for i in range(28, 32)), getter
        assert C.c_int.from_address(p + 32 * C.sizeof(C.c_void_p)).value == 1, getter
        lst = C.CFUNCTYPE(C.POINTER(C.POINTER(Param)), C.c_void_p)(words[15])(None)
        names[getter] = []
        for i in range(16):
            if not lst[i]:
                break
            q = lst[i].contents
            names[getter].append((q.name.decode(), q.has_default, q.integer.default_value, q.integer.minimum, q.integer.maximum))
    assert ("sequence-batch", 1, 0, 0, 4096) in names["b200_get_gpu_encoder_plugin"], names
    assert "sequence-batch" not in [n[0] for n in names["b200_get_encoder_plugin"]]


@needs_ref
def test_host_encoder_sequence_through_reference_libheif():
    """The "b200" table writes a 9-frame RGB sequence (200 x 136): 9 samples, all sync samples, the durations and timescale
    that were set, each sample decodable at the right size.  A 9-frame YCbCr sequence: the slice NAL of every sample is the
    one b200_hevc_encode_intra codes for that picture as a still, and FFmpeg decodes every sample to the same picture as the
    still.  A frame whose size differs from the first frame's is refused."""
    res = child("cpu")
    rgb = res["rgb"]
    assert rgb["count"] == 9
    assert rgb["sync"] == [None]                    # no 'stss': every sample is a sync sample
    assert rgb["durations"] == [1001 + k for k in range(9)]
    assert rgb["tracks"][0]["timescale"] == 30000 and rgb["tracks"][0]["handler"] == "pict"
    assert (rgb["tracks"][0]["width"], rgb["tracks"][0]["height"]) == (200, 136)
    assert rgb["ffmpeg_sizes"] == [[136, 200]] * 9
    ycc = res["ycc"]
    assert ycc["count"] == 9 and ycc["sync"] == [None] and ycc["durations"] == [40] * 9
    assert all(ycc["slices_equal_still"]), ycc["slices_equal_still"]
    assert all(ycc["frames_equal_ffmpeg_still"]), ycc["frames_equal_ffmpeg_still"]
    assert res["size_change"] is not None and "same format" in res["size_change"]["msg"], res["size_change"]


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("batch", [1, 4, 0])
def test_gpu_encoder_sequences_and_decoder_read_ahead(cuda, batch):
    """The "b200-gpu" table at sequence-batch 1, 4 and automatic (0), and the decoder plugin's read-ahead:
    - a 37-frame sequence has 37 sync samples, and the slice NAL of each is GpuEncoder.encode of that frame alone;
    - the decoder plugin, driven as libheif drives it for a track, hands back FFmpeg's decode of every sample, in push order
      with its user_data; heif_track_decode_next_image with it gives every frame in order, close to its source, from batches
      of more than one picture, and the first frame equal to the oracle plugin's (which decodes each push on its own, so it
      cannot follow a track past its first sample); a track repeated twice gives 74 frames, the second pass equal to the first;
    - RGBA: an alpha auxiliary track, reported by heif_track_has_alpha_channel; both tracks' samples decode as FFmpeg decodes them;
    - a monochrome sequence round-trips;
    - a size change mid-sequence and 10-bit frames (heif_suberror_Unsupported_bit_depth) are refused;
    - one corrupt sample fails only its own heif_track_decode_next_image, both when its slice header is broken (refused by the
      per-sample header check) and when only its slice data is (it reaches the GPU in a group with the others, the group
      fails and is decoded again one picture at a time);
    - an encoder reused after a refused frame writes the next sequence without frames of the abandoned one;
    - a still image and a grid still decode as the CPU plugin decodes them."""
    res = child("gpu", str(batch))
    s = res["seq37"]
    assert s["count"] == 37 and s["sync"] == [None] and s["durations"] == [40 + 3 * (k % 7) for k in range(37)]
    assert all(s["slices_equal_alone"]), s["slices_equal_alone"]
    if batch:
        assert s["encoder_calls"] == -(-37 // batch) and s["encoder_max_batch"] == min(batch, 37), s
    else:
        assert 1 <= s["encoder_calls"] < 37 and s["encoder_max_batch"] > 1, s
    assert s["ffmpeg_frames"] == 37 and s["decoded_gpu"] == ["ok"] * 37
    assert all(s["plugin_equal_ffmpeg"]) and s["plugin_users"] == list(range(37)), s
    assert s["first_equal_oracle_plugin"]
    assert min(s["psnr_y_ffmpeg"]) > 30, s["psnr_y_ffmpeg"]
    assert min(s["psnr_y"]) > 25, s["psnr_y"]           # after libheif's colour handling; frame k against source k: the order
    assert s["queue_pictures"] == 37 and s["queue_max_batch"] > 1 and s["queue_batches"] < 37, s
    r = res["repeat"]
    assert r["decoded"] == ["ok"] * 74 and r["md5_first"] == r["md5_second"] == r["md5_once"]
    a = res["rgba"]
    assert a["count"] == 9 and len(a["tracks"]) == 2 and a["tracks"][0]["has_alpha"], a["tracks"]
    assert a["decoded_gpu"] == ["ok"] * 9 and all(a["plugin_equal_ffmpeg"]) and all(a["alpha_plugin_equal_ffmpeg"]), a
    assert a["first_equal_oracle_plugin"]
    assert min(a["alpha_psnr"]) > 28 and min(a["rgb_psnr"]) > 28, (a["alpha_psnr"], a["rgb_psnr"])
    m = res["mono"]
    assert m["count"] == 11 and m["decoded_gpu"] == ["ok"] * 11 and not m["has_chroma"] and all(m["plugin_equal_ffmpeg"]), m
    assert min(m["psnr_y"]) > 25
    assert res["size_change"] is not None and "same format" in res["size_change"]["msg"], res["size_change"]
    assert res["ten_bit"] is not None and res["ten_bit"]["sub"] == 4000, res["ten_bit"]
    c = res["corrupt"]
    assert c["status"] == ["ok"] * 4 + ["error"] + ["ok"] * 4, c
    assert all(c["others_equal"]), c
    c = res["corrupt_data"]
    assert c["status"] == ["ok"] * 4 + ["error"] + ["ok"] * 4, c
    assert all(c["others_equal"]), c
    u = res["reuse"]
    assert u["refused"] and u["count"] == 3 and u["durations"] == [10, 20, 30] and all(u["slices_equal_alone"]), u
    assert res["still"]["md5_cpu"] == res["still"]["md5_gpu_decoder"]
    assert res["grid"]["md5_cpu"] == res["grid"]["md5_gpu_decoder"]


@pytest.mark.gpu
@needs_ref
def test_gpu_sequence_files_do_not_depend_on_the_batch(cuda):
    """The files the "b200-gpu" table writes at sequence-batch 1, 4 and automatic are byte-identical, and so are the decoded
    frames; with the read-ahead at 1 (B200_SEQ_READAHEAD=1) the decoder returns the same frames, one batch per picture."""
    md5s, frames = set(), set()
    for b in (1, 4, 0):
        s = child("gpu", str(b), "seq37")["seq37"]
        md5s.add(s["file_md5"])
        frames.add(s["md5_gpu_decoder"])
    env = dict(os.environ, B200_SEQ_READAHEAD="1")
    s = child("gpu", "0", "seq37", env=env)["seq37"]
    assert len(md5s) == 1, md5s
    assert frames == {s["md5_gpu_decoder"]}, (frames, s["md5_gpu_decoder"])
    assert s["queue_max_batch"] == 1 and s["queue_batches"] == 37, s


@pytest.mark.gpu
@needs_ref
def test_read_ahead_respects_max_total_memory(cuda):
    """A track that decodes with the read-ahead at 1 (one decoded picture alive at a time) also decodes at the default when the
    context's max_total_memory is low (8 MiB, 37 frames of 512 x 512): the read-ahead group is bounded by its decoded size,
    1/8 of that limit, so it holds 2 pictures here instead of 32."""
    one = child("memlimit", env=dict(os.environ, B200_SEQ_READAHEAD="1"))["memlimit"]
    env = dict(os.environ)
    env.pop("B200_SEQ_READAHEAD", None)
    dflt = child("memlimit", env=env)["memlimit"]
    assert one["status"] == ["ok"] * 37, one
    assert dflt["status"] == ["ok"] * 37, dflt
    assert dflt["md5"] == one["md5"]
    assert one["max_batch"] == 1 and dflt["max_batch"] == 2, (one, dflt)
