"""Child process of tests/test_gpu_encoder_speed.py (never imports torch: libheif_ref.so is loaded RTLD_GLOBAL here).
The "b200-gpu" encoder plugin's "speed" parameter inside the unmodified reference libheif: RGB, RGBA and a 3x2 grid at
speed 2, each file decoded with the FFmpeg-backed CPU plugin and with this library's decoder plugin; a file written with
speed 0 against one written without setting it; a speed-2 image sequence at sequence-batch 1 and 0 (automatic)."""
import hashlib
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
from oracle import refheif as rh  # noqa: E402
import refheif_seq as rs  # noqa: E402
from libheif_b200 import _lib  # noqa: E402
from libheif_b200.hevc_enc import synthetic_image  # noqa: E402  (pure numpy helper)

h = rs.load()
b200 = _lib.lib()
assert b200.b200_plugin_bind_libheif(None) == 0, "plugin could not resolve the libheif C API"
rh.check(h.heif_register_encoder_plugin(b200.b200_get_gpu_encoder_plugin()), "register GPU encoder plugin")
rh.check(h.heif_register_decoder_plugin(b200.b200_get_decoder_plugin()), "register decoder plugin")
rh.register_cpu_decoder()


def psnr(a, b):
    mse = np.mean((a.astype(np.float64) - b.astype(np.float64)) ** 2)
    return 99.0 if mse == 0 else float(10 * np.log10(255.0 ** 2 / mse))


def md5_file(path):
    with open(path, "rb") as f:
        return hashlib.md5(f.read()).hexdigest()


def decoded(path, chroma, want, shape):
    cpu = rh.decode_file(path, chroma=chroma, decoder_id="b200-oracle")
    gpu = rh.decode_file(path, chroma=chroma, decoder_id="b200")
    return dict(shape=list(cpu.shape), same_decoders=bool(np.array_equal(cpu, gpu)), psnr=psnr(cpu.reshape(shape), want))


res = {}
tmp = tempfile.mkdtemp()
SPEED2 = {"speed": 2}

rgb = np.stack([synthetic_image(10 + c, 200, 136, 8, False)[0] for c in range(3)], axis=2)
f = os.path.join(tmp, "rgb.heic")
rh.encode_file(f, [rh.rgb_image(rgb)], quality=70, params=SPEED2)
res["rgb"] = decoded(f, rh.CHROMA_INTERLEAVED_RGB, rgb, (136, 200, 3))

alpha = synthetic_image(20, 200, 136, 8, False)[0]
rgba = np.concatenate([rgb, alpha[:, :, None]], axis=2)
f = os.path.join(tmp, "rgba.heic")
rh.encode_file(f, [rh.rgb_image(rgba)], quality=70, params=SPEED2)
res["rgba"] = decoded(f, rh.CHROMA_INTERLEAVED_RGBA, rgba, (136, 200, 4))

srcs = [np.stack([synthetic_image(100 + 3 * k + c, 128, 128, 8, False)[0] for c in range(3)], axis=2) for k in range(6)]
f = os.path.join(tmp, "grid.heic")
rh.encode_file(f, [rh.rgb_image(t) for t in srcs], columns=3, rows=2, quality=70, params={"log2-ctb-size": 6, **SPEED2})
want = np.concatenate([np.concatenate(srcs[r * 3:(r + 1) * 3], axis=1) for r in range(2)], axis=0)
res["grid"] = decoded(f, rh.CHROMA_INTERLEAVED_RGB, want, (256, 384, 3))

# speed 0 is the default: the same file with and without setting it; speed 2 codes a different one
files = {}
for name, params in (("unset", None), ("speed0", {"speed": 0}), ("speed2", SPEED2)):
    files[name] = os.path.join(tmp, name + ".heic")
    rh.encode_file(files[name], [rh.rgb_image(rgb)], quality=70, params=params)
res["default"] = {k: md5_file(v) for k, v in files.items()}

# a speed-2 sequence, frame by frame and in automatically sized batches
frames = [tuple(synthetic_image(0x700 + k, 256, 200, 8, True)) for k in range(11)]
seq = {}
for batch in (1, 0):
    imgs = [rh.make_ycbcr_image(*x) for x in frames]
    p = os.path.join(tmp, f"seq{batch}.heif")
    rs.write_sequence(p, imgs, quality=70, params={"sequence-batch": batch, **SPEED2}, timescale=1000, durations=[40] * len(frames))
    for img in imgs:
        h.heif_image_release(img)
    seq[str(batch)] = md5_file(p)
res["sequence"] = seq
print("RESULT " + json.dumps(res))
