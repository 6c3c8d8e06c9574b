"""Child process of tests/test_hevc_gpu_encoder.py (never imports torch: libheif_ref.so is loaded RTLD_GLOBAL here).
The "b200-gpu" encoder plugin inside the unmodified reference libheif: RGB and RGBA through heif_context_encode_image (the
reference converts the colour, alpha goes through the same plugin as a monochrome picture), a 3x2 grid through
heif_context_encode_grid; each file decoded by the reference with the FFmpeg-backed CPU plugin and with this library's
decoder plugin."""
import ctypes as C
import hashlib
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
from oracle import refheif as rh  # noqa: E402
from libheif_b200 import _lib  # noqa: E402
from libheif_b200.hevc_enc import synthetic_image  # noqa: E402  (pure numpy helper)

h = rh.load()
b200 = _lib.lib()
assert b200.b200_plugin_bind_libheif(None) == 0, "plugin could not resolve the libheif C API"
rh.check(h.heif_register_encoder_plugin(b200.b200_get_gpu_encoder_plugin()), "register GPU encoder plugin")
rh.check(h.heif_register_decoder_plugin(b200.b200_get_decoder_plugin()), "register decoder plugin")
rh.register_cpu_decoder()


def has_alpha(path):
    ctx = h.heif_context_alloc()
    rh.check(h.heif_context_read_from_file(ctx, path.encode(), None), "read")
    hd = C.c_void_p()
    rh.check(h.heif_context_get_primary_image_handle(ctx, C.byref(hd)))
    a = bool(h.heif_image_handle_has_alpha_channel(hd))
    h.heif_image_handle_release(hd)
    h.heif_context_free(ctx)
    return a


def psnr(a, b):
    mse = np.mean((a.astype(np.float64) - b.astype(np.float64)) ** 2)
    return 99.0 if mse == 0 else float(10 * np.log10(255.0 ** 2 / mse))


def decoded(path, chroma):
    cpu = rh.decode_file(path, chroma=chroma, decoder_id="b200-oracle")
    gpu = rh.decode_file(path, chroma=chroma, decoder_id="b200")
    return cpu, dict(shape=list(cpu.shape), md5_cpu=hashlib.md5(cpu.tobytes()).hexdigest(), md5_gpu_decoder=hashlib.md5(gpu.tobytes()).hexdigest(),
                     has_alpha=has_alpha(path))


res = {}
tmp = tempfile.mkdtemp()
ctx = h.heif_context_alloc()
enc = C.c_void_p()
rh.check(h.heif_context_get_encoder_for_format(ctx, rh.COMPRESSION_HEVC, C.byref(enc)), "get_encoder_for_format")
res["encoder_ids"] = [h.heif_encoder_get_name(enc).decode()]
h.heif_encoder_release(enc)
h.heif_context_free(ctx)
res["encoder_ids"] = ["b200-gpu" if "GPU" in res["encoder_ids"][0] else res["encoder_ids"][0]]

# RGB 200x136 (odd chroma size: conformance window) through heif_context_encode_image
planes = [synthetic_image(10 + c, 200, 136, 8, False)[0] for c in range(3)]
rgb = np.stack(planes, axis=2)
f = os.path.join(tmp, "rgb.heic")
rh.encode_file(f, [rh.rgb_image(rgb)], quality=70)
cpu, res["rgb"] = decoded(f, rh.CHROMA_INTERLEAVED_RGB)
res["rgb"]["psnr"] = psnr(cpu.reshape(136, 200, 3), rgb)

# RGBA: the alpha plane is a second picture through the same plugin, as 4:0:0
alpha = synthetic_image(20, 200, 136, 8, False)[0]
rgba = np.concatenate([rgb, alpha[:, :, None]], axis=2)
f = os.path.join(tmp, "rgba.heic")
rh.encode_file(f, [rh.rgb_image(rgba)], quality=70)
cpu, res["rgba"] = decoded(f, rh.CHROMA_INTERLEAVED_RGBA)
cpu = cpu.reshape(136, 200, 4)
res["rgba"]["psnr"] = psnr(cpu[:, :, :3], rgb)
res["rgba"]["alpha_psnr"] = psnr(cpu[:, :, 3], alpha)

# 3x2 grid of 128x128 RGB tiles through heif_context_encode_grid (one encoder instance for every tile, grid.cc:886-906)
tiles, srcs = [], []
for k in range(6):
    t = np.stack([synthetic_image(100 + 3 * k + c, 128, 128, 8, False)[0] for c in range(3)], axis=2)
    srcs.append(t)
    tiles.append(rh.rgb_image(t))
f = os.path.join(tmp, "grid.heic")
rh.encode_file(f, tiles, columns=3, rows=2, quality=70, params={"log2-ctb-size": 6})
cpu, res["grid"] = decoded(f, rh.CHROMA_INTERLEAVED_RGB)
want = np.concatenate([np.concatenate(srcs[r * 3:(r + 1) * 3], axis=1) for r in range(2)], axis=0)
res["grid"]["psnr"] = psnr(cpu.reshape(256, 384, 3), want)

# 10-bit input: heif_suberror_Unsupported_bit_depth
y10, cb10, cr10 = synthetic_image(30, 64, 64, 10, True)
try:
    rh.encode_file(os.path.join(tmp, "ten.heic"), [rh.make_ycbcr_image(y10, cb10, cr10, 10)], quality=70)
    res["bit_depth_refused"] = False
except RuntimeError as e:
    res["bit_depth_refused"] = "/4000" in str(e)
    res["bit_depth_error"] = str(e)[:200]
print("RESULT " + json.dumps(res))
