"""One-call RGB -> HEIC grid encoder (GpuEncoder.encode_rgb_grid, b200_gpu_encode_rgb_grid_*) on a 16384^2 RGB24 picture cut
into 1024^2 tiles at QP 27, CTB 32.  The picture is assembled from 256 synthetic_image blocks of 1024^2 (seeds 0xB200 + 3k + c
for the R, G, B planes of block k), so its tiles are those of scripts/gpu_encode_bench.py's workload in RGB.

Host form (numpy RGB -> access units) and device form (CUDA tensor -> access units), alternating, median of --calls calls
each after one warm-up of each; the split into colour / upload (CUDA events) and E1 / E2 (CUDA events) / framing (host
clock) of the median call.  For comparison, heif_context_encode_grid of the unmodified reference libheif with the
"b200-gpu" plugin (one encode_image per tile) on a --ref-grid x --ref-grid sub-grid in a child process: its per-tile time,
not extrapolated.  Prints one JSON line with the card's name, power limit and maximum SM clock.

    python scripts/grid_encode_bench.py [--size 16384] [--tile 1024] [--calls 3] [--ref-grid 4] [--out DIR]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from libheif_b200.hevc_enc import synthetic_image  # noqa: E402

NCLX = dict(vui_present=1, colour_description_present=1, colour_primaries=1, transfer_characteristics=13, matrix_coefficients=6, full_range=1)


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def rgb_picture(size, block):
    n = size // block
    out = np.empty((size, size, 3), np.uint8)

    def fill(k):
        r, c = divmod(k, n)
        for ch in range(3):
            out[r * block:(r + 1) * block, c * block:(c + 1) * block, ch] = synthetic_image(0xB200 + 3 * k + ch, block, block, 8, False)[0]

    with ThreadPoolExecutor(os.cpu_count()) as ex:
        list(ex.map(fill, range(n * n)))
    return out


def child(npy, tile, qp):
    """heif_context_encode_grid of the reference libheif with the "b200-gpu" plugin (never imports torch)."""
    from libheif_b200 import _lib
    from oracle import refheif as rh
    h = rh.load()
    b200 = _lib.lib()
    assert b200.b200_plugin_bind_libheif(None) == 0
    rh.check(h.heif_register_encoder_plugin(b200.b200_get_gpu_encoder_plugin()), "register GPU encoder plugin")
    px = np.load(npy)
    g = px.shape[0] // tile
    quality = next(q for q in range(101) if 51 - (q * 45 + 50) // 100 == qp)   # the plugin's quality -> QP mapping
    images = []
    for r in range(g):
        for c in range(g):
            img = C.c_void_p()
            rh.check(h.heif_image_create(tile, tile, rh.COLORSPACE_RGB, rh.CHROMA_INTERLEAVED_RGB, C.byref(img)))
            rh.check(h.heif_image_add_plane(img, rh.CHANNEL_INTERLEAVED, tile, tile, 8))
            st = C.c_int()
            p = h.heif_image_get_plane(img, rh.CHANNEL_INTERLEAVED, C.byref(st))
            np.ctypeslib.as_array(p, shape=(tile, st.value))[:, :tile * 3] = px[r * tile:(r + 1) * tile, c * tile:(c + 1) * tile].reshape(tile, -1)
            images.append(img)
    path = os.path.join(tempfile.mkdtemp(), "grid.heic")
    rh.encode_file(path, images[:1], quality=quality, params={"log2-ctb-size": 5})                     # warm-up: device, module load
    t = time.perf_counter()
    rh.encode_file(path, images, columns=g, rows=g, quality=quality, params={"log2-ctb-size": 5})
    ms = (time.perf_counter() - t) * 1e3
    print("RESULT " + json.dumps(dict(tiles=g * g, ms=ms, quality=quality, bytes=os.path.getsize(path))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size", type=int, default=16384)
    ap.add_argument("--tile", type=int, default=1024)
    ap.add_argument("--qp", type=int, default=27)
    ap.add_argument("--calls", type=int, default=3)
    ap.add_argument("--ref-grid", type=int, default=4, help="sub-grid side for the libheif per-tile comparison (0 = skip)")
    ap.add_argument("--out", default=None)
    ap.add_argument("--child", nargs=3, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.child:
        child(a.child[0], int(a.child[1]), int(a.child[2]))
        return 0
    import torch
    from libheif_b200.hevc_enc import GpuEncoder
    assert torch.cuda.is_available(), "needs a CUDA device"
    t = time.time()
    px = rgb_picture(a.size, a.tile)
    gen_s = time.time() - t
    dpx = torch.from_numpy(px).cuda()
    torch.cuda.synchronize()
    enc = GpuEncoder()
    prm = dict(qp=a.qp, log2_ctb_size=5, **NCLX)
    runs = {"host": [], "device": []}
    outs = {}
    for it in range(a.calls + 1):
        for form, src in (("host", px), ("device", dpx)):
            t = time.perf_counter()
            r = enc.encode_rgb_grid(src, a.tile, a.tile, **prm)
            wall = (time.perf_counter() - t) * 1e3
            st = enc.stats()
            if it > 0:                                   # the first call of each form is the warm-up
                runs[form].append(dict(wall_ms=wall, colour_ms=r["colour_ms"], upload_ms=r["upload_ms"], e1_ms=st.analyse_ms,
                                       e2_ms=st.entropy_ms, framing_ms=st.framing_ms))
            outs[form] = r["tiles"]
    px_count = a.size * a.size
    res = dict(card=card(), host_cores=os.cpu_count(), size=a.size, tile=a.tile, tiles=len(outs["host"]), qp=a.qp, ctb=32, calls=a.calls,
               source_gen_s=round(gen_s, 1), host_equals_device=outs["host"] == outs["device"],
               bytes=sum(map(len, outs["host"])), bits_per_px=round(8 * sum(map(len, outs["host"])) / px_count, 4))
    for form, rs in runs.items():
        med = sorted(rs, key=lambda x: x["wall_ms"])[len(rs) // 2]
        res[form] = dict(median_ms=round(med["wall_ms"], 1), mp_per_s=round(px_count / 1e6 / (med["wall_ms"] / 1e3), 1),
                         split_of_median_call={k: round(v, 2) for k, v in med.items() if k != "wall_ms"},
                         wall_ms_all=[round(x["wall_ms"], 1) for x in rs])
    res["libheif_encode_grid"] = "not measured"
    if a.ref_grid:
        from oracle import bindings as ob
        if os.path.exists(os.path.join(ob.REF, "libheif_ref.so")):
            g = a.ref_grid
            npy = os.path.join(tempfile.mkdtemp(), "sub.npy")
            np.save(npy, np.ascontiguousarray(px[:g * a.tile, :g * a.tile]))
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", npy, str(a.tile), str(a.qp)],
                               stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=1800)
            lines = [ln for ln in r.stdout.splitlines() if ln.startswith("RESULT ")]
            if r.returncode == 0 and lines:
                c = json.loads(lines[-1][7:])
                res["libheif_encode_grid"] = dict(tiles=c["tiles"], ms=round(c["ms"], 1), per_tile_ms=round(c["ms"] / c["tiles"], 1),
                                                  quality=c["quality"], bytes=c["bytes"])
            else:
                res["libheif_encode_grid"] = "failed: " + r.stderr[-500:]
    enc.close()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "grid_encode_bench.json"), "w") as f:
            f.write(line + "\n")
    return 0 if res["host_equals_device"] else 1


if __name__ == "__main__":
    sys.exit(main())
