"""Batch-throughput probe (one GPU): K pictures (the bench grid, 16 x 16 tiles of 1024x1024) through the asynchronous fused
entry point, with ONE decoder object (D2H of picture i overlaps the kernels of picture i + 1) and with TWO decoder objects
taking the pictures alternately (own streams and device buffers each: K0 of picture i + 1 can take the SM slots the draining
K0 of picture i leaves).  Every step parses, uploads, decodes and delivers its RGB into page-locked host memory."""
import hashlib
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import torch  # noqa: E402
import libheif_b200 as lb  # noqa: E402

side = int(sys.argv[1]) if len(sys.argv) > 1 else 16
steps = int(sys.argv[2]) if len(sys.argv) > 2 else 8
os.environ.setdefault("B200_BENCH_TILE_CACHE", tempfile.mkdtemp(prefix="b200_tiles_"))
tiles = bench.make_tiles(range(side * side))
T = bench.TILE
W = H = side * T
decs = [lb.Decoder(host_threads=16), lb.Decoder(host_threads=16)]
for d in decs:
    d.set_front_end(True)
outs = [torch.empty((H, W * 3), dtype=torch.uint8, pin_memory=True).numpy() for _ in range(2)]
KEYS = ["B200_TAIL_OVERLAP"]
res = {"side": side, "steps": steps, "runs": {}}
for name, env, ndec in [("one_decoder", {}, 1), ("two_decoders", {}, 2), ("two_decoders_again", {}, 2), ("one_decoder_again", {}, 1)]:
    for k in KEYS:
        os.environ.pop(k, None)
    os.environ.update(env)
    for w in range(2 * ndec):                      # warm-up: buffers of every decoder allocated
        decs[w % ndec].decode_grid_to_rgb_host_async(tiles, side, side, lb.CHROMA_INTERLEAVED_RGB, out=outs[w % ndec])
    for d in decs[:ndec]:
        d.wait()
    for o in outs:
        o[:] = 0
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(steps):
        decs[i % ndec].decode_grid_to_rgb_host_async(tiles, side, side, lb.CHROMA_INTERLEAVED_RGB, out=outs[i % ndec])
    for d in decs[:ndec]:
        d.wait()
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3 / steps
    md5 = [hashlib.md5(o.tobytes()).hexdigest() for o in outs[:ndec]]
    res["runs"][name] = {"ms_per_step": ms, "mp_s": W * H / ms / 1e3, "md5": md5}
    print(name, res["runs"][name], file=sys.stderr, flush=True)
res["all_md5_equal"] = len({m for r in res["runs"].values() for m in r["md5"]}) == 1
print(json.dumps(res))
