"""K0-tail overlap probe (one GPU): the bench workload (16 x 16 tiles of 1024x1024) under combinations of
B200_TAIL_OVERLAP (K1 queued behind a full-occupancy K0, filling the SM slots K0's draining wavefronts leave) and
B200_CHUNK_TILES (band count of the synchronous fused call).  Prints one JSON object: per configuration the resident step
(CUDA events), the end-to-end step (one C-ABI call, host bitstreams -> page-locked host RGB), the kernel stats of the last
step and the md5 of the RGB result (must be the same everywhere)."""
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
steps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
os.environ.setdefault("B200_BENCH_TILE_CACHE", tempfile.mkdtemp(prefix="b200_tiles_"))
tiles = bench.make_tiles(range(side * side))
T = bench.TILE
W = H = side * T
dec = lb.Decoder(host_threads=16)
dec.set_front_end(True)
dev = torch.device("cuda", 0)
band = torch.empty((H, W * 3), dtype=torch.uint8, device=dev)
host_t = torch.empty((H, W * 3), dtype=torch.uint8, pin_memory=True)
host_out = host_t.numpy()
stream = torch.cuda.current_stream()
Q = str(side * side // 4)
configs = [("default", {}), ("tail1_2bands", {"B200_TAIL_OVERLAP": "1"}), ("tail_1band", {"B200_TAIL_OVERLAP": "1", "B200_CHUNKS": "0"}),
           ("notail_4bands", {"B200_CHUNK_TILES": Q}), ("default_again", {})]
KEYS = ["B200_TAIL_OVERLAP", "B200_CHUNK_TILES", "B200_CHUNKS"]
out = {"side": side, "steps": steps, "configs": {}}
for name, env in configs:
    for k in KEYS:
        os.environ.pop(k, None)
    os.environ.update(env)
    r = {}
    for _ in range(3):
        dec.decode_grid_to_rgb_host(tiles, side, side, lb.CHROMA_INTERLEAVED_RGB, out=host_out)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        dec.decode_grid_to_rgb_host(tiles, side, side, lb.CHROMA_INTERLEAVED_RGB, out=host_out)
    torch.cuda.synchronize()
    r["e2e_ms"] = (time.perf_counter() - t0) * 1e3 / steps
    st = dec.stats()
    r["e2e_stats"] = {"entropy_ms": st.entropy_ms, "recon_ms": st.recon_ms, "front_end": st.front_end, "bands": st.bands}
    r["e2e_md5"] = hashlib.md5(host_out.tobytes()).hexdigest()
    # resident leg: one launch per kernel (no bands), compressed tiles already in HBM
    os.environ["B200_CHUNKS"] = "0"
    dec.decode_grid(tiles, cols=side, rows=side)
    for _ in range(3):
        dec.rerun_device(stream)
        dec.to_rgb_device(lb.CHROMA_INTERLEAVED_RGB, out=band, stream=stream)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(stream)
    for _ in range(steps):
        dec.rerun_device(stream)
        dec.to_rgb_device(lb.CHROMA_INTERLEAVED_RGB, out=band, stream=stream)
    e1.record(stream)
    torch.cuda.synchronize()
    r["resident_ms"] = e0.elapsed_time(e1) / steps
    st = dec.stats()
    r["resident_stats"] = {"entropy_ms": st.entropy_ms, "recon_ms": st.recon_ms, "deblock_ms": st.deblock_ms, "sao_ms": st.sao_ms, "front_end": st.front_end}
    r["resident_md5"] = hashlib.md5(band.cpu().numpy().tobytes()).hexdigest()
    out["configs"][name] = r
    print(name, json.dumps(r), file=sys.stderr, flush=True)
md5s = {r["e2e_md5"] for r in out["configs"].values()} | {r["resident_md5"] for r in out["configs"].values()}
out["all_md5_equal"] = len(md5s) == 1
print(json.dumps(out))
