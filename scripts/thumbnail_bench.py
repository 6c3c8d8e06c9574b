"""Scaled decode on the bench grid (16384 x 16384 HEIC grid, 256 x 1024x1024 tiles, QP 27, CTB 32, 8-bit 4:2:0 -> RGB24):
the routes from the bitstream to an RGB picture of a requested size in host memory, run alternately in one process.

  full         b200_decode_grid_to_rgb_host at full size (what a caller scales on the host afterwards)
  thumb512     b200_decode_grid_to_rgb_scaled_host to thumbnail_size(16384, 16384, 512)
  scaled4096   b200_decode_grid_to_rgb_scaled_host to 4096 x 4096
  two_step     b200_decoder_decode_grid + full-size b200_color_convert_device + b200_scale_nearest_device to the thumb512
               size + D2H of the scaled picture

Per route: median and range of the call time (host clock around the synchronous call) and of the K6 time (CUDA events
around the colour stage of the route on the decoded canvas: the scaled or full-size conversion; two_step adds the scaler),
and the bytes copied device -> host.  Destinations are page-locked.  Checks that the scaled bytes equal the two-step
route's.  Prints the card name and power limit with each round, one JSON line at the end.

usage: python scripts/thumbnail_bench.py [--side 16] [--rounds 5] [--warmup 1]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import numpy as np  # noqa: E402
import torch  # noqa: E402
import libheif_b200 as lb  # noqa: E402

RGB = lb.CHROMA_INTERLEAVED_RGB


def card():
    """(name, power limit) of the current GPU"""
    r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    return torch.cuda.get_device_name(), r.stdout.strip() if r.returncode == 0 else "unknown"


def events_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--side", type=int, default=16, help="grid of side x side 1024x1024 tiles (16: the bench grid)")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("thumbnail_bench needs a CUDA device")
    os.environ.setdefault("B200_BENCH_TILE_CACHE", tempfile.mkdtemp(prefix="b200_tiles_"))
    side = args.side
    tiles = bench.make_tiles(range(side * side))
    W = H = side * bench.TILE
    tw, th = lb.thumbnail_size(W, H, 512)
    sizes = {"full": (W, H), "thumb512": (tw, th), "scaled4096": (4096, 4096), "two_step": (tw, th)}
    dec = lb.Decoder(host_threads=16)
    pinned = {k: torch.empty((h, w * 3), dtype=torch.uint8, pin_memory=True) for k, (w, h) in sizes.items()}
    outs = {k: t.numpy() for k, t in pinned.items()}

    def run(name):
        w, h = sizes[name]
        out = outs[name]
        t0 = time.perf_counter()
        if name == "two_step":
            dec.decode_grid(tiles, side, side)
            full = dec.to_rgb_device(RGB)
            small = lb.compose.scale_nearest_plane(full, w, h, (W, H), (w, h), 3)
            pinned[name].copy_(small)                          # page-locked destination: one D2H, synchronous
            torch.cuda.synchronize()
        else:
            dec.decode_grid_to_rgb_host(tiles, side, side, RGB, out=out, scale=None if name == "full" else (w, h))
        call_ms = (time.perf_counter() - t0) * 1e3
        # the colour stage of this route again, on the canvas the call left behind
        if name == "two_step":
            buf = {}
            k6_ms = events_ms(lambda: buf.update(f=dec.to_rgb_device(RGB)))
            k6_ms += events_ms(lambda: lb.compose.scale_nearest_plane(buf["f"], w, h, (W, H), (w, h), 3))
        else:
            k6_ms = events_ms(lambda: dec.to_rgb_device(RGB, scale=None if name == "full" else (w, h)))
        return call_ms, k6_ms

    names = list(sizes)
    for _ in range(args.warmup):
        for n in names:
            run(n)
    times = {n: {"call": [], "k6": []} for n in names}
    for r in range(args.rounds):
        name_, plim = card()
        for n in names:
            c, k = run(n)
            times[n]["call"].append(c)
            times[n]["k6"].append(k)
        print(f"round {r}: {name_}, power limit {plim}: " + ", ".join(f"{n} {times[n]['call'][-1]:.1f} ms" for n in names),
              file=sys.stderr, flush=True)
    same = bool(np.array_equal(outs["thumb512"], outs["two_step"]))
    name_, plim = card()
    res = {"card": name_, "power_limit": plim, "grid": f"{W}x{H}, {side * side} x 1024x1024 tiles, QP {bench.QP}, CTB 32, 8-bit 4:2:0 -> RGB24",
           "rounds": args.rounds, "routes": {}}
    for n in names:
        w, h = sizes[n]
        c, k = sorted(times[n]["call"]), sorted(times[n]["k6"])
        res["routes"][n] = {"size": [w, h], "call_ms_median": c[len(c) // 2], "call_ms_range": [c[0], c[-1]],
                            "k6_ms_median": k[len(k) // 2], "k6_ms_range": [k[0], k[-1]], "d2h_bytes": w * h * 3}
        print(f"{n:11s} {w}x{h}: call {c[len(c) // 2]:.2f} ms [{c[0]:.2f}, {c[-1]:.2f}], K6 {k[len(k) // 2]:.3f} ms [{k[0]:.3f}, {k[-1]:.3f}], "
              f"D2H {w * h * 3} B", file=sys.stderr)
    res["scaled_equals_two_step"] = same
    print(f"scaled == two-step: {str(same).lower()}", file=sys.stderr)
    print(json.dumps(res))
    dec.close()
    return 0 if same else 1


if __name__ == "__main__":
    sys.exit(main())
