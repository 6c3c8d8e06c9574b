"""K0 trace probe: when each decoder warp of the entropy kernel is busy.

Builds the B200_ENTROPY_TRACE variant of the library (lane 0 of a decoder warp records globaltimer when it pops a
sub-stream and when it finishes it, and the SM it runs on), decodes the bench grid with it (side x side tiles of
1024x1024, device front-end, one launch per kernel: B200_CHUNKS=0 B200_TAIL_OVERLAP=0, as bench.py's kernel leg) and
prints one JSON line: the number of sub-streams in flight over the kernel's span (in --bins equal slices), the share of
the span with fewer than 90 % of the peak number of decoders busy (ramp-up and drain), and the mean time per CTB of a
busy decoder.  Card name and power limit are part of the line.

  python scripts/k0_trace_probe.py --build-only                  # compile the variant (here)
  python scripts/k0_trace_probe.py [--lib PATH] [--out DIR]      # on the GPU: measure
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build_variant(src):
    import importlib.util
    spec = importlib.util.spec_from_file_location("_trace_build", os.path.join(src, "build.py"))
    b = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(b)
    out = os.path.join(tempfile.gettempdir(), "b200_k0_trace", "libb200heif_trace.so")
    os.makedirs(os.path.dirname(out), exist_ok=True)
    return b.build(extra_flags=["-DB200_ENTROPY_TRACE"], out=out, tag="_trace")


def child(side, reps):
    """Runs with B200_LIB = the trace variant; prints the trace of the last K0 launch as JSON."""
    os.environ["B200_CHUNKS"] = "0"
    os.environ["B200_TAIL_OVERLAP"] = "0"
    sys.path.insert(0, ROOT)
    import bench
    import torch
    import libheif_b200 as lb
    tiles = bench.make_tiles(range(side * side))
    dec = lb.Decoder(host_threads=16)
    dec.set_front_end(True)
    dec.decode_grid(tiles, cols=side, rows=side)
    for _ in range(reps):
        dec.rerun_device(torch.cuda.current_stream())
        torch.cuda.synchronize()
    k0_ms = dec.stats().entropy_ms
    n = side * side * (1024 // 32)                 # one sub-stream per CTB row of every tile (CTB 32, WPP)
    buf = (C.c_ulonglong * (3 * n))()
    lb._lib.check(lb._lib.lib().b200_debug_entropy_trace(buf, n))
    print(json.dumps({"k0_ms": k0_ms, "ctbs_per_sub": 1024 // 32, "trace": list(buf)}))


def summarise(res, nbins):
    tr = res["trace"]
    recs = [(tr[3 * i], tr[3 * i + 1], tr[3 * i + 2]) for i in range(len(tr) // 3) if tr[3 * i] and tr[3 * i + 1] >= tr[3 * i]]
    t0 = min(r[0] for r in recs); t1 = max(r[1] for r in recs); span = t1 - t0
    ev = sorted([(r[0], 1) for r in recs] + [(r[1], -1) for r in recs])
    # step function of the number of busy decoders; time-weighted per slice
    active, last, peak = 0, t0, 0
    segs = []
    for t, d in ev:
        if t > last:
            segs.append((last, t, active))
        active += d; last = t; peak = max(peak, active)
    slices = [0.0] * nbins
    below = 0
    for a, b, n in segs:
        if n < 0.9 * peak:
            below += b - a
        for k in range(nbins):
            lo, hi = t0 + span * k / nbins, t0 + span * (k + 1) / nbins
            ov = min(b, hi) - max(a, lo)
            if ov > 0:
                slices[k] += n * ov
    slices = [round(s / (span / nbins), 1) for s in slices]
    busy = [(r[1] - r[0]) / res["ctbs_per_sub"] for r in recs]
    return {"k0_ms": res["k0_ms"], "traced_span_ms": span / 1e6, "substreams": len(recs), "sms": len({r[2] for r in recs}),
            "peak_busy_decoders": peak, "busy_decoders_per_slice": slices,
            "share_of_span_below_90pct_of_peak": below / span, "mean_ctb_us_per_busy_decoder": 1e-3 * sum(busy) / len(busy),
            "mean_substream_ms": 1e-6 * sum(r[1] - r[0] for r in recs) / len(recs)}


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except Exception as e:  # noqa: BLE001 - reported, not fatal
        return f"unavailable: {e}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--src", default=os.path.join(ROOT, "libheif_b200"), help="libheif_b200 package directory whose sources are built")
    ap.add_argument("--lib", default=None, help="an already built B200_ENTROPY_TRACE library (skips the build)")
    ap.add_argument("--label", default="")
    ap.add_argument("--side", type=int, default=16)
    ap.add_argument("--reps", type=int, default=3, help="K0 runs; the trace is the last one's")
    ap.add_argument("--bins", type=int, default=20)
    ap.add_argument("--build-only", action="store_true")
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--out", default=None, help="also append the JSON line to DIR/k0_trace.jsonl")
    args = ap.parse_args()
    if args.child:
        child(args.side, args.reps)
        return
    lib = os.path.abspath(args.lib) if args.lib else build_variant(os.path.abspath(args.src))
    if args.build_only:
        print(json.dumps({"built": lib}))
        return
    env = dict(os.environ, B200_LIB=lib)
    env.setdefault("B200_BENCH_TILE_CACHE", os.path.join(tempfile.gettempdir(), "b200_tiles_probe"))
    os.makedirs(env["B200_BENCH_TILE_CACHE"], exist_ok=True)
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--side", str(args.side), "--reps", str(args.reps)],
                       env=env, capture_output=True, text=True, cwd=ROOT)
    if r.returncode != 0:
        sys.stderr.write(r.stderr[-4000:])
        raise SystemExit(r.returncode)
    line = json.dumps({"label": args.label, "gpu": gpu_info(), **summarise(json.loads(r.stdout.strip().splitlines()[-1]), args.bins)})
    print(line, flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "k0_trace.jsonl"), "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
