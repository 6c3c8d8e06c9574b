"""K0 occupancy probe: how the entropy kernel scales with the number of resident decoders per SM.

Builds library variants of one source tree (libheif_b200.build.build with extra nvcc flags), then decodes the bench grid
(side x side tiles of 1024x1024, device front-end, one launch per kernel: B200_CHUNKS=0 B200_TAIL_OVERLAP=0, as bench.py's
kernel leg) with each of them, round-robin, one child process per (round, variant), and prints one JSON line per
measurement and a summary line: best / median K0 time and G bins/s per variant, card name and power limit.

  python scripts/k0_occupancy_probe.py --build-only               # here: compile the variants
  python scripts/k0_occupancy_probe.py --rounds 3 --out DIR       # on the GPU: measure (builds what is missing)

Variants (--variants "name=flags;..."), by default: cap2, cap3, cap4 (B200_ENTROPY_MAX_BLOCKS_PER_SM), min5
(B200_ENTROPY_MIN_BLOCKS=5: five CTAs forced by __launch_bounds__) and the unmodified build.  --src names another
checkout's libheif_b200 package directory (to measure an older commit with the same script); --label prefixes the
variant names.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEFAULT_VARIANTS = "cap2=-DB200_ENTROPY_MAX_BLOCKS_PER_SM=2;cap3=-DB200_ENTROPY_MAX_BLOCKS_PER_SM=3;cap4=-DB200_ENTROPY_MAX_BLOCKS_PER_SM=4;" \
                   "min5=-DB200_ENTROPY_MIN_BLOCKS=5;default="


def parse_variants(spec):
    out = []
    for item in spec.split(";"):
        if item.strip():
            name, _, flags = item.partition("=")
            out.append((name.strip(), flags.split()))
    return out


def build_variants(src, variants, tag_prefix):
    import importlib.util
    spec = importlib.util.spec_from_file_location("_probe_build", os.path.join(src, "build.py"))
    b = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(b)
    libs = {}
    for name, flags in variants:
        out = os.path.join(src, "build", f"libb200heif_{tag_prefix}{name}.so")
        # every variant, the unmodified one too, gets a define and an object tag of its own: build() then always links it
        # to `out` and never mixes objects of two variants
        libs[name] = b.build(extra_flags=flags + ["-DB200_PROBE_VARIANT_" + name.upper()], out=out, tag="_" + tag_prefix + name)
        print(json.dumps({"built": tag_prefix + name, "lib": out, "flags": flags}), flush=True)
    return libs


def child(side, reps):
    """One measurement with the library named by B200_LIB: K0 ms of `reps` reruns after one warm-up run."""
    os.environ["B200_CHUNKS"] = "0"
    os.environ["B200_TAIL_OVERLAP"] = "0"
    sys.path.insert(0, ROOT)
    import hashlib
    import bench
    import torch
    import libheif_b200 as lb
    tiles = bench.make_tiles(range(side * side))
    dec = lb.Decoder(host_threads=16)
    dec.set_front_end(True)
    dec.decode_grid(tiles, cols=side, rows=side)
    en = []
    for _ in range(reps + 1):
        dec.rerun_device(torch.cuda.current_stream())
        torch.cuda.synchronize()
        en.append(dec.stats().entropy_ms)
    out = dec.to_rgb_device(lb.CHROMA_INTERLEAVED_RGB)
    torch.cuda.synchronize()
    md5 = hashlib.md5(out.cpu().numpy().tobytes()).hexdigest()
    print(json.dumps({"entropy_ms": en[1:], "md5": md5}))


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except Exception as e:  # noqa: BLE001 - reported, not fatal
        return f"unavailable: {e}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--src", default=os.path.join(ROOT, "libheif_b200"), help="libheif_b200 package directory whose sources are built")
    ap.add_argument("--variants", default=DEFAULT_VARIANTS)
    ap.add_argument("--label", default="", help="prefix of the variant names in the output (and of the built libraries)")
    ap.add_argument("--side", type=int, default=16)
    ap.add_argument("--reps", type=int, default=4, help="K0 runs per child process (after one warm-up run)")
    ap.add_argument("--rounds", type=int, default=2, help="round-robin passes over the variants")
    ap.add_argument("--lib", action="append", default=[], metavar="NAME=PATH", help="also measure this already built library (e.g. of another checkout)")
    ap.add_argument("--build-only", action="store_true")
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--out", default=None, help="also append the JSON lines to DIR/k0_occupancy.jsonl")
    args = ap.parse_args()
    if args.child:
        child(args.side, args.reps)
        return
    built = build_variants(os.path.abspath(args.src), parse_variants(args.variants), args.label)
    if args.build_only:
        return
    libs = {args.label + name: path for name, path in built.items()}
    for item in args.lib:
        name, _, path = item.partition("=")
        libs[name] = os.path.abspath(path)
    names = list(libs)
    env = dict(os.environ)
    env.setdefault("B200_BENCH_TILE_CACHE", os.path.join(tempfile.gettempdir(), "b200_tiles_probe"))
    os.makedirs(env["B200_BENCH_TILE_CACHE"], exist_ok=True)
    sink = open(os.path.join(args.out, "k0_occupancy.jsonl"), "a") if args.out else None

    def emit(d):
        line = json.dumps(d)
        print(line, flush=True)
        if sink:
            sink.write(line + "\n"); sink.flush()

    emit({"gpu": gpu_info()})
    times = {name: [] for name in names}
    md5s = {name: set() for name in names}
    for rnd in range(args.rounds):
        for name in names:
            env["B200_LIB"] = libs[name]
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--side", str(args.side), "--reps", str(args.reps)],
                               env=env, capture_output=True, text=True, cwd=ROOT)
            if r.returncode != 0:
                emit({"variant": name, "round": rnd, "error": r.stderr[-2000:]})
                continue
            res = json.loads(r.stdout.strip().splitlines()[-1])
            times[name] += res["entropy_ms"]; md5s[name].add(res["md5"])
            emit({"variant": name, "round": rnd, **res})
    bins = 2.0 * (args.side * 1024) ** 2          # bench.py's count: ~2.0 CABAC bins per pixel on this workload
    summary = {}
    for name in names:
        t = times[name]
        if t:
            summary[name] = {"entropy_ms_min": min(t), "entropy_ms_median": statistics.median(t), "entropy_ms_max": max(t), "n": len(t),
                                          "gbins_per_s_best": bins / (min(t) * 1e-3) / 1e9, "md5": sorted(md5s[name])}
    emit({"summary": summary, "gpu": gpu_info()})


if __name__ == "__main__":
    main()
