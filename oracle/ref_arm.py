"""
oracle/ref_arm.py -- TEST / BENCH INFRASTRUCTURE ONLY: the reference CPU path timed through the reference's own public API.

    python -m oracle.ref_arm --side 16 [--sub 8] --steps K --warmup W --threads C

builds (untimed) a HEIC grid file from the very tiles bench.py's GPU arm decodes (bench.make_tile, wrapped by
oracle/heic_writer.py), then times heif_decode_image() of the UNMODIFIED reference libheif (oracle/_ref/libheif_ref.so,
compiled from /root/reference by oracle/Makefile) with the CPU decoder plugin of the oracle (FFmpeg in the libde265
role, oracle/ref_plugin.cc) to interleaved RGB, heif_context_set_max_decoding_threads(C) -- the call and the thread
model of SURVEY.md 8(d) "CPU baseline beside it".  Prints one JSON line: per-step milliseconds, MP/s, md5 of the RGB.
Runs in its own process and never imports torch (libheif_ref.so is loaded RTLD_GLOBAL, see oracle/refheif.py).

    python -m oracle.ref_arm --decoder b200 --threads 256 [--lib libheif_ref_b200.so]

is the drop-in leg of bench.py ("e2e_plugin"): the same file, the same heif_decode_image() call of the same unmodified
library, but the decoder plugin it selects is the product's (libb200heif.so, registered with heif_register_decoder_plugin);
here the reference is the HOST APPLICATION of the product, not its checker.  --lib libheif_ref_b200.so uses the second
build that carries the GPU colour operation (SURVEY 8f N2, integration/colorconversion_b200.patch).
"""
import argparse
import ctypes as C
import hashlib
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--side", type=int, default=16, help="the full grid is side x side tiles")
    ap.add_argument("--sub", type=int, default=0, help="> 0: decode only the top-left sub x sub tiles (bounded sample)")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--threads", type=int, default=0)
    ap.add_argument("--ctb", type=int, default=5)
    ap.add_argument("--dump", default="", help="write the RGB of the last step to this file (raw bytes)")
    ap.add_argument("--decoder", default="b200-oracle", choices=["b200-oracle", "b200"], help="decoder plugin: the oracle's CPU plugin, or the product's GPU plugin")
    ap.add_argument("--lib", default="", help="reference build to load (default libheif_ref.so; libheif_ref_b200.so = + GPU colour operation)")
    args = ap.parse_args()
    if args.lib:
        os.environ["B200_REF_LIB"] = args.lib
    import numpy as np  # noqa: F401
    import bench
    from oracle import bindings as ob
    from oracle import heic_writer as hw
    from oracle import refheif as rh
    gpu = args.decoder == "b200"
    if gpu:
        if not os.path.exists(os.path.join(ob.REF, args.lib or "libheif_ref.so")):
            print(json.dumps({"unavailable": f"oracle/_ref/{args.lib or 'libheif_ref.so'} missing"}))
            return
    elif not (os.path.exists(os.path.join(ob.REF, "libheif_ref.so")) and os.path.exists(os.path.join(ob.REF, "liboracle_plugin.so")) and ob.avcodec_dir()):
        print(json.dumps({"unavailable": "oracle/_ref reference build or FFmpeg missing"}))
        return
    threads = args.threads or bench.effective_cores()
    sub = args.sub or args.side
    idx = [r * args.side + c for r in range(sub) for c in range(sub)]
    t0 = time.perf_counter()
    tiles = bench.make_tiles(idx, log2_ctb=args.ctb)
    t_gen = time.perf_counter() - t0
    tmpdir = "/dev/shm" if os.path.isdir("/dev/shm") else tempfile.gettempdir()
    path = os.path.join(tmpdir, f"b200_ref_arm_{os.getpid()}.heic")
    hw.write_heic(path, tiles, cols=sub, rows=sub)
    try:
        h = rh.load()
        stats = None
        if gpu:
            from libheif_b200 import _lib
            b200 = _lib.lib()
            if b200.b200_plugin_bind_libheif(None) != 0:
                raise RuntimeError("the plugin could not resolve the libheif C API")
            rh.check(h.heif_register_decoder_plugin(C.c_void_p(b200.b200_get_decoder_plugin())), "register decoder plugin")
        else:
            rh.register_cpu_decoder()
        out = None
        for _ in range(args.warmup):
            out = rh.decode_file(path, decoder_id=args.decoder, threads=threads)
        ts, tw = [], []
        for _ in range(args.steps):
            t = time.perf_counter()
            out = rh.decode_file(path, decoder_id=args.decoder, threads=threads)
            tw.append(time.perf_counter() - t)
            ts.append(rh.last_timing["api_s"])           # heif_context_read_from_file .. heif_decode_image (the file lives in /dev/shm)
        if gpu:
            st = (C.c_uint64 * 3)()
            b200.b200_plugin_queue_stats(st)
            stats = {"batches": int(st[0]), "pictures": int(st[1]), "largest_batch": int(st[2])}
    finally:
        os.unlink(path)
    ms = 1e3 * sum(ts) / max(1, len(ts))
    px = out.shape[0] * (out.shape[1] // 3)
    if args.dump:
        out.tofile(args.dump)
    print(json.dumps({"ms_per_step": ms, "mp_s": px / 1e6 / (ms / 1e3), "pixels": px, "width": out.shape[1] // 3, "height": out.shape[0],
                      "tiles": sub * sub, "threads": threads, "ms_per_step_incl_copy_to_numpy": 1e3 * sum(tw) / max(1, len(tw)), "steps": args.steps, "warmup": args.warmup, "rgb_md5": hashlib.md5(out.tobytes()).hexdigest(),
                      "file_bytes": sum(len(t) for t in tiles), "tile_generation_s": t_gen,
                      "plugin_queue": stats,
                      "api": (f"heif_decode_image ({args.lib or 'libheif_ref.so'}) + libb200heif.so decoder plugin, heif_context_set_max_decoding_threads" if gpu else
                              "heif_decode_image (libheif_ref.so, unmodified) + oracle CPU decoder plugin (FFmpeg), heif_context_set_max_decoding_threads")}))


if __name__ == "__main__":
    main()
