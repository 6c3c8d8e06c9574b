"""Image sequences through the unmodified reference libheif (oracle/_ref/libheif_ref.so) with this library's plugins:
heif_track_encode_sequence_image of N synthetic 8-bit 4:2:0 frames with "b200-gpu" at sequence-batch 1 and automatic (0) and
with the host table "b200", then heif_track_decode_next_image of the track with this library's decoder plugin at read-ahead 1
and at its default.  Prints frames/s, MP/s, the GPU encode calls / decoder batches the plugins ran, the md5 of the decoded
frames, and the card name and power limit, as one JSON line.

    python scripts/sequence_bench.py [--sizes 512x128,1024x32] [--repeats 3] [--quality 70] [--out DIR]

Each arm runs in a child process of its own (the reference is loaded RTLD_GLOBAL, and each arm registers one encoder table).
The frames cycle through 16 distinct synthetic_image pictures (seeds 0x5B00 + k).  Each arm first runs an untimed warm-up:
encoders encode up to 64 frames with the same heif_encoder the timed runs use (CUDA context, module load, the GPU encoder and
its page-locked staging at the batch size of the timed runs), the decoder decodes the whole track once.  Then --repeats timed
runs; the line reports each run's seconds and rates from the median.
"""
import argparse
import ctypes as C
import hashlib
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DISTINCT = 16


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def arm(kind, size, frames, quality, batch, path, repeats):
    """Child: 'encode-gpu' / 'encode-host' write the sequence to `path`; 'decode' reads it back with the decoder plugin."""
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import numpy as np
    from oracle import refheif as rh
    import refheif_seq as rs
    from libheif_b200 import _lib
    from libheif_b200.hevc_enc import synthetic_image
    h = rs.load()
    b200 = _lib.lib()
    assert b200.b200_plugin_bind_libheif(None) == 0
    out = {}
    if kind.startswith("encode"):
        table = b200.b200_get_gpu_encoder_plugin() if kind == "encode-gpu" else b200.b200_get_encoder_plugin()
        rh.check(h.heif_register_encoder_plugin(table), "register encoder")
        pics = [synthetic_image(0x5B00 + k, size, size, 8, True) for k in range(DISTINCT)]
        imgs = [rh.make_ycbcr_image(*pics[k % DISTINCT]) for k in range(frames)]
        params = {"sequence-batch": batch} if kind == "encode-gpu" else {}
        enc = rs.new_encoder(quality, params)
        rs.write_sequence(path + ".warm", imgs[:min(frames, 64)], encoder=enc)
        secs, calls = [], []
        for _ in range(repeats):
            s0 = (C.c_uint64 * 3)()
            b200.b200_plugin_encoder_stats(s0)
            t = time.perf_counter()
            rs.write_sequence(path, imgs, encoder=enc, timescale=1000, durations=[40] * frames)
            secs.append(time.perf_counter() - t)
            s1 = (C.c_uint64 * 3)()
            b200.b200_plugin_encoder_stats(s1)
            calls.append(int(s1[0] - s0[0]))
        h.heif_encoder_release(enc)
        for i in imgs:
            h.heif_image_release(i)
        out = dict(seconds=secs, gpu_calls=calls[-1], gpu_max_batch=int(s1[2]), bytes=os.path.getsize(path),
                   file_md5=hashlib.md5(open(path, "rb").read()).hexdigest())
    else:
        rh.check(h.heif_register_decoder_plugin(b200.b200_get_decoder_plugin()), "register decoder")
        rs.decode_track(path, decoder_id="b200")                                # warm-up
        secs = []
        for _ in range(repeats):
            q0 = (C.c_uint64 * 3)()
            b200.b200_plugin_queue_stats(q0)
            t = time.perf_counter()
            calls = rs.decode_track(path, decoder_id="b200")
            secs.append(time.perf_counter() - t)
            q1 = (C.c_uint64 * 3)()
            b200.b200_plugin_queue_stats(q1)
        m = hashlib.md5()
        for c in calls:
            assert c[0] == "ok", c
            for k in ("y", "cb", "cr"):
                m.update(np.ascontiguousarray(c[1][k]).tobytes())
        out = dict(seconds=secs, frames=len(calls), batches=int(q1[0] - q0[0]), max_batch=int(q1[2]), md5=m.hexdigest())
    print("ARM " + json.dumps(out))


def rates(r, frames, mp):
    if "seconds" in r:
        med = statistics.median(r["seconds"])
        r["frames_per_s"] = frames / med
        r["mp_per_s"] = mp / med
        r["frames_per_s_range"] = [frames / max(r["seconds"]), frames / min(r["seconds"])]
    return r


def run_arm(args, env=None):
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--arm"] + [str(a) for a in args], stdout=subprocess.PIPE,
                       stderr=subprocess.PIPE, text=True, env=env, timeout=3600)
    if r.returncode != 0:
        return dict(error=(r.stderr or r.stdout)[-600:])
    return json.loads([l for l in r.stdout.splitlines() if l.startswith("ARM ")][-1][4:])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="512x128,1024x32", help="SIZExFRAMES,...")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--quality", type=int, default=70)
    ap.add_argument("--out", default=None)
    ap.add_argument("--arm", nargs=7, default=None, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.arm:
        kind, size, frames, quality, batch, path, repeats = a.arm
        arm(kind, int(size), int(frames), int(quality), int(batch), path, int(repeats))
        return
    tmp = tempfile.mkdtemp()
    res = dict(card=card(), quality=a.quality, repeats=a.repeats, runs=[])
    for spec in a.sizes.split(","):
        size, frames = (int(x) for x in spec.split("x"))
        mp = size * size * frames / 1e6
        run = dict(size=size, frames=frames)
        for name, kind, batch in (("gpu_batch1", "encode-gpu", 1), ("gpu_auto", "encode-gpu", 0), ("host", "encode-host", 0)):
            path = os.path.join(tmp, f"{name}_{size}.heif")
            run["encode_" + name] = rates(run_arm([kind, size, frames, a.quality, batch, path, a.repeats]), frames, mp)
        path = os.path.join(tmp, f"gpu_auto_{size}.heif")
        for name, ra in (("readahead1", "1"), ("readahead_default", None)):
            env = dict(os.environ)
            env.pop("B200_SEQ_READAHEAD", None)
            if ra:
                env["B200_SEQ_READAHEAD"] = ra
            run["decode_" + name] = rates(run_arm(["decode", size, frames, a.quality, 0, path, a.repeats], env=env), frames, mp)
        res["runs"].append(run)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "sequence_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
