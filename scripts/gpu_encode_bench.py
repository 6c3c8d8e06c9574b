"""GPU HEVC intra encoder on the 16384^2 workload: 256 x 1024^2 synthetic_image tiles (seeds 0xB200 + k), QP 27, CTB 32,
device-resident planes -> access units in host memory.  Median of --calls calls after a warm-up; E1 / E2 times from CUDA
events, framing from the host clock; bits per pixel, luma PSNR, an in-run round trip of every access unit through
lb.Decoder (reconstruction before deblocking == the encoder's recon), and the host encoder on all host cores with the
same tiles and tool set.  Prints the card name, power limit and maximum SM clock of the run.

--speeds 0,1,2 codes the tiles at each listed mode-decision speed (b200_hevc_enc_params::speed), the speeds alternating call
by call in one process; the top-level fields are those of the first speed, and "speeds" holds per speed the median call,
E1 / E2 times, bytes, bits per pixel, luma PSNR, the decision pass's work counters and E1's resident warps per SM.  The
default (--speeds 0) prints what the script printed before speeds existed.

    python scripts/gpu_encode_bench.py [--tiles 256] [--size 1024] [--calls 5] [--speeds 0] [--out DIR]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import libheif_b200 as lb  # noqa: E402
from libheif_b200.hevc_enc import GpuEncoder, encode_intra, synthetic_image  # noqa: E402


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tiles", type=int, default=256)
    ap.add_argument("--size", type=int, default=1024)
    ap.add_argument("--calls", type=int, default=5)
    ap.add_argument("--qp", type=int, default=27)
    ap.add_argument("--host-tiles", type=int, default=0, help="tiles for the host-encoder arm (0 = all)")
    ap.add_argument("--speeds", default="0", help="comma-separated speeds, run alternately (default 0)")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    speeds = [int(x) for x in a.speeds.split(",")]
    import torch
    assert torch.cuda.is_available(), "needs a CUDA device"
    n, s = a.tiles, a.size
    t = time.time()
    with ThreadPoolExecutor(os.cpu_count()) as ex:
        tiles = list(ex.map(lambda k: synthetic_image(0xB200 + k, s, s, 8, True), range(n)))
    gen_s = time.time() - t
    dev = [tuple(torch.from_numpy(p).cuda() for p in tl) for tl in tiles]
    torch.cuda.synchronize()
    enc = GpuEncoder()
    params = dict(qp=a.qp, log2_ctb_size=5)
    sp = {k: dict(params, speed=k) if k else params for k in speeds}
    for k in speeds:
        enc.encode(dev, **sp[k])                                 # warm-up (allocations, module load)
    calls = {k: [] for k in speeds}
    for _ in range(a.calls):
        for k in speeds:                                         # speeds alternate call by call
            t = time.perf_counter()
            enc.encode(dev, **sp[k])
            wall = (time.perf_counter() - t) * 1e3
            st = enc.stats()
            calls[k].append(dict(wall_ms=wall, analyse_ms=st.analyse_ms, entropy_ms=st.entropy_ms, framing_ms=st.framing_ms))
    px = n * s * s
    dec = lb.Decoder(host_threads=os.cpu_count())
    dec.set_debug_stage(1)
    cols = int(np.sqrt(n)) if int(np.sqrt(n)) ** 2 == n else n
    per = {}
    for k in speeds:
        aus = enc.encode(dev, **sp[k])                           # the bytes every timed call of this speed produced
        st = enc.stats()
        # round trip: every access unit through this library's decoder, stopped before deblocking, == the encoder's recon
        dec.decode_grid(aus, cols=cols, rows=n // cols)
        recon_ok, psnrs = True, []
        for i in range(n):
            rec = enc.recon(i)
            got = dec.debug_tile(i, s, s)
            recon_ok &= all(np.array_equal(got[c][:rec[c].shape[0], :rec[c].shape[1]], rec[c]) for c in range(3))
            mse = np.mean((rec[0].astype(np.float64) - tiles[i][0]) ** 2)
            psnrs.append(10 * np.log10(255.0 ** 2 / max(mse, 1e-12)))
        med = {f: statistics.median(c[f] for c in calls[k]) for f in calls[k][0]}
        per[k] = dict(med=med, aus=aus, bytes=sum(map(len, aus)), psnr=float(np.mean(psnrs)), recon_ok=bool(recon_ok),
                      mode_evaluations=int(st.mode_evaluations), cu_evaluations=int(st.cu_evaluations),
                      e1_warps_per_sm=enc.e1_warps_per_sm(k))
    dec.close()
    first = per[speeds[0]]
    med, aus, total_bytes, recon_ok = first["med"], first["aus"], first["bytes"], all(v["recon_ok"] for v in per.values())
    # host encoder, all cores, same tiles and tool set
    hn = a.host_tiles or n
    hk = dict(qp=a.qp, log2_ctb_size=5, sao=0, sign_data_hiding=0, cu_qp_delta=0, wpp=1)
    t = time.perf_counter()
    with ThreadPoolExecutor(os.cpu_count()) as ex:
        host = list(ex.map(lambda k: encode_intra(*tiles[k], seed=0xB200 + k, **hk), range(hn)))
    host_ms = (time.perf_counter() - t) * 1e3
    res = dict(
        card=card(), host_cores=os.cpu_count(), tiles=n, tile_size=s, qp=a.qp, ctb=32, calls=a.calls, source_gen_s=round(gen_s, 1),
        median_wall_ms=round(med["wall_ms"], 2), median_e1_ms=round(med["analyse_ms"], 2), median_e2_ms=round(med["entropy_ms"], 2),
        median_framing_ms=round(med["framing_ms"], 2), mp_per_s=round(px / 1e6 / (med["wall_ms"] / 1e3), 1),
        bytes=total_bytes, bits_per_px=round(8 * total_bytes / px, 4), luma_psnr_recon_db=round(first["psnr"], 3),
        roundtrip_stage1_equal=bool(recon_ok),
        host_encoder=dict(tiles=hn, ms=round(host_ms, 1), mp_per_s=round(hn * s * s / 1e6 / (host_ms / 1e3), 2),
                          bytes_same_tiles=sum(map(len, host)), gpu_bytes_same_tiles=sum(map(len, aus[:hn]))),
        per_call=calls[speeds[0]])
    if speeds != [0]:
        res["speeds"] = {str(k): dict(
            median_wall_ms=round(v["med"]["wall_ms"], 2), mp_per_s=round(px / 1e6 / (v["med"]["wall_ms"] / 1e3), 1),
            median_e1_ms=round(v["med"]["analyse_ms"], 2), median_e2_ms=round(v["med"]["entropy_ms"], 2), bytes=v["bytes"],
            bits_per_px=round(8 * v["bytes"] / px, 4), luma_psnr_recon_db=round(v["psnr"], 3), roundtrip_stage1_equal=v["recon_ok"],
            mode_evaluations=v["mode_evaluations"], cu_evaluations=v["cu_evaluations"], e1_warps_per_sm=v["e1_warps_per_sm"],
            per_call=calls[k]) for k, v in per.items()}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "gpu_encode_bench.json"), "w") as f:
            f.write(line + "\n")
    enc.close()
    return 0 if recon_ok else 1


if __name__ == "__main__":
    sys.exit(main())
