"""GPU HEVC intra encoder on the 16384^2 workload: 256 x 1024^2 synthetic_image tiles (seeds 0xB200 + k), QP 27, CTB 32,
device-resident planes -> access units in host memory.  Median of --calls calls after a warm-up; E1 / E2 times from CUDA
events, framing from the host clock; bits per pixel, luma PSNR, an in-run round trip of every access unit through
lb.Decoder (reconstruction before deblocking == the encoder's recon), and the host encoder on all host cores with the
same tiles and tool set.  Prints the card name and power limit of the run.

    python scripts/gpu_encode_bench.py [--tiles 256] [--size 1024] [--calls 5] [--out DIR]
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
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
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
    aus = enc.encode(dev, **params)                              # warm-up (allocations, module load)
    calls = []
    for _ in range(a.calls):
        t = time.perf_counter()
        aus = enc.encode(dev, **params)
        wall = (time.perf_counter() - t) * 1e3
        st = enc.stats()
        calls.append(dict(wall_ms=wall, analyse_ms=st.analyse_ms, entropy_ms=st.entropy_ms, framing_ms=st.framing_ms))
    med = {k: statistics.median(c[k] for c in calls) for k in calls[0]}
    px = n * s * s
    total_bytes = sum(map(len, aus))
    # round trip: every access unit through this library's decoder, stopped before deblocking, == the encoder's recon
    dec = lb.Decoder(host_threads=os.cpu_count())
    dec.set_debug_stage(1)
    cols = int(np.sqrt(n)) if int(np.sqrt(n)) ** 2 == n else n
    dec.decode_grid(aus, cols=cols, rows=n // cols)
    recon_ok, psnrs = True, []
    for k in range(n):
        rec = enc.recon(k)
        got = dec.debug_tile(k, s, s)
        recon_ok &= all(np.array_equal(got[c][:rec[c].shape[0], :rec[c].shape[1]], rec[c]) for c in range(3))
        mse = np.mean((rec[0].astype(np.float64) - tiles[k][0]) ** 2)
        psnrs.append(10 * np.log10(255.0 ** 2 / max(mse, 1e-12)))
    dec.close()
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
        bytes=total_bytes, bits_per_px=round(8 * total_bytes / px, 4), luma_psnr_recon_db=round(float(np.mean(psnrs)), 3),
        roundtrip_stage1_equal=bool(recon_ok),
        host_encoder=dict(tiles=hn, ms=round(host_ms, 1), mp_per_s=round(hn * s * s / 1e6 / (host_ms / 1e3), 2),
                          bytes_same_tiles=sum(map(len, host)), gpu_bytes_same_tiles=sum(map(len, aus[:hn]))),
        per_call=calls)
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
