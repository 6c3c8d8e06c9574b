"""Device timing of the RGB -> YCbCr kernel against its HBM roofline (development probe; bench.py is the judged harness).
Inputs larger than L2 (16384 x 8192 x 3 B = 403 MB), median of 10 launches after 3 warm-ups, CUDA events on the launch stream."""
import sys, os, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import libheif_b200 as lb

peak = 3350.0      # H100 SXM data sheet HBM3 bandwidth
res = {"peak_gbs": peak}
w, h = 16384, 8192
for bpp in (3, 4):
    rgb = torch.randint(0, 256, (h, w, bpp), dtype=torch.uint8, device="cuda")
    for chroma, out_b in ((1, 1.5), (2, 2.0), (3, 3.0)):
        for _ in range(3):
            lb.rgb_to_ycbcr(rgb, chroma, full_range=False, want_alpha=False)
        torch.cuda.synchronize()
        ts = []
        for _ in range(10):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); lb.rgb_to_ycbcr(rgb, chroma, full_range=False, want_alpha=False); e1.record(); torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        ms = sorted(ts)[len(ts) // 2]          # includes the three plane allocations of the Python mirror (caching allocator: no cudaMalloc)
        gbs = w * h * (bpp + out_b) / ms / 1e6
        res[f"rgb{bpp * 8}_to_{ {1: '420', 2: '422', 3: '444'}[chroma]}"] = dict(ms=round(ms, 4), mp_s=round(w * h / ms / 1e3, 1), algorithmic_gb_s=round(gbs, 1), frac=round(gbs / peak, 3))
print(json.dumps(res, indent=1))
