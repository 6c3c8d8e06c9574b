"""Device timing of the RGB -> YCbCr kernel against its HBM roofline (development probe; bench.py is the judged harness).
Inputs larger than L2 (16384 x 8192 x 3 B = 403 MB; the rgb_to_ycbcr_ex layouts 8192 x 8192), median of 10 launches after 3 warm-ups, CUDA events on the launch stream."""
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


def timed(fn):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(10):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return sorted(ts)[len(ts) // 2]


# rgb_to_ycbcr_ex: RRGGBB 10 bit LE -> 4:2:0 (Op_RRGGBBxx_HDR_to_YCbCr420, full range; Op_RGB_to_YCbCr<uint16_t> behind the
# folded swap / unpack, limited range) and planar RGB 8 / 16 bit -> 4:2:0 (Op_RGB_to_YCbCr<T>)
w, h = 8192, 8192
rr = torch.randint(0, 1024, (h, w, 3), dtype=torch.int16, device="cuda").view(torch.uint16)
for full in (True, False):
    ms = timed(lambda: lb.rgb_to_ycbcr_ex(rr, 1, 10, "little", matrix_coefficients=9, colour_primaries=9, full_range=full))
    gbs = w * h * (6 + 3) / ms / 1e6
    res[f"rrggbb10le_to_420_{'full' if full else 'limited'}"] = dict(ms=round(ms, 4), algorithmic_gb_s=round(gbs, 1), frac=round(gbs / peak, 3))
for depth, dt, bps in ((8, torch.uint8, 1), (16, torch.int16, 2)):
    pl = tuple(torch.randint(0, 256, (h, w), dtype=dt, device="cuda").view(torch.uint16 if bps == 2 else torch.uint8) for _ in range(3))
    ms = timed(lambda: lb.rgb_to_ycbcr_ex(pl, 1, depth, matrix_coefficients=6, full_range=False))
    gbs = w * h * bps * (3 + 1.5) / ms / 1e6
    res[f"planar{depth}_to_420"] = dict(ms=round(ms, 4), algorithmic_gb_s=round(gbs, 1), frac=round(gbs / peak, 3))
print(json.dumps(res, indent=1))
