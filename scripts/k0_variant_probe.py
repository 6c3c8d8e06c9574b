"""K0 variant probe: decode side x side tiles of 1024x1024 (device front-end, one launch per kernel) with the library named by
B200_LIB and print one JSON line: best / mean entropy_ms over the repetitions, recon_ms, md5 of the RGB result."""
import hashlib, json, os, sys, tempfile
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench, torch
import libheif_b200 as lb
side = int(sys.argv[1]) if len(sys.argv) > 1 else 16
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 4
os.environ.setdefault("B200_BENCH_TILE_CACHE", os.path.join(tempfile.gettempdir(), "b200_tiles_shared"))
os.makedirs(os.environ["B200_BENCH_TILE_CACHE"], exist_ok=True)
os.environ["B200_CHUNKS"] = "0"
tiles = bench.make_tiles(range(side * side))
dec = lb.Decoder(host_threads=16)
dec.set_front_end(True)
en, rc, db, sa = [], [], [], []
dec.decode_grid(tiles, cols=side, rows=side)
for _ in range(reps + 1):
    dec.rerun_device(torch.cuda.current_stream())
    out = dec.to_rgb_device(lb.CHROMA_INTERLEAVED_RGB)
    torch.cuda.synchronize()
    st = dec.stats()
    en.append(st.entropy_ms); rc.append(st.recon_ms); db.append(st.deblock_ms); sa.append(st.sao_ms)
md5 = hashlib.md5(out.cpu().numpy().tobytes()).hexdigest()
print(json.dumps({"lib": os.path.basename(os.environ.get("B200_LIB", "libb200heif.so")), "tail": os.environ.get("B200_TAIL_OVERLAP", ""), "side": side, "entropy_ms_min": min(en[1:]), "entropy_ms_mean": sum(en[1:]) / reps,
                  "recon_ms_mean": sum(rc[1:]) / reps, "deblock_ms_mean": sum(db[1:]) / reps, "sao_ms_mean": sum(sa[1:]) / reps, "front_end": st.front_end, "md5": md5}))
