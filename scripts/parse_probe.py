"""Host front-end scaling probe: parse the same 64 bench tiles with 1..N threads (no GPU involved)."""
import ctypes as C, os, sys, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench
from libheif_b200 import _lib
n = 64
tiles = bench.make_tiles(range(n))
l = _lib.lib()
arr = (C.c_char_p * n)(*tiles); sizes = (C.c_size_t * n)(*[len(t) for t in tiles])
res = {}
for th in (1, 4, 8, 16, 32, 64, 128):
    if th > 2 * (os.cpu_count() or 8): break
    ms = C.c_double()
    l.b200_debug_parse_many(arr, sizes, n, th, 3, C.byref(ms))
    res[th] = {"ms": ms.value, "mp_s": n * 1.048576 / (ms.value / 1e3)}
print(json.dumps(res, indent=1))
