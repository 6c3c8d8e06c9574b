"""CPU: the Python mirror of the C ABI (libheif_b200/_lib.py) against include/.  Every ctypes struct has the size and field
offsets the C compiler gives the header's struct, the public signature table names exactly the functions the headers
declare, and every test-only entry point resolves in the built library."""
import ctypes as C
import os
import re
import subprocess

from libheif_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INCLUDE = os.path.join(ROOT, "include")

# struct of include/b200_heif.h -> its ctypes mirror
STRUCTS = {
    "b200_planes": _lib.Planes,
    "b200_geometry": _lib.Geometry,
    "b200_color_options": _lib.ColorOptions,
    "b200_rgb_image": _lib.RgbImage,
    "b200_rgb_to_ycbcr_options": _lib.RgbToYCbCrOptions,
    "b200_hevc_enc_params": _lib.EncParams,
    "b200_gpu_encode_stats": _lib.GpuEncodeStats,
    "b200_grid_encode_info": _lib.GridEncodeInfo,
    "b200_image_info": _lib.ImageInfo,
    "b200_decode_stats": _lib.DecodeStats,
}


def header(name):
    """include/<name> without its comments."""
    return re.sub(r"/\*.*?\*/|//[^\n]*", " ", open(os.path.join(INCLUDE, name)).read(), flags=re.S)


def declared_functions():
    return set(re.findall(r"\b(b200_\w+)\s*\(", header("b200_heif.h") + header("b200_heif_plugin_abi.h")))


def test_every_header_struct_has_one_mirror():
    assert set(STRUCTS) == set(re.findall(r"typedef struct (b200_\w+) \{", header("b200_heif.h")))
    assert set(STRUCTS.values()) == {v for v in vars(_lib).values() if isinstance(v, type) and issubclass(v, C.Structure)}


def test_struct_layouts_match_the_c_compiler(tmp_path):
    src = ["#include <stddef.h>", "#include <stdio.h>", '#include "b200_heif.h"', "int main(void) {"]
    want = []
    for name, cls in STRUCTS.items():
        src.append(f'  printf("{name} %zu\\n", sizeof({name}));')
        want.append(f"{name} {C.sizeof(cls)}")
        for field, *_ in cls._fields_:
            src.append(f'  printf("{name}.{field} %zu\\n", offsetof({name}, {field}));')
            want.append(f"{name}.{field} {getattr(cls, field).offset}")
    src += ["  return 0;", "}"]
    (tmp_path / "layout.c").write_text("\n".join(src) + "\n")
    exe = tmp_path / "layout"
    r = subprocess.run(["cc", "-std=c11", "-I", INCLUDE, str(tmp_path / "layout.c"), "-o", str(exe)], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout[-3000:]
    got = subprocess.run([str(exe)], stdout=subprocess.PIPE, text=True, check=True).stdout.splitlines()
    assert got == want, [(g, w) for g, w in zip(got, want) if g != w] or (len(got), len(want))


def test_function_table_names_the_header_functions():
    declared, table = declared_functions(), set(_lib.FUNCTIONS)
    assert not declared - table, f"declared in include/ but missing from _lib.FUNCTIONS: {sorted(declared - table)}"
    assert not table - declared, f"in _lib.FUNCTIONS but not declared in include/: {sorted(table - declared)}"


def test_test_only_entry_points_resolve():
    names = set(_lib.DEBUG_FUNCTIONS)
    assert all(n.startswith("b200_debug_") for n in names | set(_lib.TRACE_FUNCTIONS)), sorted(names)
    assert not (names | set(_lib.TRACE_FUNCTIONS)) & declared_functions()
    lib = _lib.lib()
    assert not [n for n in sorted(names) if not hasattr(lib, n)]
