"""Regenerates tests/golden/streams/*.au from the reference's own fixture files (needs the reference source tree and the
oracle/_ref build):

    python tests/golden/make_streams.py [--check]

Each .au is byte-for-byte what the UNMODIFIED reference libheif pushes into a decoder plugin for one coded image item
(Decoder::get_compressed_data, libheif/codecs/decoder.cc:275-308: hvcC parameter-set NALs followed by the item's NALs,
each with a 4-byte big-endian length).  They are captured by the CPU oracle plugin (oracle/ref_plugin.cc,
B200_ORACLE_DUMP_DIR) while heif_decode_image decodes the file -- run in a child process per file, because the reference
library must be loaded RTLD_GLOBAL (see oracle/refheif.py).  With --check nothing is written and only the fixture files
stored under tests/golden/fixtures/ are decoded (all but examples/example.heic); the script fails if a regenerated stream
differs from the committed one.
"""
import hashlib
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
REF = "/root/reference"
OUT = os.path.join(ROOT, "tests", "golden", "streams")
STORED = os.path.join(ROOT, "tests", "golden", "fixtures")

# (reference fixture, [names of the access units in the order the reference pushes them])
FIXTURES = [
    ("examples/example.heic", ["example_primary_1280x854"]),
    ("tests/data/rainbow-451x461.heic", ["rainbow_452x462"]),
    ("fuzzing/data/corpus/hevc32.heif", ["hevc32_64x64"]),
    ("fuzzing/data/corpus/colors-with-alpha.heic", ["colors_alpha_main_64x64", "colors_alpha_aux_64x64"]),
    ("fuzzing/data/corpus/colors-no-alpha.heic", ["colors_noalpha_64x64"]),
]

CHILD = r"""
import sys
sys.path.insert(0, %r)
from oracle import refheif as rh
rh.load(); rh.register_cpu_decoder()
rh.decode_file(sys.argv[1], decoder_id="b200-oracle", threads=1)
"""


def capture(path):
    with tempfile.TemporaryDirectory() as d:
        env = dict(os.environ, B200_ORACLE_DUMP_DIR=d)
        subprocess.run([sys.executable, "-c", CHILD % ROOT, path], check=True, env=env, stdout=subprocess.DEVNULL)
        return [open(os.path.join(d, f), "rb").read() for f in sorted(os.listdir(d))]


def main():
    check = "--check" in sys.argv
    bad = 0
    for rel, names in FIXTURES:
        if check:
            path = os.path.join(STORED, os.path.basename(rel))
            if not os.path.exists(path):
                continue
        else:
            path = os.path.join(REF, rel)
        dumps = capture(path)
        # one dump per decoder instance / pushed item, in decoding order; the primary item's stream may be pushed once per
        # decode pass, so keep the first occurrence of every distinct stream
        seen, uniq = set(), []
        for b in dumps:
            h = hashlib.md5(b).hexdigest()
            if h not in seen:
                seen.add(h); uniq.append(b)
        if len(uniq) < len(names):
            raise SystemExit(f"{rel}: expected {len(names)} access units, captured {len(uniq)}")
        for name, data in zip(names, uniq):
            dst = os.path.join(OUT, name + ".au")
            if check:
                same = os.path.exists(dst) and open(dst, "rb").read() == data
                print(("ok   " if same else "DIFF ") + name, len(data), hashlib.md5(data).hexdigest())
                bad += not same
            else:
                open(dst, "wb").write(data)
                print("wrote", dst, len(data))
    if bad:
        raise SystemExit(f"{bad} stream(s) differ from the committed fixtures")


if __name__ == "__main__":
    main()
