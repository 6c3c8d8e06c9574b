"""Records tests/golden/gpu_encoder_md5.json: the md5 of GpuEncoder.encode's access unit for seeded pictures of the
conformance matrix (tests/test_hevc_gpu_encoder.py CONF) plus the QP 0 noise worst case at CTB 64, coded with the default
parameters.  The file was written by the encoder that had a single mode search (all 35 modes, closed loop); the speed tests
pin that the default parameters and speed=0 still produce these bytes.  Needs a CUDA device:

    python tests/golden/make_gpu_encoder_md5.py [--check]
"""
import hashlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]
OUT = os.path.join(HERE, "gpu_encoder_md5.json")


def cases():
    """(id, (w, h, chroma, log2ctb, qp, source kind, extra params)) of every recorded picture."""
    from test_hevc_gpu_encoder import CONF
    out = [(f"conf{i}-{c[0]}x{c[1]}-{'420' if c[2] else '400'}-ctb{1 << c[3]}-qp{c[4]}-{c[5]}", c) for i, c in enumerate(CONF)]
    out.append(("noise-256x128-420-ctb64-qp0", (256, 128, True, 6, 0, "noise", {})))
    return out


def encode(enc, case, **params):
    from test_hevc_gpu_encoder import source
    w, h, chroma, log2ctb, qp, kind, extra = case
    return enc.encode([tuple(source(kind, w, h, chroma))], log2_ctb_size=log2ctb, qp=qp, **extra, **params)[0]


def main():
    from libheif_b200.hevc_enc import GpuEncoder
    enc = GpuEncoder()
    got = {cid: hashlib.md5(encode(enc, c)).hexdigest() for cid, c in cases()}
    enc.close()
    if "--check" in sys.argv:
        with open(OUT) as f:
            want = json.load(f)
        bad = [k for k in want if got.get(k) != want[k]]
        print("differ:", bad if bad else "none")
        return 1 if bad else 0
    with open(OUT, "w") as f:
        json.dump(got, f, indent=1, sort_keys=True)
        f.write("\n")
    print(json.dumps(got))
    return 0


if __name__ == "__main__":
    sys.exit(main())
