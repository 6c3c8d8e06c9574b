"""Build libb200heif.so in-tree with nvcc for sm_90a (H100) (called by __graft_entry__.build() and by `python -m libheif_b200.build`)."""
import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libb200heif.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "--fmad=false",
         "-Xcompiler", "-fPIC,-ffp-contract=off,-O2,-pthread", "-Xptxas", "-v"]


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.cc")))


def needs_build():
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    deps = sources() + glob.glob(os.path.join(CSRC, "*.h")) + glob.glob(os.path.join(HERE, "..", "include", "*.h"))
    return any(os.path.getmtime(p) > t for p in deps)


def build(force=False, verbose=False, extra_flags=None, out=None, tag=""):
    global OUT
    if out:
        OUT_local = out
    else:
        OUT_local = OUT
    if not force and not extra_flags and not needs_build():
        return OUT
    objs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    procs = []
    for src in sources():
        obj = os.path.join(HERE, "build", os.path.basename(src) + tag + ".o")
        objs.append(obj)
        if not force and os.path.exists(obj) and os.path.getmtime(obj) > max(
                [os.path.getmtime(src)] + [os.path.getmtime(h) for h in glob.glob(os.path.join(CSRC, "*.h")) + glob.glob(os.path.join(HERE, "..", "include", "*.h"))]):
            continue
        cmd = [NVCC] + FLAGS + (extra_flags or []) + ["-x", "cu", "-c", src, "-o", obj]
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for src, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode != 0:
            sys.stderr.write(out)
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}")
        with open(os.path.join(HERE, "build", os.path.basename(src) + ".ptxas.txt"), "w") as f:
            f.write(out)
    cmd = [NVCC, "-shared", "-o", OUT_local] + objs + ["-lpthread", "-ldl"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout)
        raise RuntimeError("link failed")
    return OUT_local


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
