"""Builds libb200track.so (H100, sm_90a) in-tree with nvcc.  ``python yolov7-tracker_b200/build.py``.

The library is a git-ignored build product.  nvcc cross-compiles without a GPU, so this also runs on a
machine without one (``__graft_entry__.build()`` calls it).
"""
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "b200track", "libb200track.so")

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC"]

# (source, extra flags).  The tracker TU is built without FMA contraction so that its fp64
# arithmetic matches NumPy's separate multiply / add bit for bit (csrc/b2t_iou.cuh).
UNITS = [
    ("b2t_tracker.cu", ["--fmad=false"]),
    ("b2t_conv.cu", []),
    ("b2t_detect.cu", []),
    ("b2t_nms.cu", []),
    ("b2t_preproc.cu", ["--fmad=false"]),
    ("b2t_gmc.cu", ["--fmad=false"]),
    ("b2t_ecc.cu", ["--fmad=false"]),
    ("b2t_reid.cu", []),
    ("b2t_osnet.cu", ["--fmad=false"]),
]


def _sources_digest():
    h = hashlib.sha1()
    for root in (CSRC, os.path.join(os.path.dirname(HERE), "include")):
        for name in sorted(os.listdir(root)):
            if name.endswith((".cu", ".cuh", ".h", ".cpp", ".inc")):
                with open(os.path.join(root, name), "rb") as f:
                    h.update(name.encode())
                    h.update(f.read())
    h.update(" ".join(ARCH + COMMON + [u for _, fl in UNITS for u in fl]).encode())
    return h.hexdigest()


def build(force=False, verbose=False):
    """Compile every translation unit and link the shared library.  Returns the library path."""
    stamp = LIB + ".stamp"
    digest = _sources_digest()
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read() == digest:
        return LIB
    objs = []
    bdir = os.path.join(HERE, "build")
    os.makedirs(bdir, exist_ok=True)
    for src, extra in UNITS:
        obj = os.path.join(bdir, src.replace(".cu", ".o"))
        cmd = [NVCC] + ARCH + COMMON + extra + ["-Xptxas", "-v"] * int(verbose) + ["-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            print(" ".join(cmd))
        r = subprocess.run(cmd, capture_output=True, text=True)
        if verbose:
            print(r.stderr)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
        objs.append(obj)
    cmd = [NVCC] + ARCH + ["-shared", "-o", LIB] + objs + ["-lcudart"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    with open(stamp, "w") as f:
        f.write(digest)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
