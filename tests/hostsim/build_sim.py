"""Builds tests/hostsim/libb2t_hostsim.so: the tracker, NMS, pre-processing, camera-motion and ReID glue kernels compiled by g++ against the fiber
simulator (cuda_sim.h).  TEST INFRASTRUCTURE ONLY -- see cuda_sim.h.  The product never loads it."""
import hashlib
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
CSRC = os.path.join(ROOT, "yolov7-tracker_b200", "csrc")
LIB = os.path.join(HERE, "libb2t_hostsim.so")


def _digest():
    h = hashlib.sha1()
    for d in (CSRC, HERE, os.path.join(ROOT, "include")):
        for n in sorted(os.listdir(d)):
            if n.endswith((".cu", ".cuh", ".h", ".cpp", ".inc")):
                h.update(open(os.path.join(d, n), "rb").read())
    return h.hexdigest()


def build(force=False):
    stamp = LIB + ".stamp"
    dg = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read() == dg:
        return LIB
    # -ffp-contract=off: no FMA contraction, like the nvcc build's --fmad=false
    cmd = ["g++", "-O2", "-g", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-DB2T_HOSTSIM",
           "-I", HERE, "-I", CSRC, "-x", "c++", os.path.join(CSRC, "b2t_tracker.cu"), "-x", "c++", os.path.join(CSRC, "b2t_nms.cu"), "-x", "c++", os.path.join(CSRC, "b2t_preproc.cu"), "-x", "c++", os.path.join(CSRC, "b2t_gmc.cu"),
           "-x", "c++", os.path.join(CSRC, "b2t_reid.cu"),
           "-x", "c++", os.path.join(HERE, "cuda_sim.cpp"), "-o", LIB]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("hostsim build failed:\n" + r.stderr[-6000:])
    open(stamp, "w").write(dg)
    return LIB


def build_variant(name, patches, units=("b2t_tracker.cu",)):
    """A simulator build of translation units `units` (csrc file names; the tracker's by default) with source edits (a test's
    injected bug): patches = [(file, old, new)], each `old` found exactly once.  Built in a temporary directory; returns the
    library's path."""
    import shutil
    import tempfile
    h = hashlib.sha1((_digest() + repr(patches) + repr(tuple(units))).encode()).hexdigest()[:16]
    out = os.path.join(tempfile.gettempdir(), "b2t_hostsim_variants_%d" % os.getuid(), "%s_%s" % (name, h))
    lib = os.path.join(out, "lib.so")
    if os.path.exists(lib):
        return lib
    src = os.path.join(out, "pkg", "csrc")                 # b2t_tracker.cu includes ../../include/b200track.h
    shutil.rmtree(out, ignore_errors=True)
    shutil.copytree(CSRC, src)
    shutil.copytree(os.path.join(ROOT, "include"), os.path.join(out, "include"))
    for fn, old, new in patches:
        p = os.path.join(src, fn)
        s = open(p).read()
        assert s.count(old) == 1, "patch for %s: %r found %d times" % (fn, old, s.count(old))
        open(p, "w").write(s.replace(old, new))
    cmd = ["g++", "-O1", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-DB2T_HOSTSIM", "-I", HERE, "-I", src]
    for u in units:
        cmd += ["-x", "c++", os.path.join(src, u)]
    cmd += ["-x", "c++", os.path.join(HERE, "cuda_sim.cpp"), "-o", lib + ".tmp"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("hostsim variant build failed:\n" + r.stderr[-6000:])
    os.replace(lib + ".tmp", lib)
    return lib


if __name__ == "__main__":
    print(build(force=True))
