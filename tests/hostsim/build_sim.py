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


if __name__ == "__main__":
    print(build(force=True))
