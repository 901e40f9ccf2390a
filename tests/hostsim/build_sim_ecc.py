"""Builds tests/hostsim/libb2t_hostsim_ecc.so: the ECC camera-motion kernels (csrc/b2t_ecc.cu) compiled by g++ against the fiber
simulator (cuda_sim.h), with csrc/b2t_nms.cu for the error-reporting entry points the unit shares.  TEST INFRASTRUCTURE ONLY -- see
cuda_sim.h.  The product never loads it.  Same flags as build_sim.py (whose library holds the other simulated units)."""
import ctypes as C
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import build_sim  # noqa: E402

LIB = os.path.join(HERE, "libb2t_hostsim_ecc.so")
SYMBOLS = ["b2t_detect_last_error", "b2t_ecc_workspace_bytes", "b2t_ecc_reset", "b2t_ecc_estimate", "b2t_ecc_workspace_layout", "b2t_ecc_warp"]


def build(force=False):
    stamp = LIB + ".stamp"
    dg = build_sim._digest()
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read() == dg:
        return LIB
    # -ffp-contract=off: no FMA contraction, like the nvcc build's --fmad=false
    cmd = ["g++", "-O2", "-g", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-DB2T_HOSTSIM", "-I", HERE, "-I", build_sim.CSRC,
           "-x", "c++", os.path.join(build_sim.CSRC, "b2t_ecc.cu"), "-x", "c++", os.path.join(build_sim.CSRC, "b2t_nms.cu"),
           "-x", "c++", os.path.join(HERE, "cuda_sim.cpp"), "-o", LIB]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("hostsim (ecc) build failed:\n" + r.stderr[-6000:])
    open(stamp, "w").write(dg)
    return LIB


_lib = None


def sim_ecc():
    """The simulated ECC library with the ctypes signatures of b200track/_lib.py."""
    global _lib
    if _lib is None:
        from b200track import _lib as L
        _lib = L.declare(C.CDLL(build()), names=SYMBOLS)
    return _lib


if __name__ == "__main__":
    print(build(force=True))
