"""not-gpu: the assignment solver's cases (tests/lap_cases.py) at reduced sizes on the simulator build, and the injected bugs
each of them must catch.  The H100 tier (tests/test_gpu_lap.py) runs the same cases at full size."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(__file__), "hostsim"))
import build_sim  # noqa: E402
import simlib  # noqa: E402
from b200track import _lib as L  # noqa: E402
import lap_cases as LC  # noqa: E402


class SimBackend:
    def __init__(self, lib):
        self.lib = lib

    def dev(self, a):
        return np.array(a, copy=True)

    ptr = staticmethod(simlib.ptr)

    def host(self, a):
        return a

    def sync(self):
        pass


@pytest.mark.parametrize("dtype", [L.F64, L.F32], ids=["f64", "f32"])
@pytest.mark.parametrize("case", sorted(LC.CASES))
def test_lap_case(case, dtype):
    rep = LC.CASES[case](SimBackend(simlib.sim()), dtype, False)
    print("%s[%s]: %s" % (case, "f64" if dtype == L.F64 else "f32", rep.line()))


def test_version():
    assert simlib.sim().b2t_version() == 107


# Injected bugs: (name, [(old, new) edits of csrc/b2t_lap.cuh], the case that must fail, its dtype)
BUGS = [
    ("edge_rule_no_guard", [("(double)thresh - (double)c > wup32(rs[i]) + wup32(cs[j])",
                             "(double)thresh - (double)c > (double)wval32(rs[i]) + (double)wval32(cs[j])")], "threshold_pairs", L.F64),
    ("previous_rule_f32", [("(double)thresh - (double)c > wup32(rs[i]) + wup32(cs[j])",
                            "thresh - c > (T)wval32(rs[i]) + (T)wval32(cs[j]) + (T)2e-6f"),
                           ("(double)thresh - (double)c1 > wup32(wkey32((float)w2)) + wup32(cs[j1])",
                            "w1 > w2 + (T)wval32(cs[j1]) + (T)2e-6f")], "regression", L.F32),
    ("w2_accepts_straddler", [("return st >= w2_base && st + cnt <= w2_end;", "return st >= w2_base && st < w2_end;")], "storage", L.F64),
    ("entry_s_cap_strict", [("sm_ok = st <= e && e < en && en <= s_cap;", "sm_ok = st <= e && e < en && en < s_cap;")], "storage", L.F64),
    ("retry_skipped_single", [("if (nq1 > 0) {", "if (nq1 > 1) {")], "single_retry", L.F64),
    ("dual_sign_u", [("if (yi >= 0) w.u[yi] = w.u[yi] + d;", "if (yi >= 0) w.u[yi] = w.u[yi] - d;")], "negative_costs", L.F64),
    ("key_zero_is_no_edge", [("return k ? k : 1u;", "return k;")], "tiny_weights", L.F64),
]


@pytest.mark.parametrize("name,edits,case,dtype", BUGS, ids=[b[0] for b in BUGS])
def test_injected_bug_is_caught(name, edits, case, dtype):
    lib = L.declare(C.CDLL(build_sim.build_variant("lap_" + name, [("b2t_lap.cuh", a, b) for a, b in edits])), names=L.TRACKER_SYMBOLS)
    with pytest.raises(AssertionError) as ei:
        LC.CASES[case](SimBackend(lib), dtype, False)
    print("%s: caught by %s: %s" % (name, case, str(ei.value).splitlines()[0][:200]))
