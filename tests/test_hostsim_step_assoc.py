"""not-gpu: every association of the fused step certified frame by frame (tests/assoc_bounds.py) under the host simulator -- on step
cases of every kind (UAVMOT included) and on short crowded streams whose association 1 lists more edges than shared memory can hold,
so that rows live in the mirror, the second window and the global edge workspace; the certifier's soundness on the float64 oracles'
own matchings; and injected bugs in the association costs, each of which must fail in the certifier while the clean build passes."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "hostsim"))
import build_sim  # noqa: E402
from simlib import sim  # noqa: E402
from b200track import _lib as L  # noqa: E402
from b200track.synth import make_reid_stream, make_strongsort_stream, make_stream  # noqa: E402
import assoc_bounds as AB  # noqa: E402
import step_bounds as SB  # noqa: E402
from test_hostsim_kalman_bounds import SimStep  # noqa: E402

CROWD_FRAMES = 4


def run(lib, case, dtype, stats=None, n_frames=None):
    """step_bounds plus the certifier over a step case ('name') or a crowded stream ('crowd_<name>'); returns the certifier"""
    f32 = dtype == "f32"
    if case.startswith("crowd_"):
        kind, fmt, frames, feats, warps, kw = AB.crowd_case(case[6:], n_frames or CROWD_FRAMES)
    else:
        kind, fmt, frames, feats, warps, kw = SB.case(case)
        if n_frames:
            frames, feats, warps = frames[:n_frames], None if feats is None else feats[:n_frames], None if warps is None else warps[:n_frames]
    trk = SimStep(lib, kind, fmt, L.F32 if f32 else L.F64, **kw)
    cert = AB.Certifier(kind, L.FMT_BY_NAME[fmt], f32, conf_thresh=kw.get("conf_thresh", 0.2), stats={} if stats is None else stats)
    nearest = 10 ** 6 if kind == "strongsort" and case.startswith("crowd_") else (16 if case.startswith("crowd_") else SB.NEAREST)
    SB.check_stream(trk, frames, warps, kind, L.FMT_BY_NAME[fmt], f32, {}, case, feats, kw.get("conf_thresh", 0.2), on_frame=cert,
                    nearest=nearest)
    return cert


@pytest.mark.parametrize("case,dtype", [("bytetrack_default", "f32"), ("sort_c04_tb8", "f64"), ("botsort_botsort", "f32"),
                                        ("bytetrack_nsa_c03_tb12_fr20", "f64"), ("feat_botsort", "f32"), ("feat_botsort", "f64"),
                                        ("feat_strongsort", "f32"), ("feat_strongsort", "f64"), ("uavmot", "f64")])
def test_step_case_associations_certify(case, dtype):
    st = {}
    cert = run(sim(), case, dtype, st, n_frames=30)
    assert st["assoc1"]["pairs"] > 0 and cert.frames == 30, st
    print("\n%s %s: %s" % (case, dtype, AB.report(st)))


@pytest.mark.parametrize("case,dtype", [("crowd_reid", "f64"), ("crowd_reid", "f32"), ("crowd_strongsort", "f64"),
                                        ("crowd_strongsort", "f32"), ("crowd_uavmot", "f64"), ("crowd_bytetrack", "f32"),
                                        ("crowd_botsort", "f32")])
def test_crowded_stream_spills_and_certifies(case, dtype):
    """association 1 lists more edges than 227 KB of mirror and second window can hold on every frame after the first"""
    st = {}
    cert = run(sim(), case, dtype, st)
    bound = AB.spill_bound(dtype == "f32")
    assert all(e > bound for e in cert.edges[1:]), "association-1 edges per frame %s, spill bound %d" % (cert.edges, bound)
    print("\n%s %s: edges %s; %s" % (case, dtype, cert.edges, AB.report(st)))


# ---------------------------------------------------------------- soundness on the float64 oracles
def _recorded(monkeypatch, module):
    """record every (cost, thresh, (matches, unmatched rows, unmatched cols)) of the oracle module's linear_assignment"""
    seen = []
    orig = module.linear_assignment

    def la(cost, thresh):
        r = orig(cost, thresh)
        seen.append((np.asarray(cost, np.float64).copy(), thresh, np.asarray(r[0]).reshape(-1, 2)))
        return r
    monkeypatch.setattr(module, "linear_assignment", la)
    return seen


def _oracle_runs(monkeypatch):
    import reid_track_oracle as RO
    import strongsort_oracle as SO
    import uavmot_oracle as UO
    out = []
    seen = _recorded(monkeypatch, RO)
    frames, feats, warps = make_reid_stream(5, 12, 60, 64)
    o = RO.ReidBotsortOracle()
    for f, fe, w in zip(frames, feats, warps):
        o.update(f, w, fe)
    out.append(("reid", list(seen)))
    seen = _recorded(monkeypatch, SO)
    frames, feats, warps = make_strongsort_stream(17, 12, 40, 64)
    o = SO.StrongSortOracle()
    for f, fe, w in zip(frames, feats, warps):
        o.update(f, fe, w)
    out.append(("strongsort", list(seen)))
    seen = _recorded(monkeypatch, UO)
    frames, _ = make_stream(9, 12, 80, img=640)
    o = UO.UavmotOracle()
    for f in frames:
        o.update(f)
    out.append(("uavmot", list(seen)))
    return out


def _iv(cost):
    return np.nextafter(cost, -np.inf), np.nextafter(cost, np.inf)


def test_oracle_matchings_certify_and_wrong_ones_fail(monkeypatch):
    """each float64 oracle's own matchings certify; two matched columns swapped, or a sub-threshold pair left unmatched, fail"""
    swapped = dropped = 0
    for name, seen in _oracle_runs(monkeypatch):
        assert len(seen) > 20, name
        for k, (cost, t, m) in enumerate(seen):
            L, U = _iv(cost)
            what = "%s solve %d" % (name, k)
            rows, cols = list(range(cost.shape[0])), list(range(cost.shape[1]))
            pairs = [tuple(map(int, p)) for p in m]
            AB.certify(what, L, U, t, pairs, rows, cols, {})
            # two matched columns swapped: a strictly worse matching (or a pair over the limit)
            for a in range(len(pairs)):
                for b in range(a + 1, len(pairs)):
                    (i, j), (p, q) = pairs[a], pairs[b]
                    if cost[i, q] + cost[p, j] > cost[i, j] + cost[p, q] + 1e-9:
                        bad = list(pairs)
                        bad[a], bad[b] = (i, q), (p, j)
                        with pytest.raises(AB.CertError, match=r"\((a|b)\)"):
                            AB.certify(what, L, U, t, bad, rows, cols, {})
                        swapped += 1
                        break
                else:
                    continue
                break
            if pairs:
                with pytest.raises(AB.CertError, match=r"\((b|c)\)"):
                    AB.certify(what, L, U, t, pairs[1:], rows, cols, {})
                dropped += 1
    assert swapped > 10 and dropped > 20, (swapped, dropped)


# ---------------------------------------------------------------- injected bugs fail in the certifier
BUGS = {
    # BoT-SORT with ReID: App without its factor 0.5 (twice the cosine distance)
    "reid_app_half_dropped": ("b2t_step.cuh", "T app_d = (T)0.5 * ((T)1 - ab / (sqrt(aa) * sqrt(bb)));",
                              "T app_d = ((T)1 - ab / (sqrt(aa) * sqrt(bb)));"),
    # StrongSORT: gamma on the appearance distance, 1 - gamma on the IoU distance
    "strongsort_gamma_swapped": ("b2t_step.cuh", "return g * iou_d + g1 * app;", "return g1 * iou_d + g * app;"),
    # UAVMOT: the pool's structure vectors taken for the detections and the other way round
    "uavmot_sv_swapped": ("b2t_step.cuh", "const StructCtx sc = {sv_t, sv_d};", "const StructCtx sc = {sv_d, sv_t};"),
    # the second edge window: each cost copied from the next edge
    "window_shifted": ("b2t_step.cuh", "wc[e - w2_base] = c.v.e_cost[e];", "wc[e - w2_base] = c.v.e_cost[e + 1];"),
}


BUG_FRAMES = {"crowd_uavmot": 6}       # S weighs 0.02: the swapped vectors first change a matching at frame 5


def _variant(name):
    fn, old, new = BUGS[name]
    return L.declare(C.CDLL(build_sim.build_variant(name, [(fn, old, new)])), names=L.TRACKER_SYMBOLS)


@pytest.mark.parametrize("bug,case,dtype", [("reid_app_half_dropped", "crowd_reid", "f64"),
                                            ("strongsort_gamma_swapped", "feat_strongsort", "f32"),
                                            ("uavmot_sv_swapped", "crowd_uavmot", "f64"),
                                            ("window_shifted", "crowd_bytetrack", "f32")])
def test_injected_association_bug_fails_in_certifier(bug, case, dtype):
    """the bug fails the certificate (not the Kalman check) at some frame; the clean build passes the same frames"""
    with pytest.raises(AB.CertError, match=r"frame \d+") as e:
        run(_variant(bug), case, dtype, n_frames=30 if not case.startswith("crowd_") else BUG_FRAMES.get(case))
    frame = int(str(e.value).split(" frame ")[1].split(":")[0].split(" ")[0])
    run(sim(), case, dtype, n_frames=frame)
    print("\n%s: %s" % (bug, str(e.value)[:300]))
