"""-m gpu: every association of the fused step on an H100 certified frame by frame (tests/assoc_bounds.py) together with the Kalman
side (tests/step_bounds.py): every step case in float32 and float64 (UAVMOT in float64), and crowded streams whose association 1 lists
more edges than 227 KB of shared memory can hold -- BoT-SORT with ReID and StrongSORT in both dtypes, UAVMOT in float64, ByteTrack
and BoT-SORT in float32 -- so that rows live in the mirror, the second window and the global edge workspace.  In float64 the crowded
ReID, StrongSORT and UAVMOT streams also give exactly the oracles' ids and boxes within 1e-9.  Four sequences in one launch, only some
of them crowded, give each sequence's output bit for bit as that sequence run alone.  Prints the largest interval width and smallest
slack per association.  Nothing here reads the reference tree."""
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from b200track import _lib as L  # noqa: E402
import assoc_bounds as AB  # noqa: E402
import step_bounds as SB  # noqa: E402

CROWD_FRAMES = 8


class Adapter:
    """TrackEngine (one sequence) with the reads step_bounds needs; check(res, dets, feats, warp), when given, sees every step"""

    def __init__(self, eng, check=None):
        self.eng, self.check = eng, check

    def step(self, dets, fe, warp):
        w = None if warp is None else np.asarray(warp).reshape(1, 6)
        d = torch.as_tensor(np.asarray(dets, np.float32).reshape(-1, 6), device="cuda:0")
        if fe is None:
            res = self.eng.step_cuda_dets([d], w)[0].copy()
        else:
            f = torch.as_tensor(np.ascontiguousarray(fe, np.float32), device="cuda:0")
            res = self.eng.step_cuda_dets([d], w, feats_list=[f])[0].copy()
        if self.check is not None:
            self.check(res, dets, fe, warp)
        return res

    @property
    def stat(self):
        return self.eng.np_stat[0]

    def read_slot(self, slot):
        return self.eng.read_slot(0, slot)

    def read_list(self, which):
        return self.eng.read_list(0, "tracked" if which == 0 else "lost")

    def read_feature(self, slot):
        return self.eng.read_feature(0, slot)


def _engine(kind, fmt, dtype, kw, n_seq=1):
    from b200track.engine import TrackEngine
    kw = dict(kw)
    return TrackEngine(kind, n_seq=n_seq, dtype=dtype, cap=kw.pop("cap", 256), dmax=kw.pop("dmax", 256), ecap=kw.pop("ecap", None),
                       kalman_format=fmt, device="cuda:0", **kw)


def _certify(case, dtype, kind, fmt, frames, feats, warps, kw, check=None, nearest=SB.NEAREST):
    f32 = dtype == "f32"
    eng = _engine(kind, fmt, dtype, kw)
    st = {}
    cert = AB.Certifier(kind, L.FMT_BY_NAME[fmt], f32, conf_thresh=kw.get("conf_thresh", 0.2), stats=st)
    counts = SB.check_stream(Adapter(eng, check), frames, warps, kind, L.FMT_BY_NAME[fmt], f32, {}, case, feats,
                             kw.get("conf_thresh", 0.2), on_frame=cert, nearest=nearest)
    print("\n%s %s: edges max %d; %s" % (case, dtype, max(cert.edges), AB.report(st)))
    return cert, counts, st


@pytest.mark.parametrize("name,dtype", SB.step_cases())
def test_step_case_associations_certify(name, dtype):
    kind, fmt, frames, feats, warps, kw = SB.case(name)
    cert, counts, st = _certify(name, dtype, kind, fmt, frames, feats, warps, kw)
    assert counts["update"] and st["assoc1"]["pairs"] > 0 and cert.frames == len(frames)


def _oracle(kind, feats):
    if kind == "strongsort":
        from strongsort_oracle import StrongSortOracle
        o = StrongSortOracle(gamma=0.1)
        return lambda f, fe, w: o.update(f, fe, w)
    if kind == "uavmot":
        from uavmot_oracle import UavmotOracle
        o = UavmotOracle()
        return lambda f, fe, w: o.update(f)
    from reid_track_oracle import ReidBotsortOracle
    o = ReidBotsortOracle()
    return lambda f, fe, w: o.update(f, w, fe)


@pytest.mark.parametrize("name,dtype", [("reid", "f64"), ("reid", "f32"), ("strongsort", "f64"), ("strongsort", "f32"), ("uavmot", "f64"),
                                        ("bytetrack", "f32"), ("botsort", "f32")])
def test_crowded_stream_spills_and_certifies(name, dtype):
    """stat word 15 beyond 227 KB / (8 + sizeof T) edges on every frame after the first; in float64 the kinds with appearance or
    structure costs also match their oracle's ids exactly and its boxes within 1e-9"""
    kind, fmt, frames, feats, warps, kw = AB.crowd_case(name, CROWD_FRAMES)
    check = None
    if dtype == "f64" and name in ("reid", "strongsort", "uavmot"):
        orc = _oracle(kind, feats)
        n = [0]

        def check(res, dets, fe, warp):
            n[0] += 1
            exp = orc(dets, fe, None if warp is None else np.asarray(warp).reshape(2, 3))
            assert res[:, 0].astype(int).tolist() == [e[0] for e in exp], "%s frame %d: ids" % (name, n[0])
            if exp:
                np.testing.assert_allclose(res[:, 1:5], np.array([e[1] for e in exp]), rtol=1e-9, atol=1e-9,
                                           err_msg="%s frame %d" % (name, n[0]))
    cert, counts, st = _certify("crowd_" + name, dtype, kind, fmt, frames, feats, warps, kw, check,
                                nearest=10 ** 6 if kind == "strongsort" else 16)
    bound = AB.spill_bound(dtype == "f32")
    assert all(e > bound for e in cert.edges[1:]), "association-1 edges per frame %s, spill bound %d" % (cert.edges, bound)


@pytest.mark.parametrize("name", ["reid", "strongsort", "uavmot"])
def test_batched_sequences_match_each_alone(name):
    """four sequences in one launch -- two crowded (spilling), two small -- give each sequence's rows bit for bit as it gives alone:
    e_app, the structure scratch and the edge workspace are per-sequence offsets"""
    from b200track.synth import make_reid_stream
    kind, fmt, _, _, _, kw = AB.crowd_case(name, 1)
    D = kw["feat_dim"]
    seqs = []
    for s in range(4):
        if s % 2 == 0:
            _, _, fr, fe, wp, _ = AB.crowd_case(name, 6, seed=300 + s)
        else:
            fr, fe, wp = make_reid_stream(400 + s, 6, 30, max(D, 4))
        seqs.append((fr, fe if D else None, wp))
    alone = []
    for fr, fe, wp in seqs:
        eng = _engine(kind, fmt, "f64", kw)
        rows = []
        for i in range(len(fr)):
            w = None if kind == "uavmot" else wp[i].reshape(1, 6)
            d = [torch.as_tensor(fr[i], device="cuda:0")]
            f = None if fe is None else [torch.as_tensor(np.ascontiguousarray(fe[i]), device="cuda:0")]
            rows.append(eng.step_cuda_dets(d, w, feats_list=f)[0].copy())
            assert eng.np_stat[0, L.STAT_ERR] == 0
        alone.append(rows)
    eng = _engine(kind, fmt, "f64", kw, n_seq=4)
    spilled = [0] * 4
    for i in range(6):
        w = None if kind == "uavmot" else np.stack([sq[2][i].reshape(6) for sq in seqs])
        d = [torch.as_tensor(sq[0][i], device="cuda:0") for sq in seqs]
        f = None if not D else [torch.as_tensor(np.ascontiguousarray(sq[1][i]), device="cuda:0") for sq in seqs]
        got = eng.step_cuda_dets(d, w, feats_list=f)
        for s in range(4):
            assert eng.np_stat[s, L.STAT_ERR] == 0
            spilled[s] = max(spilled[s], int(eng.np_stat[s, 15]))
            assert np.array_equal(got[s], alone[s][i]), "%s sequence %d frame %d differs from the sequence alone" % (name, s, i + 1)
    bound = AB.spill_bound(False)
    assert spilled[0] > bound and spilled[2] > bound and spilled[1] < bound and spilled[3] < bound, spilled
