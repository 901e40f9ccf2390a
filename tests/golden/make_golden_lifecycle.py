"""Writes tests/golden/loop_lifecycle.npz by running the UNMODIFIED reference trackers from /root/reference on
``synth.lifecycle_stream`` streams (build container only: ``python tests/golden/make_golden_lifecycle.py``).  The reference
modules come in through oracle/refshim.py, as in make_golden.py.

Per configuration ``<c>`` (CONFIGS below; ``<c>_params`` = seed, n_obj, n_frames, conf_thresh, track_buffer, frame_rate,
warp_sigma; ``<c>_kind`` / ``<c>_fmt``), per frame, ragged arrays with a per-frame count:
  <c>_out_{n,ids,cls,tlwh}      the tracks ``update`` returns: id, cls, tlwh (float64)
  <c>_trk_{n,rows,tlwh}         ``tracked_stracks`` in list order: rows = id, state, is_activated, start_frame, frame_id,
                                tracklet_len; tlwh of each
  <c>_lost_{n,rows,tlwh}        ``lost_stracks``, same columns
  <c>_tlwh_frames               the (0-based) frames whose tlwh the three *_tlwh arrays hold: every 4th and the last, to keep
                                the file small; ids, counts and the integer columns are stored for every frame
  <c>_rem_{n,ids}               the ids appended to ``removed_stracks`` during the frame, in order (the list only grows)
  <c>_digest                    sha1 of the stream
  <c>_events                    EVENTS, counted on the reference run
NSA Kalman paths (NSAKalmanFilter, with a float32 confidence): nsa_z0 / nsa_conf0 -> nsa_init_{mean,cov};
project from the float32 initiate mean (nsa_proj32_{mean,cov}); update from it (nsa_z1 -> nsa_upd32_{mean,cov});
multi_predict, then project / update from the float64 mean with nsa_conf1 (nsa_proj64_*, nsa_z2 -> nsa_upd64_*).
"""
import os
import sys

import numpy as np
import scipy

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "yolov7-tracker_b200"))

from oracle import refshim                                  # noqa: E402
from b200track.synth import lifecycle_stream, stream_digest  # noqa: E402

VERS = dict(numpy=np.__version__, scipy=scipy.__version__)
N_OBJ, N_FRAMES = 40, 200

# (name, kind, kalman_format, conf_thresh, track_buffer, frame_rate)
CONFIGS = [("%s_%s" % (k, f), k, f, 0.2, 30, 30) for k in ("sort", "bytetrack", "botsort")
           for f in ("default", "botsort", "strongsort")] + [
    ("bytetrack_c06_tb5_fr25", "bytetrack", "default", 0.6, 5, 25),
    ("sort_c04_tb8", "sort", "default", 0.4, 8, 30),
    ("botsort_c01_tb10", "botsort", "botsort", 0.1, 10, 30),
    ("bytetrack_nsa_c03_tb12_fr20", "bytetrack", "strongsort", 0.3, 12, 20),
]
EVENTS = ("prunes", "reactivated_after_10", "duplicate_drops", "empty_frames", "threshold_ties", "births")


def _warp_sigma(kind):
    return 2.0 if kind == "botsort" else 0.0


def _rows(tracks):
    rows = np.array([[t.track_id, t.state, int(t.is_activated), t.start_frame, t.frame_id, t.tracklet_len] for t in tracks],
                    np.int32).reshape(-1, 6)
    tlwh = np.array([np.asarray(t.tlwh, np.float64) for t in tracks]).reshape(-1, 4)
    return rows, tlwh


def run_config(ref, name, kind, fmt, conf, tb, fr, seed):
    ws = _warp_sigma(kind)
    frames, warps = lifecycle_stream(seed, N_FRAMES, N_OBJ, conf_thresh=conf, warp_sigma=ws)
    ref.basetrack.BaseTrack._count = 0
    opts = refshim.Opts(conf_thresh=conf, track_buffer=tb, kalman_format=fmt)
    if kind == "sort":
        trk, mod = ref.basetrack.BaseTracker(opts, frame_rate=fr), ref.basetrack
    elif kind == "bytetrack":
        trk, mod = ref.bytetrack.ByteTrack(opts, frame_rate=fr), ref.bytetrack
    else:
        trk, mod = ref.botsort.BoTSORT(opts, frame_rate=fr), ref.botsort
        trk.gmc = refshim.FixedGMC(warps)
    # count what remove_duplicate_stracks drops: a pass-through wrapper around the module's own function
    dups = [0]
    orig = mod.remove_duplicate_stracks

    def counted(a, b):
        ra, rb = orig(a, b)
        dups[0] += len(a) + len(b) - len(ra) - len(rb)
        return ra, rb

    mod.remove_duplicate_stracks = counted
    img = np.zeros((4, 4, 3), np.uint8)
    rec = {k: [] for k in ("out_n", "out_ids", "out_tlwh", "out_cls", "trk_n", "trk_rows", "trk_tlwh", "lost_n", "lost_rows",
                           "lost_tlwh", "rem_n", "rem_ids")}
    prunes = react = 0
    removed_ever = set()
    try:
        for f, dets in enumerate(frames, 1):
            lost_before = [(t, t.frame_id) for t in trk.lost_stracks]
            n_rem = len(trk.removed_stracks)
            cur = trk.update(dets.copy(), img)
            rec["out_n"].append(len(cur))
            rec["out_ids"] += [t.track_id for t in cur]
            keep_tlwh = f % 4 == 0 or f == len(frames)
            if keep_tlwh:
                rec["out_tlwh"] += [np.asarray(t.tlwh, np.float64) for t in cur]
            rec["out_cls"] += [float(t.cls) for t in cur]
            for key, lst in (("trk", trk.tracked_stracks), ("lost", trk.lost_stracks)):
                rows, tlwh = _rows(lst)
                rec[key + "_n"].append(len(lst))
                rec[key + "_rows"].append(rows)
                if keep_tlwh:
                    rec[key + "_tlwh"].append(tlwh)
            new_rem = trk.removed_stracks[n_rem:]
            rec["rem_n"].append(len(new_rem))
            rec["rem_ids"] += [t.track_id for t in new_rem]
            for t in new_rem:                     # a pruned track was confirmed; an unconfirmed one never was
                if t.is_activated and t.track_id not in removed_ever:
                    prunes += 1
                removed_ever.add(t.track_id)
            react += sum(1 for t, fid in lost_before if t.state == 1 and t.frame_id == f and f - fid >= 10)
    finally:
        mod.remove_duplicate_stracks = orig
    ties = np.array([conf, max(0.15, conf - 0.3), conf + 0.1], np.float32)
    events = [prunes, react, dups[0], sum(len(d) == 0 for d in frames),
              sum(int(np.isin(d[:, 4], ties).sum()) for d in frames), ref.basetrack.BaseTrack._count]
    out = {"digest": stream_digest(frames), "kind": kind, "fmt": fmt,
           "tlwh_frames": np.array([i for i in range(N_FRAMES) if i % 4 == 3 or i == N_FRAMES - 1], np.int32),
           "params": np.array([seed, N_OBJ, N_FRAMES, conf, tb, fr, ws], np.float64),
           "events": np.array(events, np.int64),
           "out_n": np.array(rec["out_n"], np.int32), "out_ids": np.array(rec["out_ids"], np.int32),
           "out_tlwh": np.array(rec["out_tlwh"]).reshape(-1, 4), "out_cls": np.array(rec["out_cls"], np.float32),
           "rem_n": np.array(rec["rem_n"], np.int32), "rem_ids": np.array(rec["rem_ids"], np.int32)}
    for key in ("trk", "lost"):
        out[key + "_n"] = np.array(rec[key + "_n"], np.int32)
        out[key + "_rows"] = np.concatenate(rec[key + "_rows"])
        out[key + "_tlwh"] = np.concatenate(rec[key + "_tlwh"])
    print("%-28s" % name, dict(zip(EVENTS, events)))
    return {"%s_%s" % (name, k): v for k, v in out.items()}


def nsa_fixture(ref, n=64, seed=17):
    rng = np.random.default_rng(seed)
    kf = ref.kalman_filter.NSAKalmanFilter()
    z0 = np.stack([rng.uniform(0, 1280, n), rng.uniform(0, 1280, n), rng.uniform(0.2, 2.0, n), rng.uniform(4, 300, n)],
                  1).astype(np.float32)
    out = {"nsa_z0": z0}
    for k in range(3):
        out["nsa_conf%d" % k] = rng.uniform(0.1, 0.95, n).astype(np.float32)
    z1 = (z0 + rng.normal(0, 1.0, z0.shape) * np.array([1, 1, 0.01, 1])).astype(np.float32)
    z2 = (z1 + rng.normal(0, 1.0, z0.shape) * np.array([1, 1, 0.01, 1])).astype(np.float32)
    out["nsa_z1"], out["nsa_z2"] = z1, z2
    m0, c0 = zip(*[kf.initiate(z) for z in z0])
    assert all(m.dtype == np.float32 for m in m0)
    out["nsa_init_mean"], out["nsa_init_cov"] = np.stack(m0), np.stack(c0)
    pm, ps = zip(*[kf.project(m, c, s) for m, c, s in zip(m0, c0, out["nsa_conf0"])])
    out["nsa_proj32_mean"], out["nsa_proj32_cov"] = np.stack(pm), np.stack(ps)
    um, uc = zip(*[kf.update(m, c, z, s) for m, c, z, s in zip(m0, c0, z1, out["nsa_conf0"])])
    out["nsa_upd32_mean"], out["nsa_upd32_cov"] = np.stack(um), np.stack(uc)
    mp, cp = kf.multi_predict(np.stack(um), np.stack(uc))
    out["nsa_pred_mean"], out["nsa_pred_cov"] = mp, cp
    pm, ps = zip(*[kf.project(m, c, s) for m, c, s in zip(mp, cp, out["nsa_conf1"])])
    out["nsa_proj64_mean"], out["nsa_proj64_cov"] = np.stack(pm), np.stack(ps)
    um, uc = zip(*[kf.update(m, c, z, s) for m, c, z, s in zip(mp, cp, z2, out["nsa_conf2"])])
    out["nsa_upd64_mean"], out["nsa_upd64_cov"] = np.stack(um), np.stack(uc)
    return out


def main():
    ref = refshim.load()
    out = {"configs": np.array([c[0] for c in CONFIGS]), "events": np.array(EVENTS)}
    for i, (name, kind, fmt, conf, tb, fr) in enumerate(CONFIGS):
        out.update(run_config(ref, name, kind, fmt, conf, tb, fr, seed=300 + i))
    out.update(nsa_fixture(ref))
    np.savez_compressed(os.path.join(HERE, "loop_lifecycle.npz"), **out, **{"ver_" + k: v for k, v in VERS.items()})


if __name__ == "__main__":
    main()
