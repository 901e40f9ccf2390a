"""TEST INFRASTRUCTURE: the fused step's arithmetic checked frame by frame from its own stored state, against tests/kalman_ref.py,
shared by the GPU tier (TrackEngine) and the CPU tier (the simulator's ctypes tracker).  A tracker adapter offers
step(dets, feats, warp) -> output rows, read_slot(slot) -> (mean (8,), cov (8, 8)), read_list(which) -> rows of 13 columns (id,
tlwh, cls, score, slot, state, is_activated, tracklet_len, start_frame, frame_id; which 0 = tracked, 1 = lost) and, for trackers
with appearance features, read_feature(slot).

Before and after every step every live slot is read.  Each slot live after the step must lie, within the bound, on one of the paths
its kind allows (b2t_step.cuh; oracle/trackers.py, tests/strongsort_oracle.py):
  * pool slots (Tracked and activated, or Lost): kf_predict with mean[7] zeroed when the slot was not Tracked, the process noise in
    float32 when every pool mean is still float32 (q_f32), then kf_gmc for BoT-SORT with a warp -- StrongSORT warps first and then
    predicts in float64 -- and then either nothing more (unmatched) or kf_update with one of this frame's detections;
  * unconfirmed slots (Tracked, not activated): kf_gmc for BoT-SORT with a warp, or nothing, then optionally kf_update;
  * slots born this frame: kf_initiate from one detection.
kf_update takes the detection's measurement (det_to_meas), the float32-mean flag the step holds for the slot and, for the NSA
format, the detection's score as confidence when the slot was Tracked (STrack.update) and none when it was Lost (re_activate).  The
flag is not read from the tracker: it is restated -- set on a birth, cleared by the first predict, warp or update -- so a step that
passes the wrong flag fails.  Exactly one detection may put a slot within the bound.  Every output row's tlwh is mean_to_tlwh of
its slot's new mean with that flag, and every feature is the float32 EMA of STrack.update_features (basetrack.py:323-332) of the
stored feature and the matched detection's (an update of a Tracked slot by a detection with a feature: every StrongSORT detection,
BoT-SORT's high-score ones), the detection's own feature (a birth), or unchanged.
Each frame starts from the stored state, so drift cannot accumulate: the bound does not loosen with the stream's length."""
import numpy as np

import kalman_ref as R
from b200track.synth import lifecycle_stream, make_strongsort_stream

ST_TRACKED, ST_LOST = 1, 2
NEAREST = 3              # detections tried per slot: the nearest by centre (twins of the lifecycle stream sit 1 - 2 px apart)


def _snapshot(trk, feats):
    """slot -> dict(tid, state, pool, mean, cov[, feat]) for every slot on the tracked or lost list."""
    out = {}
    for which in (0, 1):
        for r in trk.read_list(which):
            s = int(r[7])
            if s in out:
                continue
            m, c = trk.read_slot(s)
            d = dict(tid=int(r[0]), state=int(r[8]), pool=which == 1 or int(r[9]) == 1, mean=m, cov=c)
            if feats:
                d["feat"] = trk.read_feature(s)
            out[s] = d
    return out


def _sel(mask, a, b):
    (ma, Pa), (mb, Pb) = a, b
    return [x.where(mask, y) for x, y in zip(ma, mb)], [[x.where(mask, y) for x, y in zip(ra, rb)] for ra, rb in zip(Pa, Pb)]


def _take(st, i):
    m, P = st
    return [x.take(i) for x in m], [[x.take(i) for x in row] for row in P]


def _within(st, gm, gc, f32):
    """per-row bool: the whole mean and covariance within the bound; and the per-row worst err / bound."""
    rm, rc = R.stack(st[0]), R.stack_cov(st[1])
    with np.errstate(over="ignore"):
        em = np.abs(gm - rm.v.astype(np.float64)) / R.bound(rm, f32)
        ec = np.abs(gc - rc.v.astype(np.float64)) / R.bound(rc, f32)
    w = np.maximum(em.max(1), ec.reshape(len(gm), -1).max(1))
    return w <= 1.0, w


def ema_ref(old, f):
    """STrack.update_features in float32 (b2t_step.cuh ema_features): B of the smoothed, renormalised feature."""
    u = R.U32 + R.U_REF
    a = R.B(np.asarray(f, np.float32), u)
    o = R.B(np.asarray(old, np.float32), u)
    nf = np.sqrt(np.sum(np.asarray(f, np.float64) ** 2))
    nfb = R.B(np.float32(nf), u, 2.01 * R.U32 * nf)                     # sum of squares in float64, rounded to float32, sqrtf
    s = o.mul(R.B(np.float32(0.9), u)).add(a.div(nfb).mul(R.B(np.float32(0.1), u)))
    ns = float(np.sqrt(np.sum(s.v.astype(np.float64) ** 2)))
    nsb = R.B(np.float32(ns), u, float(np.sqrt(np.sum(s.e ** 2))) + 2.01 * R.U32 * ns)
    return s.div(nsb)


def check_stream(trk, frames, warps, kind, fmt, f32, stats, where="", feats=None, conf_thresh=0.2, on_frame=None, nearest=NEAREST):
    """Runs the whole stream through trk, checking every frame.  stats gets the largest err / bound per path; returns the number of
    slot transitions checked per path.  nearest: detections tried per slot (more in crowds).  A slot that leaves both lists this frame (remove_duplicate_stracks, a removed unconfirmed
    track, long-lost pruning) is read by its slot and checked like the others: its record stays until a later frame reuses it.
    on_frame (optional) is called after each frame's checks with a dict of what the association certificate
    (tests/assoc_bounds.py) needs: the frame's index, tag, detections and features, the before-state ('before', in list order), the
    checked slots ('exist'), their predicted or warped state with its bound ('base'), the float32-mean flag the association read
    ('uflag'), the detection each slot was updated with ('matched_det', -1 for none) and trk.stat when the tracker has it."""
    dt = np.float32 if f32 else np.float64
    ss = kind == "strongsort"
    counts = dict(predict=0, update=0, birth=0, unconfirmed=0, feature=0)
    flag = {}                                                         # slot -> the step's float32-mean flag, restated
    for i, f in enumerate(frames):
        tag = "%s frame %d" % (where, i + 1)
        fe = None if feats is None else feats[i]
        before = _snapshot(trk, fe is not None)
        w = None if warps is None else np.asarray(warps[i], np.float64).reshape(-1)
        res = trk.step(f, fe, w)
        after = _snapshot(trk, fe is not None)
        seen = dict(after)
        for s in before:
            if s not in after:                                        # left both lists: the slot's record is still this frame's
                m, c = trk.read_slot(s)
                seen[s] = dict(tid=before[s]["tid"], state=-1, pool=before[s]["pool"], mean=m, cov=c)
                if fe is not None:
                    seen[s]["feat"] = trk.read_feature(s)
        dets = np.asarray(f, np.float32).reshape(-1, 6)
        Z = R.det_to_meas(fmt, dets[:, :4]) if len(dets) else np.zeros((0, 4), np.float32)
        pool = [s for s, d in before.items() if d["pool"]]
        q_f32 = all(flag.get(s, False) for s in pool)
        gmc_on = w is not None and kind in ("botsort", "strongsort")
        wk = None if w is None else w.astype(dt)
        new_flag = {}

        exist = [s for s, d in seen.items() if s in before and before[s]["tid"] == d["tid"]]
        born = [s for s in after if s not in exist]
        if exist:
            E = np.array(exist)
            m0 = np.stack([before[s]["mean"] for s in exist]).astype(dt)
            c0 = np.stack([before[s]["cov"] for s in exist]).astype(dt)
            gm = np.stack([seen[s]["mean"] for s in exist])
            gc = np.stack([seen[s]["cov"] for s in exist])
            ispool = np.array([before[s]["pool"] for s in exist])
            tracked0 = np.array([before[s]["state"] == ST_TRACKED for s in exist])
            x0 = R.state(m0, c0, f32)
            if ss:
                xg = R.kf_gmc(*x0, wk) if gmc_on else x0
                pp = R.kf_predict(*xg, fmt, ~tracked0, False if gmc_on else q_f32, f32)
            else:
                pp = R.kf_predict(*x0, fmt, ~tracked0, q_f32, f32)
                if gmc_on:
                    pp = R.kf_gmc(*pp, wk)
            up = R.kf_gmc(*x0, wk) if (gmc_on and not ss) else x0
            base = _sel(ispool, pp, up)
            uflag = np.array([False if (p or (gmc_on and not ss)) else flag.get(s, False) for s, p in zip(exist, ispool)])
            ok_none, w_none = _within(base, gm, gc, f32)
            # update candidates: the NEAREST detections by centre
            nmatch = np.zeros(len(exist), int)
            matched_det = np.full(len(exist), -1)
            w_upd = np.full(len(exist), np.inf)
            if len(dets):
                d2 = ((Z[None, :, :2].astype(np.float64) - gm[:, None, :2]) ** 2).sum(-1)
                near = np.argsort(d2, axis=1)[:, :nearest]
                pi = np.repeat(np.arange(len(exist)), near.shape[1])
                pj = near.reshape(-1)
                bp = _take(base, pi)
                zb = [R.inputs(Z[pj, q].astype(dt), f32) for q in range(4)]
                conf = dets[pj, 4].astype(np.float32) if fmt == R.FMT_NSA else None
                upd = R.kf_update(*bp, fmt, zb, uflag[pi], conf, f32)
                if conf is not None and not tracked0.all():                # re_activate: no confidence
                    upd = _sel(tracked0[pi], upd, R.kf_update(*bp, fmt, zb, uflag[pi], None, f32))
                okp, wp = _within(upd, gm[pi], gc[pi], f32)
                for k in np.where(okp)[0]:
                    nmatch[pi[k]] += 1
                    matched_det[pi[k]] = pj[k]
                np.minimum.at(w_upd, pi, wp)
            for k, s in enumerate(exist):
                assert ok_none[k] or nmatch[k] >= 1, "%s: slot %d (id %d) is on no path of its kind (predict only %.3g, best update %.3g)" % (
                    tag, s, seen[s]["tid"], w_none[k], w_upd[k])
                assert nmatch[k] <= 1 and not (ok_none[k] and nmatch[k]), "%s: slot %d matches more than one path" % (tag, s)
                path = "update" if nmatch[k] else ("predict" if ispool[k] else "unconfirmed")
                counts[path] += 1
                stats[path] = max(stats.get(path, 0.0), float(w_upd[k] if nmatch[k] else w_none[k]))
                new_flag[s] = False if (nmatch[k] or ispool[k] or (gmc_on and not ss)) else flag.get(s, False)
                if fe is not None:
                    old, got = before[s]["feat"], seen[s]["feat"]
                    # BoT-SORT's low-score detections carry no feature (its association 2); every StrongSORT detection has one
                    has_feat = ss or (nmatch[k] and dets[matched_det[k], 4] >= np.float32(conf_thresh))
                    if nmatch[k] and tracked0[k] and has_feat:
                        ref = ema_ref(old, fe[matched_det[k]])
                        stats["feature"] = max(stats.get("feature", 0.0), R.check(got, ref, True, "%s: slot %d feature" % (tag, s)))
                        counts["feature"] += 1
                    else:
                        assert np.array_equal(got, old), "%s: slot %d feature changed without an update" % (tag, s)
        if born:
            im, iP = R.kf_initiate(Z, fmt, f32)
            for s in born:
                okb, wb = _within((im, iP), np.repeat(after[s]["mean"][None], len(Z), 0), np.repeat(after[s]["cov"][None], len(Z), 0), f32)
                assert okb.sum() == 1, "%s: new slot %d is the initiate of %d detections (best %.3g)" % (tag, s, int(okb.sum()), float(wb.min()))
                stats["birth"] = max(stats.get("birth", 0.0), float(wb.min()))
                counts["birth"] += 1
                new_flag[s] = True
                if fe is not None:
                    assert np.array_equal(after[s]["feat"], fe[int(np.argmax(okb))]), "%s: new slot %d feature" % (tag, s)
        flag = new_flag
        if on_frame is not None:
            on_frame(dict(i=i, tag=tag, dets=dets, feats=fe, before=before, exist=exist, base=base if exist else None,
                          uflag=uflag if exist else None, matched_det=matched_det if exist else None,
                          stat=np.asarray(trk.stat).reshape(-1).copy() if hasattr(trk, "stat") else None))
        # output rows
        if len(res):
            slots = res[:, 7].astype(int)
            mean = np.stack([after[s]["mean"] for s in slots]).astype(dt)
            m = [R.inputs(mean[:, q], f32) for q in range(8)]
            ref = R.stack(R.mean_to_tlwh(fmt, m, np.array([flag.get(s, False) for s in slots]), f32))
            stats["out"] = max(stats.get("out", 0.0), R.check(res[:, 1:5], ref, f32, "%s: output rows" % tag))
    return counts


# ---------------------------------------------------------------- streams
def edge_stream(seed=21, n_frames=60, n_obj=40):
    """4K geometry with boxes of about 2 - 8 px: a lifecycle stream's centres scaled by 3, its sizes by 0.1 (objects move ~30 box
    sizes per frame at times, so many stay lost for up to track_buffer frames), BoT-SORT warps with rotation."""
    frames, warps = lifecycle_stream(seed, n_frames, n_obj, warp_sigma=2.0)
    out = []
    for f in frames:
        f = f.copy()
        c = (f[:, :2] + f[:, 2:4]) / 2
        s = (f[:, 2:4] - f[:, :2]) * 0.1
        f[:, :2], f[:, 2:4] = c * 3 - s / 2, c * 3 + s / 2
        out.append(f.astype(np.float32))
    return out, warps


def case(name):
    """(kind, fmt, frames, feats, warps, tracker kwargs) of one step case: a lifecycle_golden configuration, the edge stream
    ('edge_<kind>'), a stream with appearance features ('feat_<kind>': StrongSORT, BoT-SORT with ReID), or UAVMOT on a lifecycle
    stream ('uavmot', default format)."""
    import lifecycle_golden as LG
    if name.startswith("edge_"):
        kind = name[5:]
        frames, warps = edge_stream()
        return kind, "botsort" if kind == "botsort" else "default", frames, None, warps if kind == "botsort" else None, dict(track_buffer=30)
    if name.startswith("feat_"):
        kind = name[5:]
        frames, feats, warps = make_strongsort_stream(17, 40, 40, 64)
        return kind, "strongsort" if kind == "strongsort" else "botsort", frames, feats, warps, dict(track_buffer=30, feat_dim=64)
    if name == "uavmot":
        frames, _ = lifecycle_stream(5, 60, 40)
        return "uavmot", "default", frames, None, None, dict(track_buffer=30)
    cfg = LG.Config(name)
    frames, warps = cfg.stream()
    return cfg.kind, cfg.fmt, frames, None, warps, dict(track_buffer=cfg.track_buffer, frame_rate=cfg.frame_rate,
                                                        conf_thresh=cfg.conf_thresh)


def step_cases():
    import lifecycle_golden as LG
    names = LG.configs() + ["edge_bytetrack", "edge_botsort", "feat_strongsort", "feat_botsort"]
    return [(c, d) for c in names for d in ("f32", "f64")] + [("uavmot", "f64")]      # UAVMOT is built in float64 only
