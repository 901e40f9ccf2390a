"""Sub-benchmarks of the default bench line (``config.sub_benchmarks``): the BASELINE.json configurations that are not the
headline, measured in the same run on the same GPU so that one command records them.

  C1  the reference's CPU-runnable plumbing case: YOLOv7-tiny on one 1280 x 1280 frame + ByteTrack update on 50 detections.
  C3  ByteTrack full loop, ~300 detections / frame, ~250 live tracks, 4 sequences per launch, detections resident in HBM,
      L2 flushed between steps: frames/s, us per step, HBM roofline of track_step_kernel (latency-bound by construction: 1 CTA per
      sequence, SURVEY 8d).
  C4  BoT-SORT (Kalman xywh + per-frame camera warp + IoU), 500 objects / frame, 8 sequences sharded over the ranks.
  GMC camera-motion estimation (SURVEY 8f row 1: FAST + ORB + Hamming 2-NN + RANSAC partial affine, tracker/botsort.py:111-235), 8
      sequences of 1280 x 1280 frames per call, the reference's own host OpenCV recipe timed beside it.
  C5  assignment-only sweep: N x M "+1" IoU cost matrix + exact LAP (lapjv semantics), N = M in {64 .. 2048}, 64 problems per
      launch, fp64 like the reference: GB/s of (write + read of every cost matrix) against the measured HBM peak.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
for p in (ROOT, os.path.join(ROOT, "yolov7-tracker_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

STREAM_WARM = 60


def _events(torch, n):
    return [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(n)]


def tracker_loop(torch, dev, kind, n_seq, n_obj, steps, seed0, hbm_gbs, warp_sigma=0.0, cap=1024, dmax=512, flush=None):
    """Device-resident fused tracker loop: returns frames/s, us/step and the roofline of track_step_kernel."""
    from b200track import _lib as L
    from b200track.engine import TrackEngine
    from b200track.synth import make_stream, pack_frames
    from bench import algorithmic_bytes
    n_frames = STREAM_WARM + steps
    streams = [make_stream(seed0 + s, n_frames, n_obj, warp_sigma=warp_sigma) for s in range(n_seq)]
    packed = [pack_frames(st[0], dmax) for st in streams]
    d_dets = torch.from_numpy(np.stack([p[0] for p in packed], 1)).to(dev)           # (F, S, dmax, 6)
    d_cnt = torch.from_numpy(np.stack([p[1] for p in packed], 1)).to(dev)
    d_warp = torch.from_numpy(np.stack([st[1].reshape(n_frames, 6) for st in streams], 1)).to(dev) if warp_sigma > 0 else None
    eng = TrackEngine(kind, n_seq=n_seq, dtype="f64", cap=cap, dmax=dmax, device=dev)
    rows = min(cap, 1024)
    d_out = torch.zeros((n_seq, rows, L.OUT_COLS), dtype=torch.float64, device=dev)
    d_stat = torch.zeros((n_frames, n_seq, L.STAT_WORDS), dtype=torch.int32, device=dev)
    for f in range(STREAM_WARM):
        eng.step_device(d_dets[f], d_cnt[f], d_out, d_stat[f], warps=None if d_warp is None else d_warp[f])
    torch.cuda.synchronize()
    ev = _events(torch, steps)
    for k in range(steps):
        f = STREAM_WARM + k
        if flush is not None:
            flush.zero_()                                    # L2 flush between timed iterations, outside the event pair
        ev[k][0].record()
        eng.step_device(d_dets[f], d_cnt[f], d_out, d_stat[f], warps=None if d_warp is None else d_warp[f])
        ev[k][1].record()
    torch.cuda.synchronize()
    ms = np.array([a.elapsed_time(b) for a, b in ev])
    st = d_stat[STREAM_WARM:].cpu().numpy()
    assert int(st[:, :, L.STAT_ERR].max()) == 0, "tracker capacity error"
    algo = float(np.mean([algorithmic_bytes(st[k], 8) for k in range(steps)]))
    us = 1e3 * float(np.median(ms))
    return {"frames_per_s": n_seq * steps / (ms.sum() / 1e3), "us_per_step_median": us, "sequences": n_seq, "steps": steps,
            "tracked_mean": float(st[:, :, L.STAT_NTRACKED].mean()), "lost_mean": float(st[:, :, L.STAT_NLOST].mean()),
            "dets_mean": float(st[:, :, L.STAT_NHI].mean() + st[:, :, L.STAT_NLO].mean()), "ids_issued_per_seq": int(st[-1, :, L.STAT_NEXT_ID].mean()),
            "roofline": {"bound": "hbm", "kernel": "track_step_kernel<double>", "algorithmic_bytes_per_launch": algo, "achieved_GBs": algo / (us * 1e-6) / 1e9,
                         "peak_GBs": hbm_gbs, "frac": algo / (us * 1e-6) / 1e9 / hbm_gbs,
                         "note": "latency-bound: one CTA per sequence, state in L2 / shared memory (SURVEY 8d)"}}


def assignment_sweep(torch, dev, hbm_gbs, sizes=(64, 128, 256, 512, 1024, 2048), batch=64):
    """C5: batched IoU cost + exact LAP per size: us per launch and GB/s of the two kernels' algorithmic traffic."""
    import ctypes as C
    from b200track import _lib as L
    lib = L.load()
    s_ptr = lambda: C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)      # noqa: E731
    out = {}
    rng = np.random.default_rng(55)
    for n in sizes:
        b = batch if n <= 1024 else 16                        # 64 x 2048^2 x 8 B = 2 GB of cost matrices: 16 problems at the largest size
        xy = rng.uniform(0, 4000, (b, n, 2))
        wh = np.stack([rng.uniform(20, 80, (b, n)), rng.uniform(40, 160, (b, n))], -1)
        a = np.round(np.concatenate([xy, xy + wh], -1))
        perm = np.stack([rng.permutation(n) for _ in range(b)])
        bb = np.round(np.take_along_axis(a, perm[..., None], 1) + rng.normal(0, 3, (b, n, 4)))
        da, db = torch.from_numpy(a).to(dev), torch.from_numpy(bb).to(dev)
        cost = torch.empty((b, n, n), dtype=torch.float64, device=dev)
        x = torch.empty((b, n), dtype=torch.int32, device=dev); y = torch.empty((b, n), dtype=torch.int32, device=dev)
        ws = torch.empty(lib.b2t_lap_workspace_bytes(L.F64, n, n, b), dtype=torch.uint8, device=dev)

        def iou():
            L.check(lib, lib.b2t_iou_cost(L.F64, C.c_void_p(da.data_ptr()), n, C.c_void_p(db.data_ptr()), n, C.c_void_p(cost.data_ptr()), n, b, 1, s_ptr()))

        def lap(t):
            L.check(lib, lib.b2t_lap_solve(L.F64, C.c_void_p(cost.data_ptr()), n, n, n, t, C.c_void_p(x.data_ptr()), C.c_void_p(y.data_ptr()),
                                           C.c_void_p(ws.data_ptr()), ws.numel(), b, s_ptr()))
        iou(); lap(0.9); torch.cuda.synchronize()
        reps = 5
        e = _events(torch, 3)
        e[0][0].record()
        for _ in range(reps):
            iou()
        e[0][1].record(); e[1][0].record()
        for _ in range(reps):
            lap(0.9)
        e[1][1].record(); e[2][0].record()
        for _ in range(reps):
            lap(0.5)
        e[2][1].record()
        torch.cuda.synchronize()
        t_iou, t_lap9, t_lap5 = (1e3 * p[0].elapsed_time(p[1]) / reps for p in e)
        matched = int((x >= 0).sum())
        mat = 8.0 * b * n * n
        out["N=M=%d" % n] = {"problems_per_launch": b, "iou_us": t_iou, "lap_us_thresh_0.9": t_lap9, "lap_us_thresh_0.5": t_lap5,
                             "iou_GBs": (mat + 64.0 * b * n) / (t_iou * 1e-6) / 1e9, "lap_GBs_0.9": mat / (t_lap9 * 1e-6) / 1e9,
                             "iou_frac_of_hbm": (mat + 64.0 * b * n) / (t_iou * 1e-6) / 1e9 / hbm_gbs, "lap_frac_of_hbm_0.9": mat / (t_lap9 * 1e-6) / 1e9 / hbm_gbs,
                             "matched_fraction_0.5": matched / float(b * n)}
        del cost, ws, da, db
        torch.cuda.empty_cache()
    return out


def gmc_estimation(torch, dev, hbm_gbs, n_seq=8, size=1280, steps=40, cpu_frames=3):
    """SURVEY 8f row 1: camera-motion estimation (tracker/botsort.py:111-235) for n_seq sequences per call on textured frames
    that move by a known shift, ~300 detection boxes masked out per frame; the reference's own GMC.apply (host OpenCV) is timed
    beside it on one sequence."""
    import time
    from b200track.gmc import GmcEstimator
    from b200track.synth import make_stream, pack_frames, textured_frame
    pool = 6
    shifts = [(3 * k, -2 * k) for k in range(pool)]                       # (dy, dx) of frame k relative to frame 0
    base = [textured_frame(7000 + s, size, size, n_rect=1200) for s in range(n_seq)]
    frames = [torch.from_numpy(np.stack([np.roll(b, sh, (0, 1)) for b in base])).to(dev) for sh in shifts]
    dets_np, cnt_np = pack_frames(make_stream(7100, n_seq, 300, img=size)[0], 320)
    dets, cnt = torch.from_numpy(dets_np).to(dev), torch.from_numpy(cnt_np).to(dev)
    est = GmcEstimator(n_seq, size, size, 2, max_kp=32768, device=dev)
    for k in range(pool):
        est.estimate(frames[k], dets, cnt, det_thresh=0.2)
    torch.cuda.synchronize()
    ev = _events(torch, steps)
    errs, kps, inl = [], [], []
    for k in range(steps):
        ev[k][0].record()
        w, st = est.estimate(frames[k % pool], dets, cnt, det_thresh=0.2)
        ev[k][1].record()
        if k % pool:                                                      # consecutive pool frames differ by (+3, -2): dx = -2, dy = +3
            wc, sc = w.cpu().numpy(), st.cpu().numpy()
            errs.append(float(max(np.abs(wc[:, 0, 2] + 2).max(), np.abs(wc[:, 1, 2] - 3).max())))
            kps.append(float(sc[:, 0].mean())); inl.append(float(sc[:, 4].mean()))
    torch.cuda.synchronize()
    us = 1e3 * float(np.median([a.elapsed_time(b) for a, b in ev]))
    px, px2 = size * size, (size // 2) * (size // 2)
    algo = n_seq * (3.0 * px + 6.0 * px2 + 2 * 40.0 * float(np.mean(kps)))         # frame read; gray / score / blur planes written and read; key points + descriptors
    out = {"frames_per_s": n_seq / (us * 1e-6), "us_per_call_median": us, "sequences": n_seq, "frame": "%dx%d uint8 BGR, working size %dx%d" % (size, size, size // 2, size // 2),
           "launches_per_call": est.launches_per_call, "keypoints_mean": float(np.mean(kps)), "ransac_inliers_mean": float(np.mean(inl)),
           "max_abs_translation_error_px": float(max(errs)), "true_motion_px": [-2, 3],
           "roofline": {"bound": "hbm", "kernel": "gmc_* (11 launches)", "algorithmic_bytes_per_call": algo, "achieved_GBs": algo / (us * 1e-6) / 1e9,
                        "peak_GBs": hbm_gbs, "frac": algo / (us * 1e-6) / 1e9 / hbm_gbs,
                        "note": "byte / integer work on 0.4 MPixel planes: launch- and latency-bound at 8 sequences, not bandwidth-bound"}}
    # ---- the reference's own estimator on the host cores (one sequence)
    try:
        import tempfile
        from oracle import build_ref, refshim
        tmp = None
        if not refshim.available() and os.path.exists(build_ref.ARCHIVE):
            tmp = tempfile.mkdtemp(prefix="b2t_ref_")
            refshim.use_root(build_ref.unpack(tmp))
        kind = "reference" if refshim.available() else "port"
        if kind == "reference":
            ref = refshim.load().botsort.GMC(method='orb', downscale=2)
        else:
            from oracle.gmc import GMCOracle
            ref = GMCOracle(estimator="cv2")
        d0 = dets_np[0, :cnt_np[0]]
        hi = d0[d0[:, 4] >= np.float32(0.2)]
        f_host = [np.ascontiguousarray(np.roll(base[0], sh, (0, 1))) for sh in shifts[:cpu_frames + 1]]
        ref.apply(f_host[0], hi)
        ms, Hs = [], []
        for k in range(1, cpu_frames + 1):
            t0 = time.perf_counter(); Hs.append(ref.apply(f_host[k], hi)); ms.append(1e3 * (time.perf_counter() - t0))
        # same frames through the GPU estimator (fresh state) for the matrix comparison
        e1 = GmcEstimator(1, size, size, 2, max_kp=32768, device=dev)
        d1, c1 = dets[:1].contiguous(), cnt[:1].contiguous()
        diffs = []
        for k in range(cpu_frames + 1):
            w, _ = e1.estimate(torch.from_numpy(f_host[k][None]).to(dev), d1, c1, det_thresh=0.2)
            if k:
                diffs.append(float(np.abs(w[0].cpu().numpy() - np.asarray(Hs[k - 1], dtype=np.float64)).max()))
        out["cpu_reference"] = {"kind": kind, "ms_per_frame": [round(v, 1) for v in ms], "frames_per_s": 1e3 / float(np.mean(ms)), "cores": 1,
                                "what": "tracker/botsort.py GMC(method='orb', downscale=2).apply, unmodified (host OpenCV %s)" % __import__("cv2").__version__ if kind == "reference"
                                        else "oracle/gmc.py restatement with cv2.estimateAffinePartial2D",
                                "max_abs_matrix_diff_vs_gpu": max(diffs)}
        if tmp:
            import shutil
            shutil.rmtree(tmp, ignore_errors=True)
    except Exception as e:                                                 # no OpenCV on the box: the GPU number stands alone
        out["cpu_reference"] = {"unavailable": "%s: %s" % (type(e).__name__, e)}
    return out


def reid_features(torch, dev, n_crops=256, steps=20, cpu_crops=16):
    """SURVEY 8f row 3: the ReID extractor (tracker/reid_models/deepsort_reid.py:63-153) on n_crops windows of one frame per call --
    crop / resize / normalise, 20 wgmma convolutions, batch-statistics BatchNorm, pooling -- with the reference's own Net timed on
    the host cores beside it (seeded weights: the 46 MB checkpoint does not travel)."""
    import time
    from b200track.reid import ReidExtractor
    from b200track.synth import textured_frame
    from oracle import reid as R
    sd = R.seeded_state_dict(3)
    frame = torch.from_numpy(textured_frame(7300, 1280, 1280, n_rect=1200)).to(dev)
    rng = np.random.default_rng(9)
    x1 = rng.uniform(0, 1100, n_crops); y1 = rng.uniform(0, 1000, n_crops)
    tlbr = np.stack([x1, y1, x1 + rng.uniform(20, 80, n_crops), y1 + rng.uniform(40, 160, n_crops)], 1)      # the C3 object sizes
    out = {}
    for mode in ("batch", "running"):
        ext = ReidExtractor(sd, device=dev, bn_mode=mode)
        f = ext.features_from_frame(frame, tlbr)
        torch.cuda.synchronize()
        ev = _events(torch, steps)
        for k in range(steps):
            ev[k][0].record(); f = ext.features_from_frame(frame, tlbr); ev[k][1].record()
        torch.cuda.synchronize()
        us = 1e3 * float(np.median([a.elapsed_time(b) for a, b in ev]))
        net = ext.last_net
        out["bn_" + mode] = {"us_per_call_median": us, "crops_per_s": n_crops / (us * 1e-6), "launches_per_call": net["launches"],
                             "conv_gflop_per_call": net["flops"] / 1e9, "conv_tflops_incl_glue": net["flops"] / (us * 1e-6) / 1e12, "batch_capacity": net["n"]}
        if mode == "batch":
            feats = f.cpu().numpy()
    out["crops"] = n_crops
    out["note"] = ("bn_batch = what the reference computes (its extractor is never switched to eval(): BatchNorm with the statistics of each call), "
                   "bn_running = eval-mode BatchNorm folded into the convolutions; host-side crop bookkeeping is inside the timed call")
    try:
        import tempfile
        from oracle import build_ref, refshim
        tmp = None
        root = refshim.REF_ROOT
        if not refshim.available() and os.path.exists(build_ref.ARCHIVE):
            tmp = tempfile.mkdtemp(prefix="b2t_ref_")
            root = build_ref.unpack(tmp)
        kind = "port"
        t = tlbr.astype(np.int64)
        fh = frame.cpu().numpy()
        crops = [fh[a[1]:a[3], a[0]:a[2]] for a in t[:cpu_crops]]
        torch.set_num_threads(min(32, len(os.sched_getaffinity(0))))
        if os.path.exists(os.path.join(root, "tracker", "reid_models", "deepsort_reid.py")):
            sys.path.insert(0, os.path.join(root, "tracker"))
            try:
                from reid_models import deepsort_reid as M
            finally:
                sys.path.remove(os.path.join(root, "tracker"))
                for k in [k for k in sys.modules if k.startswith("reid_models")]:
                    del sys.modules[k]
            net = M.Net(reid=True)                                  # training mode, like the reference's Extractor
            net.load_state_dict(sd, strict=False)
            kind = "reference"

            def run():
                with torch.no_grad():
                    return net(R.preprocess(crops))
        else:
            def run():
                with torch.no_grad():
                    return R.forward(sd, R.preprocess(crops), batch_stats=True)
        run()
        t0 = time.perf_counter(); ref = run(); dt = time.perf_counter() - t0
        ext = ReidExtractor(sd, device=dev, bn_mode="batch")
        got = ext(crops)
        out["cpu_reference"] = {"kind": kind, "crops": cpu_crops, "ms_per_call": 1e3 * dt, "crops_per_s": cpu_crops / dt, "cores": torch.get_num_threads(),
                                "what": "tracker/reid_models/deepsort_reid.py Net(reid=True), unmodified, torch-cpu fp32 (+ the oracle's restated pre-processing)" if kind == "reference"
                                        else "oracle/reid.py restatement, torch-cpu fp32",
                                "min_cosine_gpu_vs_cpu": float((got * ref.numpy()).sum(1).min())}
        if tmp:
            import shutil
            shutil.rmtree(tmp, ignore_errors=True)
    except Exception as e:
        out["cpu_reference"] = {"unavailable": "%s: %s" % (type(e).__name__, e)}
    return out


def c1_tiny_plumbing(torch, dev, size=1280):
    """BASELINE.json configs[0]: one 1280 x 1280 frame through YOLOv7-tiny (seeded random init) + decode + NMS, and one ByteTrack update on
    50 random detections -- the reference's own CPU-runnable plumbing case.  GPU: DetectorTiny (batch 1) + the fused tracker step; CPU:
    the reference's Model(cfg/deploy/yolov7-tiny.yaml) on torch-cpu + ByteTrack.update, from oracle/_ref."""
    import time
    from b200track import _lib as L
    from b200track import tiny
    from b200track.engine import TrackEngine
    from b200track.synth import make_stream, pack_frames
    sd = tiny.seeded_state_dict(0)
    det = tiny.DetectorTiny(sd, batch=1, img_size=size, device=dev, use_graph=True)
    img = torch.rand((1, 3, size, size), generator=torch.Generator().manual_seed(1)).to(dev)
    det.detect(img); det.detect(img); torch.cuda.synchronize()
    ev = _events(torch, 10)
    for k in range(10):
        ev[k][0].record(); det.detect(img); ev[k][1].record()
    torch.cuda.synchronize()
    det_us = 1e3 * float(np.median([a.elapsed_time(b) for a, b in ev]))
    frames, _ = make_stream(9100, 12, 50, img=size)
    dets_np, cnt_np = pack_frames(frames, 64)
    eng = TrackEngine("bytetrack", n_seq=1, dtype="f64", cap=256, dmax=64, device=dev)
    d_dets, d_cnt = torch.from_numpy(dets_np).to(dev), torch.from_numpy(cnt_np).to(dev)
    out = torch.zeros((1, 256, L.OUT_COLS), dtype=torch.float64, device=dev); stat = torch.zeros((1, L.STAT_WORDS), dtype=torch.int32, device=dev)
    for f in range(6):
        eng.step_device(d_dets[f:f + 1].contiguous(), d_cnt[f:f + 1].contiguous(), out, stat)
    torch.cuda.synchronize()
    ev = _events(torch, 6)
    for k in range(6):
        ev[k][0].record(); eng.step_device(d_dets[6 + k:7 + k].contiguous(), d_cnt[6 + k:7 + k].contiguous(), out, stat); ev[k][1].record()
    torch.cuda.synchronize()
    trk_us = 1e3 * float(np.median([a.elapsed_time(b) for a, b in ev]))
    res = {"detector": "YOLOv7-tiny, %dx%d, batch 1, fp16 operands: forward (50 conv launches + pools, CUDA graph) + fused decode / NMS" % (size, size),
           "detect_us": det_us, "bytetrack_update_50dets_us": trk_us, "frames_per_s": 1e6 / (det_us + trk_us), "conv_gflop": det.flops / 1e9,
           "conv_tflops_incl_glue_and_nms": det.flops / (det_us * 1e-6) / 1e12, "detections": int(det.out_count[0])}
    try:
        import tempfile
        from oracle import build_ref, refshim
        tmp = None
        if not refshim.available() and os.path.exists(build_ref.ARCHIVE):
            tmp = tempfile.mkdtemp(prefix="b2t_ref_")
            refshim.use_root(build_ref.unpack(tmp))
        if refshim.available():
            torch.set_num_threads(min(32, len(os.sched_getaffinity(0))))
            model = refshim.load_detector_model("cfg/deploy/yolov7-tiny.yaml")
            model.load_state_dict(sd, strict=False)
            general = refshim.load_general()
            trk = refshim.load().bytetrack.ByteTrack(refshim.Opts(img_size=size), frame_rate=30)
            x = img.cpu()
            with torch.no_grad():
                model(x)
                t0 = time.perf_counter(); pred = model(x)[0]; o = general.non_max_suppression(pred, 0.01, 0.45)[0]; t1 = time.perf_counter()
            for f in range(6):
                trk.update(frames[f], None)
            t2 = time.perf_counter(); trk.update(frames[6], None); t3 = time.perf_counter()
            res["cpu_reference"] = {"kind": "reference", "cores": torch.get_num_threads(), "detect_ms": 1e3 * (t1 - t0), "bytetrack_update_ms": 1e3 * (t3 - t2),
                                    "frames_per_s": 1.0 / ((t1 - t0) + (t3 - t2)), "detections": int(o.shape[0]),
                                    "what": "models/yolo.py Model(cfg/deploy/yolov7-tiny.yaml) fused, torch-cpu fp32 + utils/general.py non_max_suppression + tracker/bytetrack.py ByteTrack.update, unmodified"}
        else:
            res["cpu_reference"] = {"unavailable": "no oracle/_ref archive"}
        if tmp:
            import shutil
            shutil.rmtree(tmp, ignore_errors=True)
    except Exception as e:
        res["cpu_reference"] = {"unavailable": "%s: %s" % (type(e).__name__, e)}
    del det, eng
    torch.cuda.empty_cache()
    return res


def run_all(torch, dev, rank, world, hbm_gbs, quick=False):
    """Returns the dict stored under config.sub_benchmarks (rank 0 gathers C4 over the ranks)."""
    import torch.distributed as dist
    res = {}
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    if rank == 0:
        res["C3_bytetrack_4seq_tracker_only"] = tracker_loop(torch, dev, "bytetrack", 4, 300, 150 if quick else 400, 3000, hbm_gbs, flush=flush)
    # C4: 8 sequences sharded over the ranks (all 8 on this GPU when world == 1)
    s_local = max(1, 8 // world) if world <= 8 else 1
    c4 = tracker_loop(torch, dev, "botsort", s_local, 500, 100 if quick else 250, 4000 + rank * s_local, hbm_gbs, warp_sigma=3.0, cap=1152, dmax=576, flush=flush)
    if world > 1:
        t = torch.tensor([c4["us_per_step_median"], c4["frames_per_s"]], dtype=torch.float64, device=dev)
        parts = [torch.zeros_like(t) for _ in range(world)]
        dist.all_gather(parts, t)
        if rank == 0:
            worst = max(float(p[0]) for p in parts)
            c4 = dict(c4, frames_per_s=s_local * world / (worst * 1e-6), us_per_step_median=worst, sequences=s_local * world, ranks=world,
                      note="8 sequences sharded over the ranks; us = slowest rank's median step (max over ranks), frames/s = all sequences / that")
    if rank == 0:
        res["C4_botsort_500dets_8seq"] = c4
        res["C1_tiny_plumbing_1frame_50dets"] = c1_tiny_plumbing(torch, dev)
        res["GMC_estimation_8seq"] = gmc_estimation(torch, dev, hbm_gbs, steps=20 if quick else 40)
        res["ReID_extractor_256crops"] = reid_features(torch, dev, steps=10 if quick else 20)
        res["C5_iou_lap_sweep_fp64"] = assignment_sweep(torch, dev, hbm_gbs, sizes=(64, 256, 1024) if quick else (64, 128, 256, 512, 1024, 2048))
    del flush
    torch.cuda.empty_cache()
    return res
