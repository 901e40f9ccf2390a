"""Writes tests/golden/refchecks.npz: what the UNMODIFIED reference computes in the checks that used to run it live --
YOLOv7-tiny's own ``Model`` and the YOLOv7-w6 TRAINING graph (cfg/training/yolov7-w6.yaml, eval mode) on seeded weights (seeded
samples of their output rows and every objectness), the ReID ``Extractor`` preprocessing and ``Net`` on seeded weights, the
``GMC(method='orb')`` matrices of a short moving sequence, the text ``save_results`` writes, and the tracks of SORT / ByteTrack on
a stream with zero-width boxes.  Needs the reference tree (B2T_REFERENCE_ROOT) and opencv-python: ``python tests/golden/make_golden_refchecks.py``.
The tests that read the archive restate the inputs from the same seeds."""
import ast
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
for p in (ROOT, os.path.join(ROOT, "yolov7-tracker_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)
from oracle import refshim  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "refchecks.npz")

TINY_SEED, TINY_IMG_SEED, TINY_SHAPE, TINY_ROWS = 0, 5, (2, 3, 192, 256), 64
REID_CROP_SEED, REID_N, REID_W_SEED, REID_X_SAMPLE = 9, 5, 3, 2048
SAVE_SEED = 3
FOLD_SEED, FOLD_IMG_SEED, FOLD_ROWS = 3, 4, 128
FLAT_SEED, FLAT_FRAMES, FLAT_OBJ = 61, 30, 60


def tiny():
    from b200track import tiny as T
    sd = T.seeded_state_dict(TINY_SEED)
    model = refshim.load_detector_model("cfg/deploy/yolov7-tiny.yaml")
    model.load_state_dict(sd, strict=False)
    img = torch.rand(TINY_SHAPE, generator=torch.Generator().manual_seed(TINY_IMG_SEED))
    with torch.no_grad():
        ref = model(img)[0].double().numpy()
    rows = np.sort(np.random.default_rng(1).choice(ref.shape[0] * ref.shape[1], TINY_ROWS, replace=False))
    return {"tiny_shape": np.array(ref.shape), "tiny_obj": ref[..., 4].astype(np.float32), "tiny_row_index": rows.astype(np.int32),
            "tiny_rows": ref.reshape(-1, ref.shape[-1])[rows].astype(np.float32)}


def fold():
    """The reference's training graph (Conv + BN, auxiliary heads, IAuxDetect with implicit layers) on a seeded state dict
    (oracle.detector.seeded_training_state_dict over its own key names and shapes, stored here), eval mode, one 128 x 128 image."""
    from oracle import detector as OD
    model = refshim.load_detector_model("cfg/training/yolov7-w6.yaml", fuse=False)
    msd = model.state_dict()
    keys = [k for k in msd if not k.endswith(("anchors", "anchor_grid"))]      # the anchors are the cfg's constants
    shapes = [tuple(msd[k].shape) for k in keys]
    sd = OD.seeded_training_state_dict(keys, shapes, FOLD_SEED)
    missing = model.load_state_dict(sd, strict=False)
    assert not missing.unexpected_keys and all(k.endswith(("anchors", "anchor_grid")) for k in missing.missing_keys)
    img = torch.rand((1, 3, 128, 128), generator=torch.Generator().manual_seed(FOLD_IMG_SEED))
    with torch.no_grad():
        ref = model.eval()(img)[0].double().numpy()
    rows = np.sort(np.random.default_rng(3).choice(ref.shape[0] * ref.shape[1], FOLD_ROWS, replace=False))
    nd = max(len(sh) for sh in shapes)
    return {"fold_keys": np.array(keys), "fold_shapes": np.array([list(sh) + [-1] * (nd - len(sh)) for sh in shapes], np.int32),
            "fold_shape": np.array(ref.shape), "fold_obj": ref[..., 4].astype(np.float32), "fold_row_index": rows.astype(np.int32),
            "fold_rows": ref.reshape(-1, ref.shape[-1])[rows].astype(np.float32)}


def flat_loops():
    """SORT and ByteTrack (xyah Kalman filter) of the unmodified reference on a seeded stream in which a fraction of the boxes is
    flattened to zero width: ids per frame and the boxes of the last frame."""
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    from make_golden import run_reference
    from b200track.synth import zero_width_stream
    frames = zero_width_stream(FLAT_SEED, FLAT_FRAMES, FLAT_OBJ)
    warps = [np.eye(2, 3)] * len(frames)
    out = {}
    for kind in ("sort", "bytetrack"):
        res = run_reference(refshim.load(), kind, frames, warps)
        out["flat_%s_count" % kind] = np.array([len(r[0]) for r in res], np.int32)
        out["flat_%s_ids" % kind] = np.concatenate([r[0] for r in res])
        out["flat_%s_tlwh_last" % kind] = res[-1][1]
        assert np.isfinite(res[-1][1]).all()
    return out


def reid():
    from oracle import reid as R
    ref_root = refshim.REF_ROOT
    sys.path.insert(0, os.path.join(ref_root, "tracker"))
    try:
        from reid_models import deepsort_reid as M
    finally:
        sys.path.remove(os.path.join(ref_root, "tracker"))
    crops = R.seeded_crops(REID_CROP_SEED, REID_N)
    ext = M.Extractor(os.path.join(ref_root, "weights", "ckpt.t7"), use_cuda=False)
    x_ref = ext._preprocess(crops).numpy()
    idx = np.sort(np.random.default_rng(2).choice(x_ref.size, REID_X_SAMPLE, replace=False))
    net = M.Net(reid=True).eval()
    net.load_state_dict(R.seeded_state_dict(REID_W_SEED), strict=False)
    x = R.preprocess(crops)
    with torch.no_grad():
        f_eval = net(x).numpy()
        f_train = net.train()(x).numpy()
    return {"reid_x_shape": np.array(x_ref.shape), "reid_x_index": idx.astype(np.int32), "reid_x": x_ref.reshape(-1)[idx],
            "reid_eval": f_eval, "reid_train": f_train}


def gmc():
    import cv2
    from b200track.synth import textured_frame

    def moved(frame, angle_deg, scale, tx, ty):
        h, w = frame.shape[:2]
        M = cv2.getRotationMatrix2D((w / 2, h / 2), angle_deg, scale)
        M[:, 2] += (tx, ty)
        return cv2.warpAffine(frame, M, (w, h), flags=cv2.INTER_LINEAR, borderMode=cv2.BORDER_REFLECT_101)

    ref = refshim.load().botsort.GMC(method='orb', downscale=2)
    f = textured_frame(11, 720, 1280)
    dets = np.array([[200, 100, 420, 500, 0.9, 0], [700, 300, 900, 640, 0.7, 1]], np.float32)
    rng = np.random.default_rng(0)
    hs = []
    for _ in range(4):
        hs.append(ref.apply(f, dets))
        true = (float(rng.uniform(-6, 6)), float(rng.uniform(-6, 6)))
        f = moved(f, float(rng.uniform(-0.5, 0.5)), 1.0 + float(rng.uniform(-0.004, 0.004)), *true)
        dets = dets + np.array([true[0], true[1], true[0], true[1], 0, 0], np.float32)
    return {"gmc_H": np.array(hs)}


def save_results_frames():
    """The rows test_host_logic writes (same seed and draws)."""
    rng = np.random.default_rng(SAVE_SEED)
    frames = []
    for _ in range(4):
        n = int(rng.integers(1, 6))
        rows = np.zeros((n, 8))
        rows[:, 0] = rng.integers(1, 500, n)
        rows[:, 1:5] = rng.uniform(0, 1280, (n, 4)).round(3)
        rows[:, 5] = rng.integers(0, 10, n)
        frames.append(rows)
    return frames


def save_results():
    src = os.path.join(refshim.REF_ROOT, "tracker", "track.py")
    tree = ast.parse(open(src).read())
    fn = next(n for n in tree.body if isinstance(n, ast.FunctionDef) and n.name == "save_results")
    ns = {"os": os}
    exec(compile(ast.Module([fn], []), src, "exec"), ns)
    frames = save_results_frames()
    out = {}
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        os.chdir(tmp)
        try:
            for data_type in ("mot17", "default"):
                results = [(k + 1, [int(r[0]) for r in rows], [r[1:5] for r in rows], [r[5] for r in rows]) for k, rows in enumerate(frames)]
                ns["save_results"]("ref_%s" % data_type, "seq", results, data_type=data_type)
                out["save_results_" + data_type] = np.array(open(os.path.join("tracker", "results", "ref_%s" % data_type, "seq.txt")).read())
        finally:
            os.chdir(cwd)
    return out


if __name__ == "__main__":
    assert refshim.available(), "reference tree not present at %s" % refshim.REF_ROOT
    data = {}
    for part in (tiny, fold, reid, gmc, save_results, flat_loops):
        data.update(part())
    np.savez_compressed(OUT, **data)
    print("wrote %s (%d KB)" % (OUT, os.path.getsize(OUT) // 1024))
