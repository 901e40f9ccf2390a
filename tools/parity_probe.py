"""GPU box: how far is the wgmma detector from the fp32 oracle, per activation type and input size?

For every (size, batch) and act_dtype in {fp16, bf16}: raw-logit error against the oracle that emulates the same 16-bit rounding
and against the pure fp32 oracle, objectness error, and the post-NMS agreement SURVEY 7.2 #5 defines (kept boxes with an fp32
partner of the same class at IoU >= 0.99 and |dconf| <= 1e-2), plus looser IoU levels for context.  Prints one JSON line per
configuration; the thresholds in tests/test_gpu_detector.py are set from these numbers.

    python tools/parity_probe.py [--sizes 640:1,1280:8]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "yolov7-tracker_b200")):
    sys.path.insert(0, p)


def match_stats(ours, ref, ious=(0.99, 0.95, 0.9), dconf=1e-2):
    """ours / ref: (n, 6) post-NMS rows.  Fraction of OUR rows with a ref row of the same class, IoU >= t, |dconf| <= dconf."""
    import torchvision
    if ours.shape[0] == 0 or ref.shape[0] == 0:
        return {("iou%.2f" % t): 0.0 for t in ious}
    iou = torchvision.ops.box_iou(ours[:, :4], ref[:, :4])
    same = ours[:, 5:6] == ref[:, 5].unsqueeze(0)
    close = (ours[:, 4:5] - ref[:, 4].unsqueeze(0)).abs() <= dconf
    out = {}
    for t in ious:
        ok = ((iou >= t) & same & close).any(1)
        out["iou%.2f" % t] = float(ok.float().mean())
    ok_noconf = ((iou >= 0.99) & same).any(1)
    out["iou0.99_any_conf"] = float(ok_noconf.float().mean())
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="256:2,640:1,1280:8")
    ap.add_argument("--dtypes", default="fp16,bf16")
    ap.add_argument("--act-std", default="1.0")
    args = ap.parse_args()
    from b200track.detector import DetectorW6
    from b200track.w6 import ANCHORS, STRIDES, calibrated_state_dict, w6_layers
    from oracle import detector as OD
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    layers = w6_layers()
    for spec in args.sizes.split(","):
        size, batch = (int(v) for v in spec.split(":"))
        for act_std in [float(v) for v in args.act_std.split(",")]:
            sd = calibrated_state_dict(0, size, "cuda", act_std=act_std)
            g = torch.Generator().manual_seed(4000 + size)
            img = torch.rand((batch, 3, size, size), generator=g).cuda()
            with torch.no_grad():
                ref32, raw32 = OD.forward(layers, sd, img, ANCHORS, STRIDES, return_raw=True)
            nms32 = OD.non_max_suppression(ref32, conf_thres=0.01)
            for name in args.dtypes.split(","):
                dt = torch.float16 if name == "fp16" else torch.bfloat16
                det = DetectorW6(sd, batch=batch, img_size=size, use_graph=False, autotune=False, act_dtype=dt)
                pred = det.forward(img).clone()
                out, cnt = det.detect(img, post=False)
                torch.cuda.synchronize()
                with torch.no_grad():
                    ref16, raw16 = OD.forward(layers, sd, img, ANCHORS, STRIDES, emulate_bf16=dt, return_raw=True)
                rec = {"size": size, "batch": batch, "dtype": name, "act_std": act_std, "levels": []}
                for lvl in range(4):
                    r32, r16 = raw32[lvl], raw16[lvl]
                    got = det.raw[lvl][..., :255].reshape(batch, r32.shape[2], r32.shape[3], 3, 85).permute(0, 3, 1, 2, 4)
                    e32, e16 = (got - r32).abs(), (got - r16).abs()
                    rec["levels"].append({"std": float(r32.std()), "vs_fp32_mean": float(e32.mean()), "vs_fp32_max": float(e32.max()),
                                          "vs_fp32_relrms": float((e32 ** 2).mean().sqrt() / r32.std()),
                                          "vs_emu_mean": float(e16.mean()), "vs_emu_max": float(e16.max()),
                                          "vs_emu_relrms": float((e16 ** 2).mean().sqrt() / r16.std()),
                                          "emu_vs_fp32_relrms": float(((r16 - r32) ** 2).mean().sqrt() / r32.std())})
                rec["obj_max_err_vs_fp32"] = float((pred[..., 4] - ref32[..., 4]).abs().max())
                rec["obj_max_err_vs_emu"] = float((pred[..., 4] - ref16[..., 4]).abs().max())
                rec["obj_mean_err_vs_emu"] = float((pred[..., 4] - ref16[..., 4]).abs().mean())
                rec["cand"] = int((pred[..., 4] > 0.01).sum())
                per_img, per_img_rev, counts = [], [], []
                for b in range(batch):
                    n = int(cnt[b])
                    counts.append((n, int(nms32[b].shape[0])))
                    per_img.append(match_stats(out[b, :n], nms32[b]))
                    per_img_rev.append(match_stats(nms32[b], out[b, :n]))
                rec["kept"] = counts
                for key in per_img[0]:
                    rec["match_" + key] = [round(m[key], 4) for m in per_img]
                    rec["match_rev_" + key] = [round(m[key], 4) for m in per_img_rev]
                # emulating oracle's own NMS agreement with fp32: what ANY implementation with this rounding can reach
                nms16 = OD.non_max_suppression(ref16, conf_thres=0.01)
                rec["emu_match_iou0.99"] = [round(match_stats(nms16[b], nms32[b])["iou0.99"], 4) for b in range(batch)]
                print(json.dumps(rec), flush=True)
                del det
                torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
