"""GPU box: per-layer sweep of the wgmma conv kernel's tiling modes on the YOLOv7-w6 shapes (batch 8, 1280 x 1280).

For every layer in LAYERS and every valid (halo, mt, BLOCK_N, ring depth, K splits): checks the output against torch
(F.conv2d on the same fp16-rounded operands, fp32 accumulation) and times `reps` back-to-back launches with CUDA events.
Prints one line per configuration and the best one per layer with its distance to the layer's floor
(max(flops / tensor peak, algorithmic bytes / HBM peak), MEASURED_PEAKS.json).

    python tools/conv_layer_bench.py [--layers L5,L23] [--quick]
"""
import argparse
import itertools
import json
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "yolov7-tracker_b200")):
    sys.path.insert(0, p)

# name: (cin, cout, k, s, H = W of the input, act)
LAYERS = {
    "L1": (16, 64, 3, 1, 640),
    "L2": (64, 128, 3, 2, 640), "L5": (64, 64, 3, 1, 320), "L10": (256, 128, 1, 1, 320), "L11": (128, 256, 3, 2, 320),
    "L13+12": (256, 256, 1, 1, 160), "L14": (128, 128, 3, 1, 160), "L19": (512, 256, 1, 1, 160), "L20": (256, 512, 3, 2, 160),
    "L22+21": (512, 512, 1, 1, 80), "L23": (256, 256, 3, 1, 80), "L28": (1024, 512, 1, 1, 80), "L29": (512, 768, 3, 2, 80),
    "L31+30": (768, 768, 1, 1, 40), "L32": (384, 384, 3, 1, 40), "L37": (1536, 768, 1, 1, 40), "L38": (768, 1024, 3, 2, 40),
    "L40+39": (1024, 1024, 1, 1, 20), "L41": (512, 512, 3, 1, 20), "L46": (2048, 1024, 1, 1, 20), "L47.cv4": (512, 512, 1, 1, 20),
    "L48": (512, 384, 1, 1, 20), "L55": (192, 192, 3, 1, 40), "L67": (128, 128, 3, 1, 80), "L79": (64, 64, 3, 1, 160),
    "L104": (384, 512, 3, 2, 40), "L109": (256, 256, 3, 1, 20), "L114": (128, 256, 3, 1, 160), "L115": (256, 512, 3, 1, 80),
    "L116": (384, 768, 3, 1, 40), "L117": (512, 1024, 3, 1, 20),
}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", default="")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--quick", action="store_true", help="fewer ring depths")
    ap.add_argument("--verbose", action="store_true")
    ap.add_argument("--producers", default="1,2")
    ap.add_argument("--splits", default="1")
    ap.add_argument("--tps", default="0,1", help="halo mode: taps per weight box (0 = automatic: 3 / resident, 1 = one tap)")
    args = ap.parse_args()
    from b200track import _lib as L
    from b200track.conv import ConvPlan, pack_conv_weight
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    except Exception:
        pass
    tf_peak, hbm = float(peaks.get("bf16_tflops", 1590.0)) * 1e12, float(peaks.get("hbm_gbs", 6650.0)) * 1e9
    names = [n for n in args.layers.split(",") if n] or list(LAYERS)
    dt = torch.float16
    n = args.batch
    summary = []
    for name in names:
        cin, cout, k, s, hw = LAYERS[name]
        g = torch.Generator(device="cuda").manual_seed(abs(hash(name)) % (2 ** 31))
        x = torch.randn((n, hw, hw, cin), device="cuda", generator=g).to(dt)
        w = torch.randn((cout, cin, k, k), device="cuda", generator=g) * (1.5 / (cin * k * k) ** 0.5)
        b = torch.randn(cout, device="cuda", generator=g) * 0.5
        ho = hw // s
        ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.to(dt).float(), b, stride=s, padding=k // 2)
        ref = (ref * torch.sigmoid(ref)).permute(0, 2, 3, 1).contiguous()
        wp = pack_conv_weight(w, dtype=dt)
        flops = 2.0 * n * ho * ho * cout * k * k * cin
        abytes = 2.0 * (n * hw * hw * cin + n * ho * ho * cout + cout * cin * k * k)
        floor_us = max(flops / tf_peak, abytes / hbm) * 1e6
        halos = [0, 1] if (k == 3 and s == 1 and (cin % 64 == 0 or cin in (16, 32))) else [0]
        bns = [v for v in (64, 128, 256) if v <= max(64, (cout + 15) // 16 * 16)]
        stages_l = [0, 3] if args.quick else [0, 2, 3, 4]
        small = n * ho * ho <= 8 * 40 * 40
        splits_l = [int(v) for v in args.splits.split(",")] if small else [1]
        prods = [int(v) for v in args.producers.split(",")]
        best = None
        cat = {}
        tps_l = [int(v) for v in args.tps.split(",")]
        for halo, mt, bn, st, sp, pr, tps in itertools.product(halos, (1, 2), bns, stages_l, splits_l, prods, tps_l):
            if 2 * mt * bn > 512 or (not halo and tps != tps_l[0]):
                continue
            y = torch.full((n, ho, ho, cout), -7.0, device="cuda", dtype=dt)
            try:
                plan = ConvPlan(x, wp, b, y, n, hw, hw, cin, 0, cout, k, s, 0, block_n=bn, stages=st, halo=bool(halo), mt=mt, splits=sp, producers=pr, tps=tps)
            except L.B2TError as e:
                if args.verbose:
                    print("  %-8s halo %d mt %d bn %3d st %d sp %d: rejected (%s)" % (name, halo, mt, bn, st, sp, str(e)[-60:]))
                continue
            plan.run(); plan.run()
            torch.cuda.synchronize()
            err = (y.float() - ref).abs()
            bad = int((err > 2e-3 + 2e-3 * ref.abs()).sum())
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.reps):
                plan.run()
            e1.record()
            torch.cuda.synchronize()
            us = e0.elapsed_time(e1) * 1e3 / args.reps
            inf = plan.info
            tag = "halo %d mt %d bn %3d st %d(%d) sp %d P %d tps %d%s ob %d grid %3d smem %3dK" % (halo, mt, bn, st, inf["stages"], sp, pr, inf["tps"], "R" if inf["b_res"] else " ", inf["out_bufs"], inf["grid"], inf["smem"] // 1024)
            line = "  %-8s %s: %8.1f us %7.1f TFLOP/s  x%.2f of floor%s" % (name, tag, us, flops / us / 1e6, us / floor_us, "   WRONG: %d elems, max %.3g" % (bad, float(err.max())) if bad else "")
            if args.verbose or bad:
                print(line, flush=True)
            if not bad and (best is None or us < best[0]):
                best = (us, tag)
            key = "mt%d P%d" % (mt, pr)
            if not bad and (key not in cat or us < cat[key]):
                cat[key] = us
            del plan, y
        print("%-8s cin %4d cout %4d k%d s%d %3dx%-3d floor %6.1f us | best %7.1f us (x%.2f, %6.1f TFLOP/s): %s" %
              (name, cin, cout, k, s, hw, hw, floor_us, best[0], best[0] / floor_us, flops / best[0] / 1e6, best[1]), flush=True)
        print("           best per (mt, producers): " + "  ".join("%s %.1f" % (k_, v_) for k_, v_ in sorted(cat.items())), flush=True)
        summary.append((name, floor_us, best[0]))
        del x, w, ref
        torch.cuda.empty_cache()
    print("# sum of floors %.1f us, sum of best %.1f us over %d layers" % (sum(f for _, f, _ in summary), sum(b for _, _, b in summary), len(summary)))


if __name__ == "__main__":
    main()
