"""GPU box: per-conv-launch table of one detector step (batch 8, 1280 x 1280) WITHOUT a profiler: the autotuned configuration of
every launch, its time alone (back-to-back CUDA-event timing, the autotuner's own number) and its time INSIDE the step
(difference between the CUDA graphs of ops[0..k] and ops[0..k-1], programmatic dependent launch overlap included), next to the
layer's floors: flops / sustained tensor peak and algorithmic bytes / HBM peak (MEASURED_PEAKS.json, else the H100 SXM data sheet:
989 TFLOP/s dense fp16, 3 350 GB/s -- a power-capped card reaches less, so the floors are optimistic there).  'pp' / 'co' = consumer
schedule: ping-pong (one warpgroup's epilogue under the other's MMAs) or cooperative; 'run' / 'pat' = the 128 pixels of a sub-tile
are a run of the flattened output axis (tile_w = 128, im2col boxes) or a spatial patch (3x3 layers; 1x1 layers are always runs).

    python tools/conv_graph_table.py [out.txt]
"""
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "yolov7-tracker_b200")):
    sys.path.insert(0, p)


def graph_ms(fns, dev, reps=20):
    s = torch.cuda.Stream(device=dev)
    with torch.cuda.stream(s):
        for fn in fns:
            fn()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            for fn in fns:
                fn()
        g.replay(); torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(s)
        for _ in range(reps):
            g.replay()
        b.record(s)
        torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main(out_path=None, batch=8, size=1280):
    from b200track.detector import DetectorW6
    from b200track.w6 import calibrated_state_dict
    dev = torch.device("cuda:0")
    sd = calibrated_state_dict(0, size, dev)
    det = DetectorW6(sd, batch=batch, img_size=size, device=dev, use_graph=False)
    peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))) if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else {}
    peak, hbm = float(peaks.get("bf16_tflops_sustained", 989.0)) * 1e12, float(peaks.get("hbm_gbs", 3350.0)) * 1e9
    fns = [fn for fn, _, _ in det.ops]
    plans = [p for p in det.keep if hasattr(p, "geom")]
    out, tot_in, tot_alone, tot_floor, worst, pi = [], 0.0, 0.0, 0.0, (0.0, ""), 0
    prev = graph_ms(fns[:1], dev)
    for k in range(1, len(fns)):
        cur = graph_ms(fns[:k + 1], dev)
        fl, name = det.ops[k][1], det.ops[k][2]
        d_us, prev = (cur - prev) * 1e3, cur
        if fl <= 0:
            out.append("%-24s %-34s %35s in-graph %7.1f us" % (name, "(glue)", "", d_us))
            continue
        plan = plans[pi]; pi += 1
        g, inf, t = plan.geom, plan.info, det.tuned.get(k, {})
        ho, wo = g["h"] // g["stride"], g["w"] // g["stride"]
        cin = 12 if g["rowpack"] else g["cin"]
        by = g["n"] * (g["h"] * g["w"] * cin * 2 + ho * wo * g["cout"] * (4 if g["out_f32"] else 2)) + g["k"] * g["k"] * cin * g["cout"] * 2
        tf, th = fl / peak * 1e6, by / hbm * 1e6
        floor, alone = max(tf, th), t.get("us", float("nan"))
        px = "run" if g["k"] == 1 or t.get("tile_w") == 128 else "pat"
        cfg = "%4d>%4d k%d s%d %3dx%-3d bn%3d mt%d %s %s st%d v%d g%3d" % (g["cin"], g["cout"], g["k"], g["stride"], g["h"], g["w"], inf["bn"], inf["mt"],
                                                                "pp" if inf["pingpong"] else "co", px, inf["stages"], t.get("variant", 0), inf["grid"])
        out.append("%-24s %-55s alone %6.1f  in-graph %6.1f us %6.0f TFLOP/s  floor %6.1f (%s) x%4.1f" %
                   (name.replace("model.", "L").replace(".conv", ""), cfg, alone, d_us, fl / max(d_us, 1e-3) / 1e6, floor, "tensor" if tf >= th else "hbm", d_us / floor))
        tot_in += d_us; tot_alone += alone; tot_floor += floor
        if d_us / floor > worst[0]:
            worst = (d_us / floor, name)
    hdr = ["# one detector step, batch %d, %dx%d, fp16 activations: autotuned configuration per conv launch; 'alone' = back-to-back launches of that" % (batch, size, size),
           "# plan (CUDA events), 'in-graph' = graph(ops[0..k]) - graph(ops[0..k-1]) (what the launch adds to the step, PDL overlap included);",
           "# floor = max(flops / %.0f TFLOP/s, algorithmic bytes / %.0f GB/s) (MEASURED_PEAKS.json, else the H100 SXM data sheet)" % (peak / 1e12, hbm / 1e9)]
    tail = ["# conv launches: in-graph %.1f us, alone %.1f us, sum of floors %.1f us; worst launch x%.1f (%s); whole forward graph %.1f us" %
            (tot_in, tot_alone, tot_floor, worst[0], worst[1], prev * 1e3)]
    text = "\n".join(hdr + out + tail)
    print(text)
    if out_path:
        open(out_path, "w").write(text + "\n")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else None)
