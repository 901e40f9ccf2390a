"""GPU: TFLOP/s of the wgmma conv kernel on the dominant YOLOv7-w6 shapes (batch 8) + whole-forward timing."""
import os, sys, json
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "yolov7-tracker_b200"))
import torch
from b200track.conv import ConvPlan, pack_conv_weight

def bench(n, h, cin, cout, k, s, reps=20):
    x = torch.randn((n, h, h, cin), device="cuda").to(torch.bfloat16)
    w = torch.randn((cout, cin, k, k), device="cuda") * 0.05
    b = torch.zeros(cout, device="cuda")
    ho = h // s
    y = torch.zeros((n, ho, ho, cout), dtype=torch.bfloat16, device="cuda")
    p = ConvPlan(x, pack_conv_weight(w), b, y, n, h, h, cin, 0, cout, k, s, 0)
    for _ in range(3): p.run()
    torch.cuda.synchronize()
    a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps): p.run()
    e.record(); torch.cuda.synchronize()
    ms = a.elapsed_time(e) / reps
    return ms, p.flops / ms / 1e9

if __name__ == "__main__":
    B = int(sys.argv[1]) if len(sys.argv) > 1 else 8
    shapes = [(320, 64, 64, 3, 1), (160, 128, 128, 3, 1), (80, 256, 256, 3, 1), (40, 384, 384, 3, 1), (640, 64, 128, 3, 2), (320, 128, 256, 3, 2),
              (160, 256, 512, 3, 2), (80, 512, 256, 1, 1), (20, 512, 512, 3, 1), (160, 256, 128, 1, 1), (640, 16, 64, 3, 1), (40, 1536, 384, 1, 1)]
    for h, ci, co, k, s in shapes:
        ms, tf = bench(B, h, ci, co, k, s)
        print("B=%d %4dx%-4d %4d->%-4d k%d s%d : %8.3f ms  %7.1f TFLOP/s" % (B, h, h, ci, co, k, s, ms, tf))
    from b200track.detector import DetectorW6
    from b200track.w6 import calibrated_state_dict
    det = DetectorW6(calibrated_state_dict(0, 1280, "cuda"), batch=B, img_size=1280, use_graph=True)
    g = torch.Generator().manual_seed(5)
    img = torch.rand((B, 3, 1280, 1280), generator=g).cuda()
    det.detect(img); torch.cuda.synchronize()
    for mode in ("graph",):
        a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(5): det.detect()
        e.record(); torch.cuda.synchronize()
        ms = a.elapsed_time(e) / 5
        print("detect (forward+decode+NMS) batch %d: %.2f ms -> %.1f img/s, %.1f TFLOP/s conv; dets/img %s" % (B, ms, B / ms * 1e3, det.flops / ms / 1e9, det.out_count.tolist()))
    # per-op breakdown without graph
    torch.cuda.synchronize()
    times = []
    for fn, fl, name in det.ops:
        a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); e.record(); torch.cuda.synchronize()
        times.append((a.elapsed_time(e), fl, name))
    tot = sum(t for t, _, _ in times)
    print("autotuned (BLOCK_N, stages, variant) per conv op:", {det.ops[i][2]: v for i, v in det.tuned.items()} if hasattr(det, "tuned") else None)
    print("sum of per-op times %.2f ms; conv flops %.1f GF/img" % (tot, det.flops / B / 1e9))
    for t, fl, name in sorted(times, key=lambda x: -x[0])[:25]:
        print("   %-22s %7.3f ms  %6.1f TF/s" % (name, t, fl / t / 1e9 if t > 0 else 0))
    a, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(); det._nms_launch(True); e.record(); torch.cuda.synchronize()
    det.decode()
    ncand = ((det.pred[..., 4] > 0.01) & ((det.pred[..., 5:] * det.pred[..., 4:5]).max(-1).values > 0.01)).sum(1)
    print("nms: %.3f ms; candidates per image %s of %d" % (a.elapsed_time(e), ncand.tolist(), det.n_total))
    print("obj logit stats per level:", [(float(r[..., 4::85].mean()), float(r[..., 4::85].std())) for r in det.raw])
