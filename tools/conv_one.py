"""GPU box: run ONE configuration of one w6 layer a few times (for a profiler).  python tools/conv_one.py L23 halo=1 mt=1 bn=256 stages=0 producers=2 splits=1"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "yolov7-tracker_b200"), os.path.join(ROOT, "tools")):
    sys.path.insert(0, p)
from conv_layer_bench import LAYERS  # noqa: E402
from b200track.conv import ConvPlan, pack_conv_weight  # noqa: E402

name = sys.argv[1]
kw = dict(halo=0, mt=1, bn=0, stages=0, producers=0, splits=1, reps=3, batch=8)
for a in sys.argv[2:]:
    k, v = a.split("=")
    kw[k] = int(v)
cin, cout, k, s, hw = LAYERS[name]
n = kw["batch"]
dt = torch.float16
x = torch.randn((n, hw, hw, cin), device="cuda").to(dt)
w = torch.randn((cout, cin, k, k), device="cuda") * (1.5 / (cin * k * k) ** 0.5)
b = torch.randn(cout, device="cuda") * 0.5
y = torch.zeros((n, hw // s, hw // s, cout), device="cuda", dtype=dt)
plan = ConvPlan(x, pack_conv_weight(w, dtype=dt), b, y, n, hw, hw, cin, 0, cout, k, s, 0, block_n=kw["bn"], stages=kw["stages"], halo=bool(kw["halo"]),
                mt=kw["mt"], splits=kw["splits"], producers=kw["producers"])
print(name, kw, plan.info)
for _ in range(kw["reps"]):
    plan.run()
torch.cuda.synchronize()
