"""DeepSORT's gallery appearance cost on the tensor cores (b2t_gallery_distance) at the C4 scale.

    python tools/gallery_bench.py [--slots 2800] [--budget 100] [--dets 300] [--dim 512] [--iters 50]

The default is one frame of 8 sequences x about 350 pool tracks with full 100-entry galleries against 300 detection rows at
feat_dim 512, as one launch.  Prints the card's name and power limit, then the kernel time (CUDA events over --iters launches after
warm-up, median of 5 windows) and the packing of the detection rows (b2t_gallery_pack), with
  * the tensor work: 3 fp16 products per multiply-add (hi.hi + hi.lo + lo.hi), 2 flops each, against the data sheet's dense
    989 TFLOP/s fp16 for the H100 SXM;
  * the gallery bytes read once per frame, against the data sheet's 3.35 TB/s of HBM3.
Nothing is written."""
import argparse
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "yolov7-tracker_b200"))
from b200track.engine import ops                     # noqa: E402

FP16_TENSOR_FLOPS = 989e12
HBM_BYTES_PER_S = 3.35e12


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True).stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name()


def timed(fn, iters):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    times = []
    for _ in range(5):
        ev[0].record()
        for _ in range(iters):
            fn()
        ev[1].record()
        torch.cuda.synchronize()
        times.append(ev[0].elapsed_time(ev[1]) / iters)
    return sorted(times)[2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--slots", type=int, default=2800)
    ap.add_argument("--budget", type=int, default=100)
    ap.add_argument("--dets", type=int, default=300)
    ap.add_argument("--dim", type=int, default=512)
    ap.add_argument("--iters", type=int, default=50)
    a = ap.parse_args()
    o = ops()
    g = torch.Generator(device="cuda").manual_seed(0)
    gal = o.gallery_pack(torch.randn((a.slots, a.budget, a.dim), device="cuda", generator=g))
    det_f = torch.randn((a.dets, a.dim), device="cuda", generator=g)
    dets = o.gallery_pack(det_f)
    counts = torch.full((a.slots,), a.budget, dtype=torch.int32, device="cuda")
    for _ in range(10):
        o.gallery_distance(gal, counts, dets, a.dim)
    torch.cuda.synchronize()
    ms = timed(lambda: o.gallery_distance(gal, counts, dets, a.dim), a.iters)
    ms_pack = timed(lambda: o.gallery_pack(det_f), a.iters)
    mac = float(a.slots) * a.budget * a.dets * a.dim
    flops = 3 * 2 * mac
    gbytes = float(gal.numel()) * 2
    t_flop, t_hbm = flops / FP16_TENSOR_FLOPS * 1e3, gbytes / HBM_BYTES_PER_S * 1e3
    print("card: %s" % card())
    print("gallery distance: %d slots x %d entries x %d detections x %d dims (%.1f G multiply-adds, %.0f MB of gallery)"
          % (a.slots, a.budget, a.dets, a.dim, mac / 1e9, gbytes / 1e6))
    print("  kernel %.3f ms: %.0f TFLOP/s of fp16 tensor work (bound %.3f ms at 989 TFLOP/s), %.2f TB/s of gallery "
          "(bound %.3f ms at 3.35 TB/s)" % (ms, flops / ms / 1e9, t_flop, gbytes / ms / 1e9, t_hbm))
    print("  share of the larger bound: %.0f %%" % (100 * max(t_flop, t_hbm) / ms))
    print("  packing %d detection rows: %.4f ms" % (a.dets, ms_pack))


if __name__ == "__main__":
    main()
