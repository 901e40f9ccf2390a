"""Writes tests/golden/w6_plan.json: the launch plan DetectorW6 builds (every b2t_conv_desc, op order, head levels) for two
input sizes, recorded WITHOUT a GPU by tests/plan_dryrun.py.  It was written from the build whose plan passed the GPU parity
tests of round 1, so that later planner changes can be checked against it on CPU.

    python tests/golden/make_golden_plan.py
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
for p in (ROOT, os.path.join(ROOT, "yolov7-tracker_b200"), os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)


def snapshot(batch, size):
    from plan_dryrun import dry_run_plan
    det, plan = dry_run_plan(batch, size)
    levels = [{"h": lv.h, "w": lv.w, "stride": lv.stride, "level_off": lv.level_off, "raw_pitch": lv.raw_pitch, "anchors": list(lv.anchors)}
              for lv in det.head_levels]
    return {"batch": batch, "size": size, "n_total": det.n_total, "ops": [n for _, _, n in det.ops], "convs": plan, "levels": levels, "launches": det.launch_log,
            "flops_ops": sum(1 for _, f, _ in det.ops if f > 0)}


if __name__ == "__main__":
    out = [snapshot(1, 256), snapshot(2, 640)]
    json.dump(out, open(os.path.join(HERE, "w6_plan.json"), "w"))
    print("wrote w6_plan.json:", [(s["batch"], s["size"], len(s["convs"]), s["n_total"]) for s in out])
