"""n13 benchmark: medians of ActivePoints.accumulate and resubstitute on the room window and a seeded 2000-point window at
640x480, 8 frames, against n12's linearize with and without the Jacobian download and apply_res (which now also takes the
data) in the same run, the C oracle's accumulate in the reference's float-tier mode on one CPU thread, and the kernels'
time from torch.profiler in a run of its own.  Prints the card's name and power limit and one JSON line."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import accumulate as A  # noqa: E402
from oracle import linearize as L  # noqa: E402
from tandem_b200 import ActivePoints, ImagePyramid  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        return f"unknown ({e})"


def med(f, iters):
    t = []
    for _ in range(iters):
        t0 = time.perf_counter()
        f()
        t.append(time.perf_counter() - t0)
    return float(np.median(t)) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--profile", action="store_true")
    a = ap.parse_args()
    out = dict(card=card())
    for name in ("room", "seeded"):
        win = A.case(name)
        inp = A.inputs(win)
        fp = []
        for g in win["gray"]:
            p = ImagePyramid(win["w"], win["h"], 1)
            p.build(np.ascontiguousarray(g, np.float32))
            fp.append(p)
        d = ActivePoints(win["w"], win["h"], len(win["host"]))
        d.load(win["n_frames"], win["host"], win["u"], win["v"], win["color"], win["weights"], win["res_point"], win["res_target"])
        pc = A.precalc(win)
        lin = lambda j: d.linearize(fp, pc, win["frame_th"], win["calib4"], win["idepth"], win["idepth"], jacobians=j)
        lin(False)
        d.apply_res()
        x = A.solve(d.accumulate(**inp))
        for _ in range(5):
            d.accumulate(**inp)
            d.resubstitute(x)
        r = dict(residuals=len(win["res_point"]), points=len(win["host"]))
        if a.profile:
            import torch
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(a.iters):
                    d.accumulate(**inp)
                    d.resubstitute(x)
                    d.apply_res()
                torch.cuda.synchronize()
            ker = {}
            for e in prof.key_averages():
                if e.device_type.name == "CUDA" and "k_" in e.key:
                    ker[e.key] = ker.get(e.key, 0.0) + e.device_time_total / a.iters / 1e3
            r["kernel_ms_per_iteration"] = {k.split("k_")[-1][:24]: round(v, 4) for k, v in ker.items() if "k_" in k}
        else:
            r["accumulate_ms"] = med(lambda: d.accumulate(**inp), a.iters)
            r["resubstitute_ms"] = med(lambda: d.resubstitute(x), a.iters)
            r["linearize_no_jacobians_ms"] = med(lambda: lin(False), a.iters)
            r["linearize_with_jacobians_ms"] = med(lambda: lin(True), a.iters)
            import torch
            r["apply_res_ms"] = med(lambda: (d.apply_res(), torch.cuda.synchronize()), a.iters)   # the set's stream included
            o = A.AccumulateOracle(win)
            o.linearize(win["idepth"], win["idepth"], pc, win["frame_th"], 0)
            o.apply_res()
            r["oracle_tiers_ms"] = med(lambda: o.accumulate(inp, A.TIERS), max(3, a.iters // 10))
        out[name] = r
    print(json.dumps(out))


if __name__ == "__main__":
    main()
