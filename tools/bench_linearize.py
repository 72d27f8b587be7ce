"""n12: linearizeAll on the device (ActivePoints.linearize, one launch chain, blocking) at 640x480 with 8 frames, for two
windows of oracle/linearize.py:

  room:    the points n9's C oracle activates on room_640x480_8f, with their IN residuals
  seeded:  2000 points at the scene's depth, each with a random subset of the other frames as targets

Each window runs the optimize()-shaped sequence of oracle/linearize.py (linearize -> apply, perturbed -> apply, perturbed,
linearize(fix)) over and over.  Reported per window, as medians over the calls: the wall time of one linearize call without
the Jacobian download, with it into pageable memory, and with it into page-locked memory; the kernel time of one call
(torch.profiler, CUDA activity of the call's kernels, in a run of its own); and the single-thread CPU time of the C oracle
(oracle/linearize_oracle.c, the reference's statements in C) for the same call.  The card's name and power limit are read in
the same run.

    python tools/bench_linearize.py [--iters 25] [--out out/bench_linearize.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import linearize as L  # noqa: E402
from tandem_b200 import ActivePoints, ImagePyramid  # noqa: E402
from tandem_b200._lib import pinned_empty  # noqa: E402

KERNELS = ("k_linearize", "k_finish", "k_points", "DeviceRadixSort", "Onesweep", "Histogram", "Exclusive")


class Device:
    """ActivePoints with the call signature of oracle/linearize.py's run_sequence."""

    def __init__(self, d, fp, calib4):
        self.d, self.fp, self.calib4 = d, fp, calib4

    def linearize(self, ids, idz, precalc, frame_th, fix):
        return self.d.linearize(self.fp, precalc, frame_th, self.calib4, ids, idz, fix=fix)

    def apply_res(self):
        self.d.apply_res()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=25)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    card = smi.stdout.strip().splitlines()[0] if smi.returncode == 0 else "unknown"
    res = dict(card=card)
    for name, win in (("room", L.window("room", "base")), ("seeded", L.window("seeded", "base"))):
        fp = []
        for g in win["gray"]:
            p = ImagePyramid(win["w"], win["h"], 1)
            p.build(np.ascontiguousarray(g, np.float32))
            fp.append(p)
        d = ActivePoints(win["w"], win["h"], len(win["host"]), **win["settings"])
        m = len(win["res_point"])
        seq = L.steps(win)
        pinned = dict(jacobians=pinned_empty((m, L.JACOBIAN_FLOATS), np.float32))

        def sequence(mode, times):
            d.load(win["n_frames"], win["host"], win["u"], win["v"], win["color"], win["weights"], win["res_point"], win["res_target"])
            th = win["frame_th"].copy()
            for st in seq:
                kw = dict(jacobians=mode != "none", out=pinned if mode == "pinned" else None)
                t0 = time.perf_counter()
                r = d.linearize(fp, st["precalc"], th, win["calib4"], st["idepth_scaled"], st["idepth_zero_scaled"], fix=st["fix"], **kw)
                times.append((time.perf_counter() - t0) * 1e3)
                if st["apply"]:
                    d.apply_res()
                th[-1] = r["new_frame_energy_th"]
            return r

        out = dict(points=len(win["host"]), residuals=m)
        o = L.LinearizeOracle(win)
        ref = L.run_sequence(o, win)
        d.load(win["n_frames"], win["host"], win["u"], win["v"], win["color"], win["weights"], win["res_point"], win["res_target"])
        dev = L.run_sequence(Device(d, fp, win["calib4"]), win)
        out["equals_oracle"] = all(L.compare(b, x, exact_energy=False) == [] for (_, x, _), (_, b, _) in zip(ref, dev))
        for mode in ("none", "pageable", "pinned"):
            t = []
            for it in range(a.iters + 1):
                sequence(mode, t if it > 0 else [])
            out[f"wall_ms_{mode}"] = float(np.median(t))
        kern = []
        for _ in range(3):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                st = seq[0]
                d.linearize(fp, st["precalc"], win["frame_th"], win["calib4"], st["idepth_scaled"], st["idepth_zero_scaled"],
                            jacobians=False)
                torch.cuda.synchronize()
            kern.append(sum(e.device_time_total for e in prof.events()
                            if e.device_time_total > 0 and any(k in e.name for k in KERNELS)) / 1e3)
        out["kernel_ms"] = float(np.median(kern))
        cpu = []
        for _ in range(5):
            o.load()
            st = seq[0]
            t0 = time.perf_counter()
            o.linearize(st["idepth_scaled"], st["idepth_zero_scaled"], st["precalc"], win["frame_th"], 0)
            cpu.append((time.perf_counter() - t0) * 1e3)
        out["cpu_oracle_ms"] = float(np.median(cpu))
        out["jacobian_mb"] = m * L.JACOBIAN_FLOATS * 4 / 1e6
        res[name] = out
        print(name, out, flush=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
