"""n9: activatePointsMT's solve (optimizeImmaturePoint for every candidate) at 640x480 with 8 frames - 7 hosts of 1500
immature points each, traced three times, and the newest keyframe - for two candidate lists:

  all:     every activatable point (canActivate of FullSystem.cpp:769-774)
  subset:  500 of them

For each, the device path (ImmaturePoints.activate, one launch, blocking) is timed as the median wall time of one call and
the median kernel time (torch.profiler, CUDA activity of k_activate, in a run of its own), against the single-thread CPU
time of the C oracle (oracle/activate_oracle.c, the reference's statements in C) on the same candidates.  The card's name
and power limit are read in the same run.

    python tools/bench_activate.py [--iters 30] [--out out/bench_activate.json]
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

from oracle import activate as A  # noqa: E402
from oracle import trace as T  # noqa: E402
from oracle.cpu import FrontOracle  # noqa: E402
from oracle.pins_coarse_ref import K4  # noqa: E402
from tandem_b200 import ImagePyramid, ImmaturePoints  # noqa: E402

W, H, HOSTS, POINTS = 640, 480, 7, 1500


def window():
    front = FrontOracle()
    rng = np.random.default_rng(5)
    frames = []
    for j in range(HOSTS + 1):
        p = T.pose(j - 6.0)
        g = T.gray(p, H, W).astype(np.float32)
        dI = T.level0(g, front)
        f = dict(slot=j if j < HOSTS else -1, pose=p, gray=g, dI=dI)
        if j < HOSTS:
            u, v = T.select(dI, POINTS, rng)
            f.update(u=u, v=v, type=np.ones(len(u), np.float32), u2=u[:0], v2=v[:0])
        frames.append(f)
    traces = []
    for k in (0.5, 1.0, 1.5):
        c2w = T.pose(k)
        g = T.gray(c2w, H, W).astype(np.float32)
        traces.append(dict(gray=g, dI=T.level0(g, front),
                           params={f["slot"]: T.frame_params("real", c2w, f["pose"], K4(H, W)) for f in frames[:HOSTS]}))
    n = HOSTS + 1
    pc = np.full((n, n, 14), np.nan, np.float32)
    for a in range(n):
        for b in range(n):
            if a != b:
                Tm = np.linalg.inv(frames[b]["pose"]) @ frames[a]["pose"]
                pc[a, b, :9] = Tm[:3, :3].astype(np.float32).ravel()
                pc[a, b, 9:12] = Tm[:3, 3].astype(np.float32)
                pc[a, b, 12:] = (1.0, 0.0)
    return dict(w=W, h=H, calib4=np.array(K4(H, W), np.float32), frames=frames, traces=traces, precalc=pc,
                variants=[({}, "act")])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    card = smi.stdout.strip().splitlines()[0] if smi.returncode == 0 else "unknown"
    c = window()
    o = A.build_points(c)
    d = ImmaturePoints(W, H, 2048)
    fp = []
    for f in c["frames"]:
        p = ImagePyramid(W, H, 1)
        p.build(f["gray"])
        fp.append(p)
        if f["slot"] >= 0:
            d.add(f["slot"], p, f["u"], f["v"])
    for t in c["traces"]:
        tp = ImagePyramid(W, H, 1)
        tp.build(t["gray"])
        slots = [f["slot"] for f in c["frames"][:HOSTS]]
        d.trace(tp, slots, [t["params"][s][0] for s in slots], [t["params"][s][1] for s in slots],
                [t["params"][s][2] for s in slots])
    (s, cf_all, ci_all, r_all), = A.run_oracle(c, o)
    sub = np.sort(np.random.default_rng(1).choice(len(cf_all), 500, replace=False))
    slots = [f["slot"] for f in c["frames"]]
    res = dict(card=card, w=W, h=H, frames=HOSTS + 1, points=int(sum(d.count(f["slot"]) for f in c["frames"][:HOSTS])))
    for name, idx in (("all", np.arange(len(cf_all))), ("subset", sub)):
        cf, ci = cf_all[idx], ci_all[idx]
        got = d.activate(slots, fp, c["precalc"], c["calib4"], cf, ci)
        same = bool(np.array_equal(got["result"], r_all["result"][idx]))
        wall = []
        for it in range(a.iters + 3):
            t0 = time.perf_counter()
            d.activate(slots, fp, c["precalc"], c["calib4"], cf, ci)
            if it >= 3:
                wall.append((time.perf_counter() - t0) * 1e3)
        kern = []
        for _ in range(5):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                d.activate(slots, fp, c["precalc"], c["calib4"], cf, ci)
                torch.cuda.synchronize()
            kern += [e.device_time_total / 1e3 for e in prof.events() if "k_activate" in e.name]
        cpu = []
        recs = np.concatenate([A.point_records(o.pts[slots[j]], ci[cf == j]) for j in np.unique(cf)])
        order = np.concatenate([np.flatnonzero(cf == j) for j in np.unique(cf)])
        for _ in range(5):
            t0 = time.perf_counter()
            A.activate(W, H, [f["dI"] for f in c["frames"]], c["precalc"], c["calib4"], cf[order], recs)
            cpu.append((time.perf_counter() - t0) * 1e3)
        res[name] = dict(candidates=int(len(cf)), wall_ms=float(np.median(wall)), kernel_ms=float(np.median(kern)) if kern else None,
                         cpu_oracle_ms=float(np.median(cpu)), equals_oracle=same,
                         results=dict(zip(*[x.tolist() for x in np.unique(got["result"], return_counts=True)])))
        print(name, res[name], flush=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
