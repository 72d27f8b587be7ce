"""n8: one traceNewCoarse at 640x480 with 7 active keyframes of ~1500 immature points each, two workloads:

  fresh:   points just added (idepth_max NaN): every point runs the full search over maxPixSearch = 0.027 (w + h) pixels
  traced:  the same points after three traces into nearby frames: most skip, a few search their shorter intervals

For each, the device path (ImmaturePoints.trace, one launch for all hosts) is timed as the median wall time of one call
(host clock around the trace and the synchronising count() behind it) and the median kernel time (torch.profiler, CUDA
activity of k_trace, in a run of its own), against the single-thread CPU time of the C oracle (oracle/trace_oracle.c, the
reference's statements in C) on the same points and frame.  The card's name and power limit are read in the same run.

    python tools/bench_trace.py [--iters 30] [--out out/bench_trace.json]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import trace as T  # noqa: E402
from oracle.cpu import FrontOracle  # noqa: E402
from oracle.pins_coarse_ref import K4  # noqa: E402
from tandem_b200 import ImagePyramid, ImmaturePoints  # noqa: E402

W, H, HOSTS, POINTS = 640, 480, 7, 1500


def scene():
    front = FrontOracle()
    rng = np.random.default_rng(5)
    hosts = []
    for j in range(HOSTS):
        p = T.pose(j - 6.0)
        g = T.gray(p, H, W).astype(np.float32)
        dI = T.level0(g, front)
        u, v = T.select(dI, POINTS, rng)
        hosts.append(dict(slot=j, pose=p, gray=g, dI=dI, u=u, v=v))
    frames = []
    for k in (0.5, 1.0, 1.5, 2.0):
        c2w = T.pose(k)
        g = T.gray(c2w, H, W).astype(np.float32)
        frames.append(dict(gray=g, dI=T.level0(g, front),
                           params=[T.frame_params("real", c2w, hh["pose"], K4(H, W)) for hh in hosts]))
    return hosts, frames


def prepare(d, hosts, hp, frames, fp, traced):
    n = 0
    for hh, p in zip(hosts, hp):
        d.drop_host(hh["slot"])
        n += d.add(hh["slot"], p, hh["u"], hh["v"])
    if traced:
        for f, p in zip(frames[:3], fp[:3]):
            trace(d, hosts, f, p)
    d.count(0)
    return n


def trace(d, hosts, f, p):
    d.trace(p, [hh["slot"] for hh in hosts], [q[0] for q in f["params"]], [q[1] for q in f["params"]],
            [q[2] for q in f["params"]])


def cpu_ms(hosts, frames, traced, iters):
    ts = []
    for _ in range(iters):
        o = T.TraceOracle(W, H)
        for hh in hosts:
            o.add(hh["slot"], hh["dI"], hh["u"], hh["v"])
        if traced:
            for f in frames[:3]:
                o.trace(f["dI"], {hh["slot"]: f["params"][j] for j, hh in enumerate(hosts)})
        f = frames[3]
        t0 = time.perf_counter()
        o.trace(f["dI"], {hh["slot"]: f["params"][j] for j, hh in enumerate(hosts)})
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    card = smi.stdout.strip().splitlines()[0] if smi.returncode == 0 else "unknown"
    hosts, frames = scene()
    hp = [ImagePyramid(W, H, 1) for _ in hosts]
    for p, hh in zip(hp, hosts):
        p.build(hh["gray"])
    fp = [ImagePyramid(W, H, 1) for _ in frames]
    for p, f in zip(fp, frames):
        p.build(f["gray"])
    d = ImmaturePoints(W, H, 2048)
    res = dict(card=card, w=W, h=H, hosts=HOSTS)
    for name, traced in (("fresh", False), ("traced", True)):
        wall = []
        for it in range(a.iters + 3):
            n = prepare(d, hosts, hp, frames, fp, traced)
            t0 = time.perf_counter()
            trace(d, hosts, frames[3], fp[3])
            d.count(0)
            if it >= 3:
                wall.append((time.perf_counter() - t0) * 1e3)
        kern = []
        for _ in range(5):
            prepare(d, hosts, hp, frames, fp, traced)
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                trace(d, hosts, frames[3], fp[3])
                d.count(0)
                torch.cuda.synchronize()
            kern += [e.device_time_total / 1e3 for e in prof.events() if "k_trace" in e.name]
        st = np.concatenate([d.get(hh["slot"])["status"] for hh in hosts])
        res[name] = dict(points=int(n), wall_ms=float(np.median(wall)), kernel_ms=float(np.median(kern)) if kern else None,
                         cpu_oracle_ms=cpu_ms(hosts, frames, traced, 5), status_counts=np.bincount(st, minlength=6).tolist())
        print(name, res[name], flush=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
