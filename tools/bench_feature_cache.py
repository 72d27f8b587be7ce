"""What the MVSNet feature cache saves on TANDEM's sliding keyframe window: 640x480, 7 views, reference at V-2, abl03,
mixed16.  Two handles run the same sliding sequence, one through CallAsync (FeatureNet on all 7 views, 7 uploads) and one
through CallAsyncIds (keyframe index as the id: FeatureNet on the one view each window adds, one upload); they alternate in
blocks of windows within one process.  The images cycle through a set of rendered frames while the ids keep increasing,
so every cached window adds exactly one new id.

    python tools/bench_feature_cache.py [--windows 200] [--warmup 20] [--block 10] [--iters 200]

Reports, with the card name and power limit read in the same run:
  * the median wall time of CallAsync -> GetResult per window, with pageable and with page-locked images and maps;
  * the device time per forward of the resident window (CUDA events, run_resident / run_resident_new): the full forward
    against the steady state (FeatureNet on the newest view only);
  * FeatureNet's share of one profiled full forward (per-kernel events, the f.* / preprocess rows).
Prints one JSON line."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tandem_b200 import DrMvsnet, DrMvsnetOutput, default_weights  # noqa: E402
from tandem_b200._lib import pinned_empty  # noqa: E402
from tandem_b200.synthetic import mvs_plane_window  # noqa: E402

H, W, V = 480, 640, 7
REF = V - 2
DMIN, DMAX, DISCARD = 0.5, 5.0, 2.5


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        q = f"nvidia-smi unavailable: {e}"
    return q


def wall_times(bgrs, c2ws, K, pinned, a):
    """Median ms of CallAsync -> GetResult per window, uncached and cached, alternating in blocks."""
    nimg = len(bgrs)
    weights = default_weights("abl03_view_aggregation")
    h = {"uncached": DrMvsnet(weights, precision="mixed16"), "cached": DrMvsnet(weights, precision="mixed16")}
    outs = {k: DrMvsnetOutput(H, W, pinned=pinned) for k in h}
    if pinned:
        for m in h.values():
            m.set_option("eager_d2h", 0)
    times = {k: [] for k in h}
    pos = {k: 0 for k in h}           # next window start (keyframe index) per handle
    total = a.warmup + a.windows
    path = "uncached"
    while min(pos.values()) < total:
        for _ in range(a.block):
            if pos[path] >= total:
                break
            m, w = h[path], pos[path]
            ids = list(range(w, w + V))
            imgs = [bgrs[i % nimg] for i in ids]
            poses = [c2ws[i % nimg] for i in ids]
            t0 = time.perf_counter()
            if path == "uncached":
                m.CallAsync(H, W, V, REF, imgs, K, poses, DMIN, DMAX, DISCARD)
            else:
                m.CallAsyncIds(H, W, V, REF, ids, [im if (w == 0 or i == w + V - 1) else None for i, im in zip(ids, imgs)], K,
                               poses, DMIN, DMAX, DISCARD)
            m.GetResult(out=outs[path])
            t1 = time.perf_counter()
            if w >= a.warmup:
                times[path].append((t1 - t0) * 1e3)
            pos[path] += 1
        path = "cached" if path == "uncached" else "uncached"
    assert h["cached"].feature_cache()[1] == 1
    for k in ("depth", "depth_dense"):   # the same last window on both handles
        assert np.array_equal(getattr(outs["cached"], k), getattr(outs["uncached"], k), equal_nan=True), k
    return {k: float(np.median(v)) for k, v in times.items()}, h["cached"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=200, help="timed windows per path")
    ap.add_argument("--warmup", type=int, default=20, help="untimed windows per path first")
    ap.add_argument("--block", type=int, default=10, help="windows per path before switching to the other")
    ap.add_argument("--iters", type=int, default=200, help="resident forwards per device-time sample")
    a = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_feature_cache: no CUDA device (this measurement only runs on the GPU)")
    nimg = 24
    win = mvs_plane_window(V=nimg, H=H, W=W, f=525.0, z_plane=2.0, baseline=0.02, seed=3)
    bgrs, c2ws, K = [np.ascontiguousarray(b) for b in win["bgrs"]], win["c2ws"], win["K"]
    res = {}
    wall_pageable, _ = wall_times(bgrs, c2ws, K, False, a)
    pb = []
    for b in bgrs:
        p = pinned_empty(b.shape, np.uint8)
        p[...] = b
        pb.append(p)
    wall_pinned, m = wall_times(pb, c2ws, K, True, a)
    res["wall_ms_pageable"] = wall_pageable
    res["wall_ms_pinned"] = wall_pinned

    # device time of the resident window on the cached handle: full forward vs FeatureNet on the newest view only
    m.run_resident(10)
    m.run_resident_new(1, 10)
    full, steady = [], []
    for _ in range(5):
        full.append(m.run_resident(a.iters)[0] / a.iters)
        steady.append(m.run_resident_new(1, a.iters)[0] / a.iters)
    res["device_ms_per_forward"] = {"full": float(np.median(full)), "n_new_1": float(np.median(steady)),
                                    "full_samples": full, "n_new_1_samples": steady}
    rows = m.profile()
    fnet = sum(r[1] for r in rows if r[0].startswith(("f.", "preprocess")))
    res["profiled_full_forward_ms"] = {"total": float(sum(r[1] for r in rows)), "featurenet": float(fnet)}
    print(json.dumps({
        "metric": "MVSNet feature cache on a sliding window: CallAsync -> GetResult wall medians and resident device time (ms)",
        "shape": f"{W}x{H}, {V} views, ref {REF}, abl03, mixed16", "windows_per_path": a.windows, "warmup_per_path": a.warmup,
        "block": a.block, "iters": a.iters, "card": card(), **res,
    }))


if __name__ == "__main__":
    main()
