"""One keyframe's tracking references at 640x480 with 4 levels (SURVEY 8f n7), two ways:

  host:   makeCoarseDepthL0 on the CPU (the C oracle, oracle/coarse_ref_oracle.c, standing in for the reference's host loops),
          then one setReference upload per level 1..3 and n1's dense call on level 0 (tdm_tracker_set_reference_dense with the
          sparse arrays and the idepth[0] image from the host)
  device: tdm_tracker_set_coarse_tracking_ref, one call

~2000 sparse points and a host dense depth map from a RoomScene keyframe.  The two paths alternate; each reports the median
wall time per keyframe (host clock around the blocking calls) and its device time (kernels + copies per keyframe, from a
torch.profiler run of its own).  The card's name and power limit are read in the same run.

    python tools/bench_coarse_ref.py [--iters 50] [--out out/bench_coarse_ref.json]
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle.coarse_ref import CoarseRefOracle  # noqa: E402
from tandem_b200 import ImagePyramid, set_coarse_tracking_ref  # noqa: E402
from test_coarse_ref_gpu import H, K0, L, W, fusion_render, room_keyframe, trackers  # noqa: E402

AFF = np.zeros(2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    gray, pts, T = room_keyframe()
    _, depth = fusion_render()
    pyr = ImagePyramid(W, H, L)
    pyr.build(gray)
    gray_levels = [np.ascontiguousarray(pyr.level(l)[0][..., 0]) for l in range(L)]
    dev_ts = trackers(W, H, L, K0)
    host_ts = trackers(W, H, L, K0)
    oracle = CoarseRefOracle(W, H, L)

    def device_path():
        return set_coarse_tracking_ref(dev_ts, pts, pyr, depth=depth, T_depth_to_ref=T, ref_aff_g2l=AFF)

    def host_path():
        pc_n, idepth0 = oracle._make_coarse_depth(oracle._l.coarse_ref_oracle, pts, gray_levels, False)
        for l in range(1, L):
            host_ts[l].setReference(pc_n[l], *[a[:pc_n[l]] for a in oracle.level_arrays(l)], 1.0, AFF)
        sparse = [a[:pc_n[0] + 1] for a in oracle.level_arrays(0)]
        pc_n[0] = host_ts[0].setReferenceDense(T, 1.0, AFF, depth=depth, dense_only=False, sparse=sparse, idepth0=idepth0,
                                               pyramid=pyr)
        return pc_n

    a, b = device_path(), host_path()
    assert a == b, (a, b)
    for l in range(L):   # same references both ways
        assert all(np.array_equal(x, y) for x, y in zip(dev_ts[l].getReference(a[l]), host_ts[l].getReference(b[l])))
    for _ in range(5):
        device_path(); host_path()
    wall = {"host": [], "device": []}
    for _ in range(args.iters):
        for name, f in (("host", host_path), ("device", device_path)):
            t0 = time.perf_counter()
            f()
            wall[name].append((time.perf_counter() - t0) * 1e3)
    dev_ms = {}
    for name, f in (("host", host_path), ("device", device_path)):
        n = 10
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(n):
                f()
        tot = sum(e.device_time_total for e in prof.key_averages())   # us over kernels and copies
        dev_ms[name] = tot / n / 1e3
    res = dict(gpu=gpu, size=[W, H], levels=L, points=int(len(pts[0])), pc_n=a, iters=args.iters,
               host=dict(median_wall_ms=float(np.median(wall["host"])), device_ms=dev_ms["host"]),
               device=dict(median_wall_ms=float(np.median(wall["device"])), device_ms=dev_ms["device"]))
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
