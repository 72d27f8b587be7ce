"""One keyframe's tracking references plus MVSNet's depth range at 640x480 with 4 levels, three ways:

  nodia:  tdm_tracker_set_coarse_tracking_ref_nodia, one call: n7 plus the undilated level-0 cloud and its 0.2 quantile
  n7:     tdm_tracker_set_coarse_tracking_ref alone (what an integrator runs today, next to the host work below)
  host:   the host work the nodia outputs replace: makeCoarseDepthL0 on the CPU (the C oracles oracle/coarse_ref_oracle.c,
          every level, and oracle/coarse_nodia_oracle.c, its undilated cloud, standing in for the reference's loops), then the
          0.2 quantile (np.partition, an nth_element)

For 2000 and 8000 sparse points from a RoomScene keyframe and a host dense depth map.  The three alternate; each reports the
median wall time per keyframe (host clock around the blocking calls) and, for the device paths, the device time (kernels +
copies per keyframe, from a torch.profiler run of its own).  The card's name and power limit are read in the same run.

    python tools/bench_coarse_nodia.py [--iters 50] [--out out/bench_coarse_nodia.json]
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

from oracle.coarse_nodia import CoarseNodiaOracle  # noqa: E402
from oracle.coarse_ref import CoarseRefOracle  # noqa: E402
from tandem_b200 import ImagePyramid, set_coarse_tracking_ref, set_coarse_tracking_ref_nodia  # noqa: E402
from test_coarse_ref_gpu import H, K0, L, W, fusion_render, room_keyframe, trackers  # noqa: E402

AFF = np.zeros(2)
FRACTION = 0.2


def run(n, depth, iters):
    import torch
    gray, pts, T = room_keyframe(0, n)
    pyr = ImagePyramid(W, H, L)
    pyr.build(gray)
    gray_levels = [np.ascontiguousarray(pyr.level(l)[0][..., 0]) for l in range(L)]
    nodia_ts, n7_ts = trackers(W, H, L, K0), trackers(W, H, L, K0)
    oracle, nodia_oracle = CoarseRefOracle(W, H, L), CoarseNodiaOracle(W, H)

    def nodia_path():
        return set_coarse_tracking_ref_nodia(nodia_ts, pts, pyr, FRACTION, depth=depth, T_depth_to_ref=T, ref_aff_g2l=AFF)

    def n7_path():
        return set_coarse_tracking_ref(n7_ts, pts, pyr, depth=depth, T_depth_to_ref=T, ref_aff_g2l=AFF)

    def host_path():
        oracle._make_coarse_depth(oracle._l.coarse_ref_oracle, pts, gray_levels, False)
        m = nodia_oracle.make(pts, gray_levels[0])
        ids = nodia_oracle.nodia[2 * W * H:2 * W * H + m]
        k = int(np.float32(np.float32(FRACTION) * np.float32(m)))
        return m, np.float32(1.0) / np.partition(ids, k)[k]

    (pc_n, m, dq), pc_n7, (hm, hdq) = nodia_path(), n7_path(), host_path()
    assert pc_n == pc_n7 and m == hm and np.float32(dq) == hdq, (pc_n, pc_n7, m, hm, dq, hdq)
    paths = (("nodia", nodia_path), ("n7", n7_path), ("host", host_path))
    for _ in range(5):
        for _, f in paths:
            f()
    wall = {name: [] for name, _ in paths}
    for _ in range(iters):
        for name, f in paths:
            t0 = time.perf_counter()
            f()
            wall[name].append((time.perf_counter() - t0) * 1e3)
    res = dict(points=n, pc_n=pc_n, pc_n_nodia=m, depth_quantile=float(dq))
    for name, f in paths:
        r = dict(median_wall_ms=float(np.median(wall[name])))
        if name != "host":
            k = 10
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(k):
                    f()
            r["device_ms"] = sum(e.device_time_total for e in prof.key_averages()) / k / 1e3   # us over kernels and copies
        res[name] = r
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()[0]
    _, depth = fusion_render()
    line = json.dumps(dict(gpu=gpu, size=[W, H], levels=L, fraction=FRACTION, iters=args.iters,
                           runs=[run(n, depth, args.iters) for n in (2000, 8000)]))
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
