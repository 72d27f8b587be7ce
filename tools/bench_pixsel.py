"""n10: a new keyframe's pixel selection at 640x480 on 8 RoomScene keyframes, density 1500 (setting_desiredImmatureDensity):

  make_new_traces  ImmaturePoints.make_new_traces: makeMaps and the ImmaturePoint constructor, the map kept on the device
  make_maps        PixelSelector.make_maps with the map copied back to the host

Each keyframe's call starts from the potential the keyframe sequence gives it (carried from keyframe to keyframe, as in DSO),
so every repetition does the same work.  Reported per path: the median wall time of one blocking call and the median kernel
time of one call (torch.profiler, the CUDA activity of every kernel of the call, in a run of its own), and for
make_new_traces the median time of k_chain alone (the serial walk of the cells).  Against it: the single-thread CPU time of
the C oracles on the same pyramid (oracle/pixsel_oracle.c: makeHists + makeMaps; oracle/trace_oracle.c: the constructor for
the selected pixels).  Also per keyframe: the potential, whether it re-selected, the selected and kept points, and the
cells whose selection depends on their direction (the cells k_chain resolves one by one).  The card's name and power limit
are read in the same run.

    python tools/bench_pixsel.py [--iters 20] [--out out/bench_pixsel.json]
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

from oracle import pixsel as P  # noqa: E402
from oracle import trace as T  # noqa: E402
from tandem_b200 import ImagePyramid, ImmaturePoints, PixelSelector  # noqa: E402

W, H, KEYFRAMES, DENSITY = 640, 480, 8, 1500.0
KERNELS = ("k_hist", "k_smooth", "k_mask", "k_chain", "k_pick", "k_decide", "k_rowcount", "k_scan", "k_subsample", "k_emit",
           "k_add")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    card = smi.stdout.strip().splitlines()[0] if smi.returncode == 0 else "unknown"
    grays = [T.gray(T.pose(0.8 * k), H, W).astype(np.float32) for k in range(KEYFRAMES)]
    lv = [P.levels(g) for g in grays]
    pyr = []
    for g in grays:
        p = ImagePyramid(W, H, 3)
        p.build(g)
        pyr.append(p)
    # the sequence on the oracle: each keyframe's starting potential, and what the device must give
    o = P.PixelSelectorOracle(W, H)
    seq = [o.make_maps_on(dI, ag, DENSITY) for dI, ag in lv]
    sel = PixelSelector(W, H)
    d = ImmaturePoints(W, H, 8000)
    per_kf, same = [], True
    for k, r in enumerate(seq):
        sel.potential = r["pot_before"]
        m, got = sel.make_maps(pyr[k], DENSITY)
        same &= bool(np.array_equal(m, r["map"])) and got["num_selected"] == r["ret"]
        u, v, t = P.new_traces(r["map"], W, H)
        sel.potential = r["pot_before"]
        nt = d.make_new_traces(0, sel, pyr[k], DENSITY)
        d.drop_host(0)
        to = T.TraceOracle(W, H)
        kept = to.add(0, lv[k][0], u, v, t)
        same &= nt["n_added"] == kept and bool(np.array_equal(nt["u"], to.pts[0]["u"].astype(np.int32)))
        per_kf.append(dict(potential_before=r["pot_before"], potential_used=r["pot_used"], reselected=r["reselected"],
                           selected=r["ret"], kept=nt["n_added"], nonuniform_cells=got["nonuniform_cells"],
                           cells=-(-W // r["pot_used"]) * -(-H // r["pot_used"])))

    def run_nt(k):
        sel.potential = seq[k]["pot_before"]
        d.make_new_traces(0, sel, pyr[k], DENSITY)
        d.drop_host(0)

    def run_mm(k):
        sel.potential = seq[k]["pot_before"]
        sel.make_maps(pyr[k], DENSITY)

    res = dict(card=card, w=W, h=H, keyframes=KEYFRAMES, density=DENSITY, equals_oracle=same, per_keyframe=per_kf)
    for name, fn in (("make_new_traces", run_nt), ("make_maps", run_mm)):
        for k in range(KEYFRAMES):
            fn(k)
        wall = []
        for _ in range(a.iters):
            for k in range(KEYFRAMES):
                t0 = time.perf_counter()
                fn(k)
                wall.append((time.perf_counter() - t0) * 1e3)
        kern, per = [], {n: [] for n in KERNELS}
        for _ in range(3):
            for k in range(KEYFRAMES):
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    fn(k)
                    torch.cuda.synchronize()
                ev = [e for e in prof.events() if any(n in e.name for n in KERNELS)]
                kern.append(sum(e.device_time_total for e in ev) / 1e3)
                for n in KERNELS:
                    per[n].append(sum(e.device_time_total for e in ev if n + "(" in e.name or n + "<" in e.name) / 1e3)
        res[name] = dict(wall_ms=float(np.median(wall)), kernel_ms=float(np.median(kern)), chain_ms=float(np.median(per["k_chain"])),
                         per_kernel_ms={n: float(np.median(v)) for n, v in per.items() if max(v) > 0})
        print(name, res[name], flush=True)
    cpu = []
    for _ in range(3):
        for k, (dI, ag) in enumerate(lv):
            oo = P.PixelSelectorOracle(W, H)
            oo.rp = o.rp
            oo.potential = seq[k]["pot_before"]
            t0 = time.perf_counter()
            r = oo.make_maps_on(dI, ag, DENSITY)
            u, v, t = P.new_traces(r["map"], W, H)
            T.TraceOracle(W, H).add(0, dI, u, v, t)
            cpu.append((time.perf_counter() - t0) * 1e3)
    res["cpu_oracle_ms"] = float(np.median(cpu))
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
