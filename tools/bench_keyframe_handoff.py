"""Per-keyframe cost of the MVSNet -> TSDF handoff: TANDEM's backend step (TandemBackendImpl::CallSequential,
tandem_backend.cpp:137-200) GetResult(k) -> CallAsync(k+1) -> integrate(k) -> RenderAsync -> GetRenderResult, with the
integration either through the host (IntegrateScanAsync of GetResult's depth, the reference BGR image and pose: D2H, staging
memcpy, H2D) or read on the device (IntegrateScanFromMvsnet).  The two paths alternate in blocks of keyframes in one process,
each on its own fusion handle, behind one engine; host memory is pageable as in TANDEM (cv::Mat data, malloc'd result).

    python tools/bench_keyframe_handoff.py [--keyframes 200] [--warmup 20] [--block 10] [--pinned]

Reports medians per keyframe: wall time of the whole step and of each call, and the device time of integrate + render on the
fusion stream (CUDA events), with the card name and power limit read in the same run.  Prints one JSON line."""
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
from tandem_b200.fusion import DrFusion, DrFusionOptions  # noqa: E402
from tandem_b200.synthetic import mvs_plane_window  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        q = f"nvidia-smi unavailable: {e}"
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--keyframes", type=int, default=200, help="timed keyframes per path")
    ap.add_argument("--warmup", type=int, default=20, help="untimed keyframes per path first")
    ap.add_argument("--block", type=int, default=10, help="keyframes per path before switching to the other")
    ap.add_argument("--pinned", action="store_true", help="page-locked result maps and images instead of pageable memory")
    ap.add_argument("--precision", default="mixed16", choices=["mixed16", "fp32"])
    a = ap.parse_args()

    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_keyframe_handoff: no CUDA device (this measurement only runs on the GPU)")
    H, W, V = 480, 640, 7
    nf = 24
    win = mvs_plane_window(V=nf, H=H, W=W, f=525.0, z_plane=2.0, baseline=0.02, seed=3)
    bgrs, c2ws, K = win["bgrs"], win["c2ws"], win["K"]
    if a.pinned:
        from tandem_b200._lib import pinned_empty
        pb = []
        for b in bgrs:
            p = pinned_empty(b.shape, np.uint8)
            p[...] = b
            pb.append(p)
        bgrs = pb
    nw = nf - V + 1
    ref = V - 2
    m = DrMvsnet(default_weights("abl03_view_aggregation"), precision=a.precision)
    out = DrMvsnetOutput(H, W, pinned=a.pinned)
    if a.pinned:
        m.set_option("eager_d2h", 0)
    fo = DrFusionOptions(height=H, width=W, fx=float(K[0, 0]), fy=float(K[1, 1]), cx=float(K[0, 2]), cy=float(K[1, 2]))
    fus = {"host": DrFusion(fo), "device": DrFusion(fo)}
    streams = {k: torch.cuda.ExternalStream(f.stream()) for k, f in fus.items()}
    rec = {k: dict(step=[], get=[], call=[], integrate=[], render=[], get_render=[], device=[]) for k in fus}

    def call(w):
        m.CallAsync(H, W, V, ref, bgrs[w:w + V], K, c2ws[w:w + V], 0.5, 5.0, 2.5)

    done = {k: 0 for k in fus}
    total = a.warmup + a.keyframes
    path, in_block, w = "host", 0, 0
    call(w)
    while min(done.values()) < total:
        if done[path] >= total or in_block == a.block:
            other = "device" if path == "host" else "host"
            if done[other] < total:
                path = other
            in_block = 0
        f, st = fus[path], streams[path]
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        r = m.GetResult(out=out)                                        # (1) GetResult(k)
        t1 = time.perf_counter()
        call((w + 1) % nw)                                              # (3.5) CallAsync(k+1)
        t2 = time.perf_counter()
        e0.record(st)
        if path == "host":                                              # (3) integrate(k)
            f.IntegrateScanAsync(bgrs[w + ref], r.depth, c2ws[w + ref])
        else:
            f.IntegrateScanFromMvsnet(m)
        t3 = time.perf_counter()
        f.RenderAsync([c2ws[w + ref]])                                  # (4)
        e1.record(st)
        t4 = time.perf_counter()
        f.GetRenderResult()                                             # (5)
        t5 = time.perf_counter()
        e1.synchronize()
        if done[path] >= a.warmup:
            R = rec[path]
            R["step"].append((t5 - t0) * 1e3)
            R["get"].append((t1 - t0) * 1e3)
            R["call"].append((t2 - t1) * 1e3)
            R["integrate"].append((t3 - t2) * 1e3)
            R["render"].append((t4 - t3) * 1e3)
            R["get_render"].append((t5 - t4) * 1e3)
            R["device"].append(e0.elapsed_time(e1))
        done[path] += 1
        in_block += 1
        w = (w + 1) % nw
    m.GetResult(out=out)
    for f in fus.values():
        f.Synchronize()
    med = {k: {n: float(np.median(v)) for n, v in R.items()} for k, R in rec.items()}
    print(json.dumps({
        "metric": "per-keyframe backend step GetResult -> CallAsync -> integrate -> RenderAsync -> GetRenderResult, medians (ms)",
        "shape": f"{W}x{H}, {V} views, {a.precision}", "host_memory": "page-locked" if a.pinned else "pageable",
        "keyframes_per_path": a.keyframes, "warmup_per_path": a.warmup, "block": a.block,
        "card": card(), "host_path": med["host"], "device_path": med["device"],
        "saved_ms": {n: med["host"][n] - med["device"][n] for n in med["host"]},
        "device_ms_note": "CUDA events on the fusion stream around integrate + RenderAsync",
    }))


if __name__ == "__main__":
    main()
