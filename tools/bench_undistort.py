"""n11: one camera frame from the raw 8-bit image to its pyramid, at 640x480 (TUM-mono-like: 640x480 raw, photometric
calibration mode 2) and 752x480 -> 640x480 (EuRoC-like: mode 1), 5 pyramid levels with gamma weights:

  undistort_gray   Undistorter.frame, grey only: the u8 upload, k_undistort and the pyramid's kernels
  undistort_bgr    Undistorter.frame with the BGR remap returned to the host (one host wait)
  pyramid_build    ImagePyramid.build of the host float image - the path this replaces, which still needs the host undistort
  cpu_oracle       the C oracles on one CPU thread: processFrame + remap, the BGR remap and the gamma-weighted makeImages
                   (oracle/undistort_oracle.c, -O2, no FMA contraction), the host work the device path replaces

Per GPU path: the median wall time of one call followed by a device synchronise, over --frames frames after --warmup, and
the median per-call device time (torch.profiler in a run of its own: the summed CUDA kernel time and the summed
host-to-device copy time of a call).  The card's name and power limit are read in the same run.

    python tools/bench_undistort.py [--frames 300] [--warmup 30] [--out out/bench_undistort.json]
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

from oracle import undistort as U  # noqa: E402
from tandem_b200 import ImagePyramid, Undistorter  # noqa: E402

LEVELS = 5
CAMERAS = {"tum_640x480": (640, 480, 640, 480, "v16", 2), "euroc_752x480_to_640x480": (752, 480, 640, 480, "v8", 1)}


def camera_inputs(w_org, h_org, w, h, vig):
    rx, ry = U.remap_tables(w_org, h_org, w, h)
    resp = U.response("gamma")
    frames = [U.render(w_org, h_org, k) for k in range(4)]
    return rx, ry, resp, U.vignette(vig, w_org, h_org), frames


def cpu_oracle_ms(w_org, h_org, w, h, rx, ry, resp, vignette, mode, gray, bgr, B, reps):
    l = U._lib()
    G = np.zeros(256, np.float32)
    vinv = np.zeros(w_org * h_org, np.float32)
    valid = l.undistort_oracle_create(U._p(resp), resp.size, U._p(vignette, U._sp), w_org * h_org, mode, U._p(G), U._p(vinv))
    scratch = np.zeros(w_org * h_org, np.float32)
    img = np.zeros(w * h, np.float32)
    bo = np.zeros(3 * w * h, np.uint8)
    tot = sum((w >> k) * (h >> k) for k in range(LEVELS))
    dI, ag = np.zeros(3 * tot, np.float32), np.zeros(tot, np.float32)
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        l.undistort_oracle_frame(U._p(gray, U._up), w_org, h_org, w, h, U._p(rx), U._p(ry), valid, mode, 1, U._p(G), U._p(vinv),
                                 ctypes.c_float(10.0), ctypes.c_float(1.0), U._p(scratch), U._p(img))
        l.undistort_oracle_bgr(U._p(bgr, U._up), w_org, h_org, w, h, U._p(rx), U._p(ry), U._p(bo, U._up))
        l.undistort_oracle_make_images(U._p(img), w, h, LEVELS, U._p(B), U._p(dI), U._p(ag))
        ts.append(time.perf_counter() - t0)
    return 1e3 * float(np.median(ts)), img.reshape(h, w)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--warmup", type=int, default=30)
    ap.add_argument("--cpu-reps", type=int, default=30)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    card = smi.stdout.strip().splitlines()[0] if smi.returncode == 0 else "unknown"
    res = dict(card=card, levels=LEVELS, frames=a.frames, cameras={})
    for cam, (w_org, h_org, w, h, vig, mode) in CAMERAS.items():
        rx, ry, resp, vignette, frames = camera_inputs(w_org, h_org, w, h, vig)
        u = Undistorter(w_org, h_org, w, h, rx, ry, resp, vignette, mode)
        G = u.get_gamma()
        u.set_gamma(G)
        B = U.set_gamma(G, np.arange(256, dtype=np.float32))
        p = ImagePyramid(w, h, LEVELS)
        bgr_out = np.empty((h, w, 3), np.uint8)
        host_float = [U.render(w, h, k)[0].astype(np.float32) for k in range(len(frames))]

        def run(path, i):
            g, b = frames[i % len(frames)]
            if path == "undistort_gray":
                u.frame(g, 10.0, p)
            elif path == "undistort_bgr":
                u.frame(g, 10.0, p, bgr=b, bgr_out=bgr_out)
            else:
                p.build(host_float[i % len(frames)])

        out = {}
        for path in ("undistort_gray", "undistort_bgr", "pyramid_build"):
            for i in range(a.warmup):
                run(path, i)
            torch.cuda.synchronize()
            ts = []
            for i in range(a.frames):
                t0 = time.perf_counter()
                run(path, i)
                torch.cuda.synchronize()
                ts.append(time.perf_counter() - t0)
            n_prof = 50
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for i in range(n_prof):
                    run(path, i)
                torch.cuda.synchronize()
            kern = copy = 0.0
            for e in prof.events():
                if e.device_type.name != "CUDA":
                    continue
                nm = e.name
                dur = e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
                if "Memcpy HtoD" in nm:
                    copy += dur
                elif "Memcpy" not in nm and "Memset" not in nm:
                    kern += dur
            out[path] = dict(wall_ms_median=1e3 * float(np.median(ts)), wall_ms_p10=1e3 * float(np.percentile(ts, 10)),
                             wall_ms_p90=1e3 * float(np.percentile(ts, 90)), kernel_ms_per_call=kern / n_prof / 1e3,
                             h2d_ms_per_call=copy / n_prof / 1e3)
        cpu_ms, img = cpu_oracle_ms(w_org, h_org, w, h, rx, ry, resp, vignette, mode, frames[0][0], frames[0][1], B, a.cpu_reps)
        out["cpu_oracle"] = dict(ms_median=cpu_ms)
        # the timed device path computes what the oracle computes
        u.frame(frames[0][0], 10.0, p)
        out["device_equals_oracle"] = bool(np.array_equal(p.level(0)[0][..., 0], img))
        res["cameras"][cam] = out
        print(cam, json.dumps(out), flush=True)
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
