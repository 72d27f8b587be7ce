"""Secondary measurements (SURVEY.md §8d configs 3/4): TSDF integrate + ray-cast at the initDr map size with a stream
of synthetic 640x480 depth maps, the level-0 tracker evaluation, the coarse-to-fine track of a frame (host-driven chain of
per-level tdm_tracker_track calls vs one tdm_tracker_track_pyramid), and - when oracle/_ref is present - the REFERENCE's own
dr_fusion (compiled unmodified for sm_90a) on the same inputs on the same GPU.  --retrack times the motion-hypothesis loop of
FullSystem::trackNewCoarse (host loop over tdm_tracker_track_pyramid vs one tdm_tracker_track_new_coarse).
    python tools/bench_fusion_tracker.py [n_frames] [--pyramid-only | --retrack]
Prints one JSON line per measurement."""
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tandem_b200 import CudaCoarseTracker, DrFusion, DrFusionOptions, ImagePyramid, track_pyramid  # noqa: E402
from tandem_b200.synthetic import RoomScene, circle_trajectory, look_at_pose, tracker_case  # noqa: E402

_fp = ctypes.POINTER(ctypes.c_float)
args = [a for a in sys.argv[1:] if not a.startswith("--")]
n_frames = int(args[0]) if args else 40


def gpu_name_and_power_limit():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def coarse_to_fine_leg(n=200, warmup=20, levels=4, H=480, W=640):
    """Per-frame coarse-to-fine track at 640x480 over 4 levels, set up as tandem_b200/loop.py does (device pyramid of the new
    frame, dense reference per level): (a) tdm_tracker_track level by level from the host, (b) one tdm_tracker_track_pyramid.
    The two alternate frame by frame in the same run; the frames cycle through small camera motions around the reference."""
    fx = 320.0
    K = (fx, fx, 319.5, 239.5)
    scene = RoomScene()
    ref_pose = look_at_pose((0.3, 0.0, -0.2), (2.5, 0.2, 0.5))
    bgr_r, depth_r = scene.render(ref_pose, H, W, *K)
    gw = np.array([0.114, 0.587, 0.299], np.float32)
    pyr_ref = ImagePyramid(W, H, levels)
    pyr_ref.build(bgr_r.astype(np.float32) @ gw)
    trk = []
    for l in range(levels):
        t = CudaCoarseTracker(W >> l, H >> l)
        t.init()
        t.setK(W >> l, H >> l, fx / 2 ** l, fx / 2 ** l, (K[2] + 0.5) / 2 ** l - 0.5, (K[3] + 0.5) / 2 ** l - 0.5)
        t.setReferenceDense(np.eye(4), 1.0, np.zeros(2), depth=np.ascontiguousarray(depth_r[::2 ** l, ::2 ** l]), dense_only=True,
                            ref_gray=np.ascontiguousarray(pyr_ref.level(l)[0][..., 0]))
        trk.append(t)
    grays = []
    for k in range(8):
        a = 2 * np.pi * k / 8
        pose = look_at_pose((0.3 + 0.03 * np.cos(a), 0.01 * np.sin(a), -0.2 + 0.02 * np.sin(a)), (2.5, 0.2 + 0.02 * np.cos(a), 0.5))
        grays.append(scene.render(pose, H, W, *K)[0].astype(np.float32) @ gw)
    pyr = ImagePyramid(W, H, levels)
    its = (10, 20, 50, 50)
    modes = dict(affine_opt_mode_a=1e12, affine_opt_mode_b=1e8)

    def chain():
        T, aff, dev = np.eye(4), np.zeros(2), 0.0
        for l in range(levels - 1, -1, -1):
            r = trk[l].track(T, aff, 1.0, max_iterations=its[l])
            T, aff, dev = r["refToNew"], r["aff"], dev + r["device_ms"]
        return dev

    def pyramid():
        return track_pyramid(trk, np.eye(4), np.zeros(2), 1.0, max_iterations=its, **modes)["device_ms"]

    wall = {"chain": [], "pyramid": []}
    dev = {"chain": [], "pyramid": []}
    evals = []
    for f in range(warmup + n):
        pyr.build(grays[f % len(grays)])
        for l in range(levels):
            trk[l].setNewFromPyramid(pyr, l)
        for name, fn in (("chain", chain), ("pyramid", pyramid)) if f % 2 == 0 else (("pyramid", pyramid), ("chain", chain)):
            t0 = time.perf_counter()
            d = fn()
            if f >= warmup:
                wall[name].append((time.perf_counter() - t0) * 1e3)
                dev[name].append(d)
        if f >= warmup:
            evals.append(int(track_pyramid(trk, np.eye(4), np.zeros(2), 1.0, max_iterations=its, **modes)["evaluations"].sum()))
    med = {k: float(np.median(v)) for k, v in wall.items()}
    print(json.dumps({"what": "coarse-to-fine track of one frame, 640x480, 4 levels (median over frames)", "frames": n, "warmup": warmup,
                      "gpu(name, power limit)": gpu_name_and_power_limit(),
                      "chain_wall_ms(track per level from the host)": med["chain"],
                      "pyramid_wall_ms(one track_pyramid)": med["pyramid"],
                      "chain_device_ms(sum of per-level event times)": float(np.median(dev["chain"])),
                      "pyramid_device_ms": float(np.median(dev["pyramid"])),
                      "host_waits_per_frame": {"chain": levels, "pyramid": 1},
                      "evaluations_per_frame(median)": float(np.median(evals)),
                      "wall_speedup": med["chain"] / med["pyramid"]}))


def retrack_leg(n=200, warmup=20, levels=4, H=480, W=640):
    """Per-frame motion-hypothesis loop (FullSystem::trackNewCoarse) at 640x480 over 4 levels with the full 31-try list of
    FullSystem.cpp:437-530 around a last motion far larger than the true one (oracle/pins_retrack.py): (a) the loop on the host
    over track_pyramid (one host wait per try), (b) one track_new_coarse call.  Two lastCoarseRMSE settings: 0 (no try is good
    enough: all 31 run, most abort on the coarsest level) and 2 (the first try that reaches the true pose stops the loop).
    The two ways alternate frame by frame in the same run."""
    from oracle import pins_retrack as R
    from oracle.retrack_driver import track_new_coarse as host_loop
    from tandem_b200 import track_new_coarse
    fx = 320.0
    K = (fx, fx, 319.5, 239.5)
    scene = RoomScene()
    ref_pose = look_at_pose((0.3, 0.0, -0.2), (2.5, 0.2, 0.5))
    bgr_r, depth_r = scene.render(ref_pose, H, W, *K)
    gw = np.array([0.114, 0.587, 0.299], np.float32)
    pyr_ref = ImagePyramid(W, H, levels)
    pyr_ref.build(bgr_r.astype(np.float32) @ gw)
    trk = []
    for l in range(levels):
        t = CudaCoarseTracker(W >> l, H >> l)
        t.init()
        t.setK(W >> l, H >> l, fx / 2 ** l, fx / 2 ** l, (K[2] + 0.5) / 2 ** l - 0.5, (K[3] + 0.5) / 2 ** l - 0.5)
        t.setReferenceDense(np.eye(4), 1.0, np.zeros(2), depth=np.ascontiguousarray(depth_r[::2 ** l, ::2 ** l]), dense_only=True,
                            ref_gray=np.ascontiguousarray(pyr_ref.level(l)[0][..., 0]))
        trk.append(t)
    grays, tries = [], []
    for k in range(8):
        a = 2 * np.pi * k / 8
        pose = look_at_pose((0.3 + 0.03 * np.cos(a), 0.01 * np.sin(a), -0.2 + 0.02 * np.sin(a)), (2.5, 0.2 + 0.02 * np.cos(a), 0.5))
        grays.append(scene.render(pose, H, W, *K)[0].astype(np.float32) @ gw)
        tries.append(R.motion_tries(R.FAR, np.linalg.inv(pose.astype(np.float64)) @ ref_pose.astype(np.float64)))
    pyr = ImagePyramid(W, H, levels)
    its = (10, 20, 50, 50)
    modes = dict(affine_opt_mode_a=1e12, affine_opt_mode_b=1e8)
    aff0 = np.zeros(2)
    for rmse0 in (0.0, 2.0):
        rmse = np.full(5, rmse0)
        waits = [0]

        def host(tr):
            dev = [0.0]

            def tp(T, aff, min_res):
                r = track_pyramid(trk, T, aff, 1.0, max_iterations=its, min_res_for_abort=min_res, **modes)
                dev[0] += r["device_ms"]
                waits[0] += 1
                return r
            r = host_loop(tp, tr, aff0, rmse)
            return r, dev[0]

        def device(tr):
            r = track_new_coarse(trk, tr, aff0, 1.0, rmse, max_iterations=its, **modes)
            return r, r["device_ms"]

        wall = {"host": [], "device": []}
        dev = {"host": [], "device": []}
        n_tries, n_evals, n_waits = [], [], []
        for f in range(warmup + n):
            pyr.build(grays[f % len(grays)])
            for l in range(levels):
                trk[l].setNewFromPyramid(pyr, l)
            tr = tries[f % len(tries)]
            for name, fn in (("host", host), ("device", device)) if f % 2 == 0 else (("device", device), ("host", host)):
                waits[0] = 0
                t0 = time.perf_counter()
                r, d = fn(tr)
                if f >= warmup:
                    wall[name].append((time.perf_counter() - t0) * 1e3)
                    dev[name].append(d)
                    if name == "host":
                        n_waits.append(waits[0])
                    else:
                        n_tries.append(r["tries"])
                        n_evals.append(sum(int(t["evaluations"].sum()) for t in r["per_try"]))
        med = {k: float(np.median(v)) for k, v in wall.items()}
        print(json.dumps({"what": "motion-hypothesis loop of one frame, 640x480, 4 levels, 31 tries (median over frames)",
                          "last_coarse_rmse": rmse0, "frames": n, "warmup": warmup, "gpu(name, power limit)": gpu_name_and_power_limit(),
                          "host_loop_wall_ms(track_pyramid per try)": med["host"], "track_new_coarse_wall_ms": med["device"],
                          "host_loop_device_ms(sum of per-try event times)": float(np.median(dev["host"])),
                          "track_new_coarse_device_ms": float(np.median(dev["device"])),
                          "host_waits_per_frame": {"host_loop": float(np.median(n_waits)), "track_new_coarse": 1},
                          "tries_per_frame(median)": float(np.median(n_tries)), "evaluations_per_frame(median)": float(np.median(n_evals)),
                          "wall_speedup": med["host"] / med["device"]}))


if "--pyramid-only" in sys.argv:
    coarse_to_fine_leg()
    sys.exit(0)
if "--retrack" in sys.argv:
    retrack_leg()
    sys.exit(0)
H, W = 480, 640
intr = dict(fx=320.0, fy=320.0, cx=319.5, cy=239.5)
scene = RoomScene()
poses = circle_trajectory(n_frames, radius=1.0)
frames = [scene.render(p, H, W, **intr, noise_sigma=0.002, dropout=0.02, seed=k) for k, p in enumerate(poses)]
for p in poses:
    p[:3, 3] += np.float32(5.12)     # keep block (0,0,0) out of the map (reference quirk, SURVEY Appendix B.2)

opt = DrFusionOptions(height=H, width=W, **intr)
f = DrFusion(opt)
t0 = time.perf_counter()
for (bgr, depth), pose in zip(frames, poses):
    f.IntegrateScanAsync(bgr, depth, pose)
    f.RenderAsync([pose])
    f.GetRenderResult()
f.Synchronize()
e2e_ms = (time.perf_counter() - t0) * 1e3 / n_frames
st = f.stats()
vis = st["visible_blocks"]
alg = vis * 512 * 16 + 7 * H * W
res = {}
DEFAULTS = {"raycast_shared": 1, "fast_div": 0}
for name, opts in (("default", {}), ("raycast_lookup_per_voxel", {"raycast_shared": 0}), ("fast_div", {"fast_div": 1})):
    for k, dv in DEFAULTS.items():
        f.set_option(k, opts.get(k, dv))
    f.run_resident(3)
    mi, mr = f.run_resident(20)
    res[name] = {"allocate_ms": f.last_alloc_ms(), "allocate+integrate_ms": mi / 20, "raycast_ms": mr / 20}
for k, dv in DEFAULTS.items():
    f.set_option(k, dv)
mi = res["default"]["allocate+integrate_ms"] * 20
mr = res["default"]["raycast_ms"] * 20
print(json.dumps({"what": "tsdf ours", "frames": n_frames, "allocated_blocks": st["allocated_blocks"], "visible_blocks_last": vis,
                  "e2e_ms_per_frame(integrate+render+copies)": e2e_ms, "resident_allocate+integrate_ms": mi / 20,
                  "resident_allocate_ms": res["default"]["allocate_ms"],
                  "resident_raycast_ms": mr / 20, "integrate_algorithmic_GB": alg / 1e9,
                  "integrate_GBps": alg / (mi / 20 * 1e-3) / 1e9, "ab": res}))
# marching cubes over the 10 m box of tandem_backend.cpp:80-81 (shifted with the scene)
lo = np.float32([0.12, 0.12, 0.12]); up = np.float32([10.12, 10.12, 10.12])
f.ExtractMeshAsync(lo, up)
t0 = time.perf_counter()
mv, mc = f.GetMeshSync()
wall = (time.perf_counter() - t0) * 1e3
f.ExtractMeshAsync(lo, up); f.GetMeshSync()
print(json.dumps({"what": "mesh ours (block-sparse marching cubes, 1000^3-cell box)", "triangles": len(mv) // 3,
                  "blocks": st["allocated_blocks"], "device_ms(classify+scan+emit)": f.last_mesh_ms(), "GetMeshSync_wall_ms(first call, incl. D2H)": wall}))

ref_lib = os.path.join(ROOT, "oracle", "_ref", "libdr_fusion_ref.so")
if os.path.exists(ref_lib):
    l = ctypes.CDLL(ref_lib)
    l.ref_fusion_create.restype = ctypes.c_void_p
    r = ctypes.c_void_p(l.ref_fusion_create(ctypes.byref(opt)))
    rb, rd = np.zeros((H, W, 3), np.uint8), np.zeros((H, W), np.float32)
    ti = tr = 0.0
    nref = min(n_frames, 10)
    for (bgr, depth), pose in list(zip(frames, poses))[:nref]:
        b, d = np.ascontiguousarray(bgr), np.ascontiguousarray(depth)
        t0 = time.perf_counter()
        l.ref_fusion_integrate(r, ctypes.c_void_p(b.ctypes.data), d.ctypes.data_as(_fp), pose.ctypes.data_as(_fp))
        l.ref_fusion_sync(r)
        t1 = time.perf_counter()
        l.ref_fusion_render(r, pose.ctypes.data_as(_fp), ctypes.c_void_p(rb.ctypes.data), rd.ctypes.data_as(_fp), H * W)
        t2 = time.perf_counter()
        ti += t1 - t0
        tr += t2 - t1
    l.ref_fusion_get_mesh.restype = ctypes.c_longlong
    t0 = time.perf_counter()
    nm = l.ref_fusion_get_mesh(r, lo.ctypes.data_as(_fp), up.ctypes.data_as(_fp), None, None, ctypes.c_longlong(0))
    tm = (time.perf_counter() - t0) * 1e3
    print(json.dumps({"what": "tsdf reference dr_fusion (unmodified, sm_90a)", "frames": nref,
                      "integrate_ms_per_frame(wall)": ti * 1e3 / nref, "render_ms_per_frame(wall)": tr * 1e3 / nref,
                      "GetMesh_wall_ms(10 m box)": tm, "mesh_triangles": nm // 3}))
    l.ref_fusion_destroy(r)

c = tracker_case()
t = CudaCoarseTracker(c["w"], c["h"])
t.init()
t.setK(c["w"], c["h"], c["fx"], c["fy"], c["cx"], c["cy"])
t.setReference(c["n"], c["pc_u"], c["pc_v"], c["pc_idepth"], c["pc_color"], c["ref_exposure"], c["ref_aff"])
t.setNew(c["dInew"])
t.calcRes(c["refToNew"], c["new_exposure"], c["new_aff"], c["cutoffTH"])   # run_resident re-runs the fused kernel on these
ms = t.run_resident(200)
t0 = time.perf_counter()
for _ in range(200):
    t.calcResAndG(c["refToNew"], c["new_exposure"], c["new_aff"], c["cutoffTH"])
wall_fused = (time.perf_counter() - t0) / 200 * 1e6
t0 = time.perf_counter()
for _ in range(200):
    t.calcRes(c["refToNew"], c["new_exposure"], c["new_aff"], c["cutoffTH"])
    t.calcG(c["new_exposure"], c["new_aff"])
wall_two = (time.perf_counter() - t0) / 200 * 1e6
print(json.dumps({"what": "tracker ours", "n_points": c["n"], "kernel_us(fused, device)": ms / 200 * 1e3,
                  "wall_us(fused call incl sync)": wall_fused, "wall_us(calcRes+calcG calls)": wall_two,
                  "algorithmic_MB": (16 * c["n"] + 12 * c["w"] * c["h"] + 416) / 1e6}))

# ---- comparators the north-star names (VERDICT r01 item 3): the tandem CPU tracker on this box's host cores (single thread, as
# the reference: CoarseTracker::calcRes + calcGSSSE, restated in oracle/tracker_oracle.c and pinned to the reference kernels) and
# the reference's own CUDA kernels (calcResKernelNew + calcGKernel<float>, compiled unmodified) on this GPU, same inputs.
from oracle.cpu import TrackerOracle  # noqa: E402  (comparator only; never on the product path)
orc = TrackerOracle(c["w"], c["h"])
orc.setK(c["w"], c["h"], c["fx"], c["fy"], c["cx"], c["cy"])
orc.setReference(c["n"], c["pc_u"], c["pc_v"], c["pc_idepth"], c["pc_color"], c["ref_exposure"], c["ref_aff"])
orc.setNew(c["dInew"])
orc.calcRes(c["refToNew"], c["new_exposure"], c["new_aff"], c["cutoffTH"]); orc.calcG(c["new_exposure"], c["new_aff"])
reps = 10
t0 = time.perf_counter()
for _ in range(reps):
    orc.calcRes(c["refToNew"], c["new_exposure"], c["new_aff"], c["cutoffTH"])
t1 = time.perf_counter()
for _ in range(reps):
    orc.calcG(c["new_exposure"], c["new_aff"])
t2 = time.perf_counter()
cpu_res_us, cpu_g_us = (t1 - t0) / reps * 1e6, (t2 - t1) / reps * 1e6
print(json.dumps({"what": "tracker CPU baseline (oracle/tracker_oracle.c = CoarseTracker::calcRes + calcGSSSE, gcc -O2, 1 thread)",
                  "n_points": c["n"], "calcRes_us": cpu_res_us, "calcG_us": cpu_g_us, "pair_us": cpu_res_us + cpu_g_us,
                  "host_threads_used": 1, "host_threads_available": os.cpu_count(),
                  "ours_kernel_speedup": (cpu_res_us + cpu_g_us) / (ms / 200 * 1e3)}))
trk_lib = os.path.join(ROOT, "oracle", "_ref", "libtracker_ref.so")
if os.path.exists(trk_lib):
    l = ctypes.CDLL(trk_lib)
    if hasattr(l, "ref_tracker_eval_timed"):
        aff = orc._aff(c["new_exposure"], c["new_aff"])
        T = np.ascontiguousarray(c["refToNew"], np.float32)
        Ki = np.array([1.0 / c["fx"], 0, -c["cx"] / c["fx"], 0, 1.0 / c["fy"], -c["cy"] / c["fy"], 0, 0, 1], np.float32)
        o7, o45 = np.zeros(7, np.float32), np.zeros(45, np.float32)
        mr, mg = ctypes.c_float(0), ctypes.c_float(0)
        fl = ctypes.c_float
        rc = l.ref_tracker_eval_timed(c["w"], c["h"], fl(c["fx"]), fl(c["fy"]), fl(c["cx"]), fl(c["cy"]), T.ctypes.data_as(_fp),
                                      Ki.ctypes.data_as(_fp), fl(aff[0]), fl(aff[1]), fl(c["ref_aff"][1]), fl(9.0), fl(c["cutoffTH"]),
                                      c["n"], c["pc_u"].ctypes.data_as(_fp), c["pc_v"].ctypes.data_as(_fp),
                                      c["pc_idepth"].ctypes.data_as(_fp), c["pc_color"].ctypes.data_as(_fp),
                                      np.ascontiguousarray(c["dInew"]).ctypes.data_as(_fp), o7.ctypes.data_as(_fp),
                                      o45.ctypes.data_as(_fp), None, 200, ctypes.byref(mr), ctypes.byref(mg))
        print(json.dumps({"what": "tracker reference kernels (calcResKernelNew + calcGKernel<float>, unmodified, sm_90a) on this GPU",
                          "rc": rc, "n_points": c["n"], "calcRes_kernel_us(device)": mr.value * 1e3, "calcG_kernel_us(device)": mg.value * 1e3,
                          "pair_us(device)": (mr.value + mg.value) * 1e3, "ours_fused_kernel_us(device)": ms / 200 * 1e3,
                          "ours_speedup": (mr.value + mg.value) * 1e3 / (ms / 200 * 1e3),
                          "note": "device time of the kernels + the per-call output memsets only; the reference's host wrapper adds a blocking sync and D2H per call (cuda_coarse_tracker.cpp:195-356)"}))

coarse_to_fine_leg()
