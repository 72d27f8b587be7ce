"""GPU parity of SURVEY 8(f) n7: tdm_tracker_set_coarse_tracking_ref (CoarseTracker::setCoarseTrackingRef with
makeCoarseDepthL0, every level in one call) against the CPU restatement oracle/coarse_ref_oracle.c chained with n1's dense block,
which tests/test_coarse_ref_cpu.py pins to the reference's own function bodies.  Every level's pc_n and its four arrays,
slot pc_n included, are compared bit for bit."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from oracle import pins_coarse_ref as P
from oracle.coarse_ref import CoarseRefOracle
from tandem_b200 import (CudaCoarseTracker, DrFusion, DrFusionOptions, ImagePyramid, set_coarse_tracking_ref, track_new_coarse,
                         track_pyramid)
from tandem_b200._lib import TandemError, lib
from tandem_b200.synthetic import RoomScene, look_at_pose

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "reference_pins_coarse_ref.npz")
AFF = np.array([0.02, 1.5])


def level_K(l, K):
    fx, fy, cx, cy = K
    return (fx / 2 ** l, fy / 2 ** l, (cx + 0.5) / 2 ** l - 0.5, (cy + 0.5) / 2 ** l - 0.5)   # CoarseTracker::makeK


def trackers(w, h, levels, K, n_max=0):
    ts = []
    for l in range(levels):
        t = CudaCoarseTracker(w >> l, h >> l)
        t.init(n_max)
        t.setK(w >> l, h >> l, *level_K(l, K))
        ts.append(t)
    return ts


def same(a, b):
    return np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True)


def assert_levels_match(ts, pc_n, oracle):
    exp_n = oracle[0]
    assert pc_n == exp_n
    for l, t in enumerate(ts):
        got = t.getReference(pc_n[l] + 1)
        for k, (a, b) in enumerate(zip(got, oracle[1][l])):
            assert same(a, b), (l, k, np.flatnonzero(~((a == b) | (np.isnan(a) & np.isnan(b))))[:10])


@pytest.mark.parametrize("name", list(P.CASES))
def test_coarse_ref_matches_pinned_oracle(name):
    T = np.load(GOLDEN)[f"{name}_T"]
    (h, w), levels, gray_levels, depth, kfs = P.case_inputs(name)
    expect = P.run_oracle(name, T)
    pyr = ImagePyramid(w, h, levels)
    pyr.build(P.gray_image(h, w, 0))
    for l in range(levels):   # the colours the device reads equal the oracle's (n2 is bit exact)
        assert same(pyr.level(l)[0][..., 0], gray_levels[l])
    ts = trackers(w, h, levels, P.K4(h, w))
    for kf, exp in zip(kfs, expect):
        pc_n = set_coarse_tracking_ref(ts, kf["points"], pyr, depth=depth if kf["dense"] else None, T_depth_to_ref=T,
                                       tracking_step=kf["step"], dense_only=kf["dense_only"], rgbd_init=kf["rgbd"],
                                       ref_exposure=1.25, ref_aff_g2l=AFF)
        assert_levels_match(ts, pc_n, exp)


# ---- a synthetic keyframe at 640x480: ~2000 projected sparse points, dense depth from the host and from a DrFusion render
H, W, L = 480, 640, 4
K0 = (320.0, 320.0, 319.5, 239.5)
POSE_REF = look_at_pose((0.3, 0.0, -0.2), (2.5, 0.2, 0.5))
POSE_DEPTH = look_at_pose((0.32, 0.01, -0.19), (2.5, 0.22, 0.48))
POSE_NEW = look_at_pose((0.33, 0.01, -0.18), (2.5, 0.22, 0.52))


def room_keyframe(seed=0, n=2000):
    s = RoomScene()
    bgr, depth = s.render(POSE_REF, H, W, *K0)
    gray = bgr.astype(np.float32) @ P.GRAY_W
    rng = np.random.default_rng(seed)
    ys, xs = np.nonzero(depth > 0)
    pick = rng.choice(len(ys), n, replace=False)
    x, y, z = xs[pick], ys[pick], depth[ys[pick], xs[pick]]
    pts = ((x + rng.uniform(-0.4, 0.4, n)).astype(np.float32), (y + rng.uniform(-0.4, 0.4, n)).astype(np.float32),
           (1.0 / z * (1 + 0.01 * rng.standard_normal(n))).astype(np.float32), rng.uniform(1e-3, 2.0, n).astype(np.float32))
    T = np.linalg.inv(POSE_REF.astype(np.float64)) @ POSE_DEPTH.astype(np.float64)
    return gray, pts, T


def fusion_render():
    s = RoomScene()
    fus = DrFusion(DrFusionOptions(height=H, width=W, fx=K0[0], fy=K0[1], cx=K0[2], cy=K0[3], num_render_streams=1))
    for k in range(3):
        pose = look_at_pose((0.3 + 0.02 * k, 0.0, -0.2), (2.5, 0.2, 0.5))
        bgr, d = s.render(pose, H, W, *K0)
        fus.IntegrateScanAsync(bgr, d, pose)
        fus.RenderAsync([POSE_DEPTH])
        _, depth = fus.GetRenderResult()
    return fus, np.array(depth[0], np.float32).reshape(H, W)


def oracle_run(gray_levels, pts, depth, T, **kw):
    o = CoarseRefOracle(W, H, L)
    pc_n = o.set_coarse_tracking_ref(pts, gray_levels, depth=depth, T_depth_to_ref=T, K4=K0, **kw)
    return pc_n, o.result(pc_n)


@pytest.fixture(scope="module")
def room():
    gray, pts, T = room_keyframe()
    pyr = ImagePyramid(W, H, L)
    pyr.build(gray)
    gray_levels = [np.ascontiguousarray(pyr.level(l)[0][..., 0]) for l in range(L)]
    fus, depth = fusion_render()
    assert (depth > 0).mean() > 0.5
    return dict(gray=gray, pts=pts, T=T, pyr=pyr, gray_levels=gray_levels, fus=fus, depth=depth)


@pytest.mark.parametrize("source", ["host", "fusion", "none"])
def test_room_keyframe_matches_oracle(room, source):
    ts = trackers(W, H, L, K0)
    depth = None if source == "none" else room["depth"]
    kw = dict(depth=room["depth"]) if source == "host" else dict(fusion=room["fus"]) if source == "fusion" else {}
    pc_n = set_coarse_tracking_ref(ts, room["pts"], room["pyr"], T_depth_to_ref=room["T"], ref_aff_g2l=AFF, **kw)
    exp = oracle_run(room["gray_levels"], room["pts"], depth, room["T"])
    assert exp[0][0] > 2000 and all(n > 0 for n in exp[0])
    assert_levels_match(ts, pc_n, exp)


def test_two_keyframes_in_a_row_keep_the_stale_slot(room):
    # keyframe 1 has fewer points, so slot pc_n of keyframe 1 holds what keyframe 0 (or its rejected candidate) left there
    ts = trackers(W, H, L, K0)
    o = CoarseRefOracle(W, H, L)
    for seed, n in ((0, 2000), (1, 300)):
        _, pts, _ = room_keyframe(seed, n)
        pts[2][::50] = -pts[2][::50]                      # rejected candidates
        pc_n = set_coarse_tracking_ref(ts, pts, room["pyr"], depth=room["depth"], T_depth_to_ref=room["T"], ref_aff_g2l=AFF)
        exp_n = o.set_coarse_tracking_ref(pts, room["gray_levels"], depth=room["depth"], T_depth_to_ref=room["T"], K4=K0)
        assert_levels_match(ts, pc_n, (exp_n, o.result(exp_n)))


def _raw_call(ts, n_levels, n, pts, pyr):
    fp = ctypes.POINTER(ctypes.c_float)
    hs = (ctypes.c_void_p * max(len(ts), 1))(*[t._h for t in ts])
    arrs = [None if a is None else np.ascontiguousarray(a, np.float32) for a in pts]
    aff = np.zeros(2)
    pc_n = np.zeros(5, np.int32)
    return lib().tdm_tracker_set_coarse_tracking_ref(
        hs, n_levels, 0, n, *[None if a is None else a.ctypes.data_as(fp) for a in arrs], None if pyr is None else pyr._h,
        None, None, 0, None, 1, 0, 1.0, aff.ctypes.data_as(ctypes.POINTER(ctypes.c_double)),
        pc_n.ctypes.data_as(ctypes.POINTER(ctypes.c_int)))


def test_errors_launch_nothing_and_a_valid_call_follows(room):
    ts = trackers(W, H, L, K0)
    pts, pyr = room["pts"], room["pyr"]
    exp = oracle_run(room["gray_levels"], pts, room["depth"], room["T"])

    def valid():
        pc_n = set_coarse_tracking_ref(ts, pts, pyr, depth=room["depth"], T_depth_to_ref=room["T"], ref_aff_g2l=AFF)
        assert_levels_match(ts, pc_n, exp)

    valid()
    bad_size = CudaCoarseTracker(W >> 1, (H >> 1) + 2)
    bad_size.init()
    no_k = CudaCoarseTracker(W, H)
    no_k.init()
    pyr_short, pyr_other = ImagePyramid(W, H, 2), ImagePyramid(W - 2, H, L)
    pyr_short.build(room["gray"])
    pyr_other.build(np.zeros((H, W - 2), np.float32))
    u_out = pts[0].copy()
    u_out[1234] = W - 0.5                                 # + 0.5f -> W: outside
    rgbd_out = [a.copy() for a in pts]
    rgbd_out[0][7] = -1.5
    cases = [
        lambda: set_coarse_tracking_ref([], pts, pyr),                                               # n_levels 0
        lambda: set_coarse_tracking_ref(ts + ts[:2], pts, pyr),                                      # n_levels 6
        lambda: set_coarse_tracking_ref([ts[0], bad_size, ts[2]], pts, pyr),                         # level size
        lambda: set_coarse_tracking_ref([no_k] + ts[1:], pts, pyr),                                  # no setK on level 0
        lambda: set_coarse_tracking_ref(ts, pts, pyr_short),                                         # too few pyramid levels
        lambda: set_coarse_tracking_ref(ts, pts, pyr_other),                                         # other level-0 size
        lambda: set_coarse_tracking_ref(ts, (u_out,) + tuple(pts[1:]), pyr),                         # point outside (float)
        lambda: set_coarse_tracking_ref(ts, rgbd_out, pyr, rgbd_init=True),                          # point outside (double)
        lambda: set_coarse_tracking_ref(ts, pts, pyr, depth=room["depth"], fusion=room["fus"], T_depth_to_ref=room["T"]),
        lambda: set_coarse_tracking_ref(ts, pts, pyr, depth=room["depth"]),                          # no T_depth_to_ref
        lambda: set_coarse_tracking_ref(ts, pts, pyr, depth=room["depth"], T_depth_to_ref=room["T"], tracking_step=0),
    ]
    for k, c in enumerate(cases):
        with pytest.raises(TandemError):
            c()
        valid()
    assert _raw_call(ts, L, 10, (None, None, None, None), pyr) < 0          # null point arrays
    assert _raw_call(ts, L, 0, (None,) * 4, None) < 0                       # null pyramid
    valid()


def test_capacity_error_leaves_every_level_empty(room):
    ts = trackers(W, H, L, K0)
    ts[2] = CudaCoarseTracker(W >> 2, H >> 2)
    ts[2].init(100)                                       # far too small for level 2
    ts[2].setK(W >> 2, H >> 2, *level_K(2, K0))
    with pytest.raises(TandemError):
        set_coarse_tracking_ref(ts, room["pts"], room["pyr"], ref_aff_g2l=AFF)
    new = ImagePyramid(W, H, L)
    new.build(room["gray"])
    for l, t in enumerate(ts):
        t.setNewFromPyramid(new, l)
    with pytest.raises(TandemError):                      # no reference to track against
        track_pyramid(ts, np.eye(4), np.zeros(2), 1.0)
    ok = trackers(W, H, L, K0)
    pc_n = set_coarse_tracking_ref(ok, room["pts"], room["pyr"], ref_aff_g2l=AFF)
    assert_levels_match(ok, pc_n, oracle_run(room["gray_levels"], room["pts"], None, None))


def test_tracking_after_the_call_equals_tracking_after_set_reference(room):
    ts = trackers(W, H, L, K0)
    pc_n = set_coarse_tracking_ref(ts, room["pts"], room["pyr"], depth=room["depth"], T_depth_to_ref=room["T"],
                                   ref_exposure=1.0, ref_aff_g2l=AFF)
    exp = oracle_run(room["gray_levels"], room["pts"], room["depth"], room["T"])
    ref = trackers(W, H, L, K0)
    for l, t in enumerate(ref):
        t.setReference(exp[0][l], *[a[:exp[0][l]] for a in exp[1][l]], 1.0, AFF)
    bgr, _ = RoomScene().render(POSE_NEW, H, W, *K0)
    new = ImagePyramid(W, H, L)
    new.build(bgr.astype(np.float32) @ P.GRAY_W)
    for group in (ts, ref):
        for l, t in enumerate(group):
            t.setNewFromPyramid(new, l)
    drop = ("device_ms",)
    a, b = (track_pyramid(g, np.eye(4), AFF, 1.05, affine_opt_mode_a=1e12, affine_opt_mode_b=1e8) for g in (ts, ref))
    assert a["ok"] and all(same(a[k], b[k]) for k in a if k not in drop)
    T_try = np.stack([np.eye(4)] * 3)
    T_try[1][:3, 3] = (0.01, 0, 0)
    T_try[2][:3, 3] = (0, 0.01, 0)
    rmse = np.full(5, np.nan)
    a, b = (track_new_coarse(g, T_try, AFF, 1.05, rmse, affine_opt_mode_a=1e12, affine_opt_mode_b=1e8) for g in (ts, ref))
    for k in a:
        if k == "per_try":
            assert all(same(x[j], y[j]) for x, y in zip(a[k], b[k]) for j in x)
        elif k not in drop:
            assert same(a[k], b[k]), k


def test_shim_runs_set_coarse_tracking_ref():
    exe = os.path.join(ROOT, "tests", "cpp", "shim_coarse_ref")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "shim_coarse_ref: OK" in r.stdout
