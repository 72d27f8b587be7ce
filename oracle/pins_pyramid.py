"""Inputs of the coarse-to-fine pin (SURVEY.md 8f n5): one synthetic scene, four pyramid levels, five cases.

Every level is built the way tandem_b200/loop.py builds it on the device: the new frame's pyramid (FrameHessian::makeImages,
n2) and, per level, a dense tracking reference (n1) from the reference view's depth sub-sampled to that level and the
reference view's grey pyramid level.  Here both come from the CPU restatements oracle/front_oracle.c, which equal the device
kernels bit for bit, so the same inputs drive the reference's body (oracle/gen_reference_pins_pyramid.py), the restatement
(oracle/pyramid_driver.py) and, rebuilt on the GPU, tdm_tracker_track_pyramid."""
import numpy as np

from tandem_b200.synthetic import RoomScene, look_at_pose

H, W, LEVELS = 240, 320, 4
K0 = (160.0, 160.0, 159.5, 119.5)
GRAY_W = np.array([0.114, 0.587, 0.299], np.float32)
REF_AFF = np.array([0.01, 1.5])
NAN5 = (float("nan"),) * 5

# name -> call arguments (coarse_cutoff, new_exposure, mode_a, mode_b, min_res_for_abort); ref_exposure is 1
CASES = {
    "converge": dict(coarse_cutoff=20.0, new_exposure=1.05, mode_a=1e12, mode_b=1e8, min_res=NAN5),
    "repeat": dict(coarse_cutoff=5.0, new_exposure=1.05, mode_a=1e12, mode_b=1e8, min_res=NAN5),
    "abort": dict(coarse_cutoff=20.0, new_exposure=1.05, mode_a=1e12, mode_b=1e8, min_res=(np.nan, np.nan, 1.0, np.nan, np.nan)),
    # exposure ratio e^2: `a` moves to about -2; with a prior on it (mode != 0) |a| > 1.2 rejects the result (:923-924), with
    # mode 0 the relative brightness check (:928-930) sees the compensated ratio and accepts
    "affine": dict(coarse_cutoff=20.0, new_exposure=float(np.exp(2.0)), mode_a=1e12, mode_b=1e8, min_res=NAN5),
    "affine_mode0": dict(coarse_cutoff=20.0, new_exposure=float(np.exp(2.0)), mode_a=0.0, mode_b=0.0, min_res=NAN5),
    "fixed_a": dict(coarse_cutoff=20.0, new_exposure=1.05, mode_a=-1.0, mode_b=1e8, min_res=NAN5),
    "fixed_ab": dict(coarse_cutoff=20.0, new_exposure=1.05, mode_a=-1.0, mode_b=-1.0, min_res=NAN5),
}


def intrinsics(w):
    """K0 scaled to an image w pixels wide (pins: 320, benchmark: 640)."""
    s = w / W
    return (K0[0] * s, K0[1] * s, (K0[2] + 0.5) * s - 0.5, (K0[3] + 0.5) * s - 0.5)


def level_K(l, K=K0):
    fx, fy, cx, cy = K
    return (fx / 2 ** l, fy / 2 ** l, (cx + 0.5) / 2 ** l - 0.5, (cy + 0.5) / 2 ** l - 0.5)   # globalCalib.cpp:84-90


def scene(h=H, w=W):
    """(gray_new (h,w), gray_ref (h,w), depth_ref (h,w), refToNew (4,4) true relative pose)."""
    s = RoomScene()
    ref_pose = look_at_pose((0.3, 0.0, -0.2), (2.5, 0.2, 0.5))
    new_pose = look_at_pose((0.33, 0.01, -0.18), (2.5, 0.22, 0.52))
    bgr_r, depth_r = s.render(ref_pose, h, w, *intrinsics(w))
    bgr_n, _ = s.render(new_pose, h, w, *intrinsics(w))
    T = np.linalg.inv(new_pose.astype(np.float64)) @ ref_pose.astype(np.float64)
    return bgr_n.astype(np.float32) @ GRAY_W, bgr_r.astype(np.float32) @ GRAY_W, depth_r, T


def level_inputs():
    """Per level l: dict(w, h, K, n, pc (u, v, idepth, color; n + 1 entries each), dI (h, w, 3) of the new frame)."""
    from oracle.cpu import FrontOracle
    f = FrontOracle()
    gray_n, gray_r, depth_r, _ = scene()
    new_pyr = f.make_images(gray_n, LEVELS)
    ref_pyr = f.make_images(gray_r, LEVELS)
    out = []
    for l in range(LEVELS):
        K = level_K(l)
        d = np.ascontiguousarray(depth_r[::2 ** l, ::2 ** l])
        g = np.ascontiguousarray(ref_pyr[l][0][..., 0])
        n, arrs, _ = f.dense_reference(d, np.eye(4), K, 1, True, None, None, g)
        out.append(dict(w=W >> l, h=H >> l, K=K, n=n, pc=arrs, dI=new_pyr[l][0]))
    return out


def oracle_trackers(levels):
    """One oracle/tracker_oracle.c tracker per level, set up from level_inputs()."""
    from oracle.cpu import TrackerOracle
    ts = []
    for x in levels:
        t = TrackerOracle(x["w"], x["h"])
        t.setK(x["w"], x["h"], *x["K"])
        t.setReference(x["n"], *[a[:x["n"]] for a in x["pc"]], 1.0, REF_AFF)
        t.setNew(x["dI"])
        ts.append(t)
    return ts
