"""Inputs of the n7 pin (SURVEY.md 8f): CoarseTracker::setCoarseTrackingRef with makeCoarseDepthL0 on every level.

Each case is one or more keyframes set one after the other on the same arrays (the second one sees the slots the first left
behind).  The points are seeded random plus the situations the reference's loops treat specially: many points on one pixel in
different orders, points in the 2-pixel border and on rows 0 / h-1, on the columns the flat-index dilation wraps (0, w-1), a
u whose float and double `+ 0.5` round differently (0.49999997f), idepth <= 0 (a rejected candidate behind the last accepted
point: the stale slot), and non-finite grey values.  Dense maps are RoomScene renders at a pose near the keyframe's."""
import hashlib

import numpy as np

from tandem_b200.synthetic import RoomScene, look_at_pose

GRAY_W = np.array([0.114, 0.587, 0.299], np.float32)
POSE_D = look_at_pose((0.3, 0.0, -0.2), (2.5, 0.2, 0.5))
POSE_R = look_at_pose((0.34, 0.02, -0.17), (2.5, 0.25, 0.45))

# name -> (h, w), levels, keyframes: list of dict(rgbd, n (random points), seed, dense (None | "host"), dense_only, step)
CASES = {
    "mono_640x480_l4_dense": ((480, 640), 4, [dict(rgbd=0, n=8000, seed=1, dense="host", dense_only=0, step=1)]),
    "mono_640x480_l4_empty": ((480, 640), 4, [dict(rgbd=0, n=0, seed=2, dense=None, dense_only=0, step=1)]),
    "mono_640x480_l4_dense_only": ((480, 640), 4, [dict(rgbd=0, n=0, seed=3, dense="host", dense_only=1, step=2)]),
    "rgbd_130x96_l3_dense": ((96, 130), 3, [dict(rgbd=1, n=3000, seed=4, dense="host", dense_only=0, step=2)]),
    "rgbd_130x96_l3": ((96, 130), 3, [dict(rgbd=1, n=3000, seed=5, dense=None, dense_only=0, step=1)]),
    "mono_80x60_l2_dense_only": ((60, 80), 2, [dict(rgbd=0, n=400, seed=6, dense="host", dense_only=1, step=2)]),
    "mono_130x96_l3_two_keyframes": ((96, 130), 3, [dict(rgbd=0, n=1500, seed=7, dense="host", dense_only=0, step=1),
                                                    dict(rgbd=0, n=200, seed=8, dense="host", dense_only=0, step=1)]),
    "rgbd_80x60_l2_two_keyframes": ((60, 80), 2, [dict(rgbd=1, n=300, seed=9, dense=None, dense_only=0, step=1),
                                                  dict(rgbd=1, n=0, seed=10, dense="host", dense_only=0, step=2)]),
}


def K4(h, w):
    f = 160.0 * w / 320.0
    return (f, f, (w - 1) / 2.0, (h - 1) / 2.0)


def gray_image(h, w, seed):
    """Keyframe grey image: the RoomScene view at POSE_R with a few non-finite pixels."""
    bgr, _ = RoomScene().render(POSE_R, h, w, *K4(h, w))
    g = bgr.astype(np.float32) @ GRAY_W
    rng = np.random.default_rng(100 + seed)
    for val in (np.inf, np.nan, -np.inf):
        ys, xs = rng.integers(2, h - 2, 3), rng.integers(2, w - 2, 3)
        g[ys, xs] = val
    g[h - 4, w // 2] = np.nan
    return g


def dense_depth(h, w):
    _, depth = RoomScene().render(POSE_D, h, w, *K4(h, w), dropout=0.02, seed=1)
    return depth


def points(h, w, kf):
    """(u, v, idepth, hessian) float32 in input order."""
    rng = np.random.default_rng(kf["seed"])
    n = kf["n"]
    u = list(rng.uniform(-0.49, w - 0.51, n))
    v = list(rng.uniform(-0.49, h - 0.51, n))
    idepth = list(rng.uniform(0.1, 2.0, n))
    if n:
        # many points on one pixel, in different orders / mixed with others
        for k in range(12):
            u.insert(k * (len(u) // 13), 17.2 + 0.01 * k)
            v.insert(k * (len(v) // 13), 9.6 - 0.01 * k)
            idepth.insert(k * (len(idepth) // 13), 0.3 + 0.11 * k)
        # border band, rows 0 / h-1, wrap columns 0 / w-1
        for (x, y) in ((0.0, 5.0), (1.2, 7.0), (w - 1.0, 11.0), (w - 1.4, 3.0), (5.0, 0.0), (9.0, h - 1.0), (w - 2.0, h - 2.0),
                       (0.0, h - 3.0), (w - 1.0, 2.0), (3.0, 3.0)):
            u.append(x); v.append(y); idepth.append(float(rng.uniform(0.2, 1.5)))
        # float vs double rounding of + 0.5
        u += [0.49999997, 2.49999997, 4.4999995]
        v += [6.0, 0.49999997, 8.4999995]
        idepth += [0.7, 0.8, 0.9]
        # idepth <= 0, one of them behind every accepted point of level 0 (the stale slot)
        u += [40.0, 41.0, w - 3.0]
        v += [20.0, 20.0, h - 3.0]
        idepth += [-0.5, 0.0, -1.0]
    u, v, idepth = (np.array(a, np.float32) for a in (u, v, idepth))
    m = len(u)
    hess = (rng.uniform(0.1, 5.0, m) if kf["rgbd"] else rng.uniform(1e-4, 3.0, m)).astype(np.float32)
    if kf["rgbd"]:
        # RGB-D rounds in double: keep every point inside for (int)(u + 0.5)
        u = np.clip(u, -0.49, w - 0.51).astype(np.float32)
        v = np.clip(v, -0.49, h - 0.51).astype(np.float32)
    return u, v, idepth, hess


def digest(*arrays):
    """sha256 over the bytes of the arrays; every NaN is replaced by one canonical NaN first."""
    h = hashlib.sha256()
    for a in arrays:
        a = np.ascontiguousarray(a)
        if a.dtype.kind == "f":
            a = np.where(np.isnan(a), np.array(np.nan, a.dtype), a)
        h.update(str((a.dtype.str, a.shape)).encode())
        h.update(a.tobytes())
    return h.hexdigest()


def case_inputs(name):
    """(size, levels, gray pyramid [(h_l, w_l) grey of level l], dense depth, [keyframes with their points])."""
    from oracle.cpu import FrontOracle
    (h, w), levels, kfs = CASES[name]
    pyr = FrontOracle().make_images(gray_image(h, w, 0), levels)
    gray_levels = [np.ascontiguousarray(p[0][..., 0]) for p in pyr]
    depth = dense_depth(h, w) if any(k["dense"] for k in kfs) else None
    return (h, w), levels, gray_levels, depth, [dict(k, points=points(h, w, k) if k["n"] else None) for k in kfs]


def run_oracle(name, T_depth_to_ref):
    """Runs the case through oracle/coarse_ref_oracle.c; returns [(pc_n, per-level arrays incl. slot pc_n)] per keyframe."""
    from oracle.coarse_ref import CoarseRefOracle
    (h, w), levels, gray_levels, depth, kfs = case_inputs(name)
    o = CoarseRefOracle(w, h, levels)
    out = []
    for kf in kfs:
        pc_n = o.set_coarse_tracking_ref(kf["points"], gray_levels, kf["rgbd"], depth if kf["dense"] else None, T_depth_to_ref,
                                         K4(h, w), kf["step"], kf["dense_only"])
        out.append((pc_n, o.result(pc_n)))
    return out
