"""Inputs of the tests that are pinned against the reference's own code, and the digest those tests compare.

The reference runs only where its sources are (oracle/gen_reference_pins.py compiles and runs it there); what it computed
on these inputs is stored under tests/golden/ so that the pins hold on any checkout."""
import hashlib

import numpy as np

from tandem_b200.synthetic import RoomScene, circle_trajectory, look_at_pose, tracker_case

MAKE_IMAGES_CASES = [((480, 640), 4), ((96, 130), 2), ((60, 80), 3)]
DENSE_REF_CASES = [(1, False, (240, 320)), (2, True, (240, 320)), (1, True, (120, 160)), (3, False, (480, 640))]
LM_CASES = [("identity", False, False, 20.0), ("near", False, False, 20.0), ("identity", True, True, 20.0),
            ("identity", False, True, 20.0), ("identity", True, False, 20.0), ("identity", False, False, 0.8)]


def digest(*arrays):
    """sha256 over the bytes of the arrays; every NaN is replaced by one canonical NaN first (the pins compare with
    equal_nan semantics)."""
    h = hashlib.sha256()
    for a in arrays:
        a = np.ascontiguousarray(a)
        if a.dtype.kind == "f":
            a = np.where(np.isnan(a), np.array(np.nan, a.dtype), a)
        h.update(str((a.dtype.str, a.shape)).encode())
        h.update(a.tobytes())
    return h.hexdigest()


def make_images_input(size):
    h, w = size
    rng = np.random.default_rng(3)
    gray = (rng.random((h, w)) * 255).astype(np.float32)
    gray[5, 7] = np.inf
    return gray


def dense_reference_input(step, with_sparse, size):
    h, w = size
    f = 160.0 * w / 320.0
    K4 = (f, f, (w - 1) / 2.0, (h - 1) / 2.0)
    scene = RoomScene()
    pose_d = look_at_pose((0.3, 0.0, -0.2), (2.5, 0.2, 0.5))
    pose_r = look_at_pose((0.34, 0.02, -0.17), (2.5, 0.25, 0.45))
    _, depth = scene.render(pose_d, h, w, *K4, dropout=0.02, seed=1)
    bgr_r, _ = scene.render(pose_r, h, w, *K4)
    gray_r = bgr_r.astype(np.float32) @ np.array([0.114, 0.587, 0.299], np.float32)
    rng = np.random.default_rng(5)
    sparse, idepth0 = None, None
    if with_sparse:
        ns = 500
        sparse = [rng.integers(3, w - 3, ns + 1).astype(np.float32), rng.integers(3, h - 3, ns + 1).astype(np.float32),
                  rng.uniform(0.2, 2.0, ns + 1).astype(np.float32), rng.uniform(0, 255, ns + 1).astype(np.float32)]
        idepth0 = np.zeros((h, w), np.float32)
        idepth0[sparse[1][:ns].astype(int), sparse[0][:ns].astype(int)] = sparse[2][:ns]
    return dict(depth=depth, pose_d=pose_d, pose_r=pose_r, K4=K4, step=step, dense_only=not with_sparse, sparse=sparse,
                idepth0=idepth0, gray_r=gray_r)


def lm_case():
    return tracker_case(H=120, W=160, fx=80.0, fy=80.0, cx=79.5, cy=59.5)


def lm_start(c, start):
    return np.eye(4) if start == "identity" else np.array(c["refToNew"], np.float64) @ np.linalg.inv(
        np.array([[1, 0, 0, 0.004], [0, 1, 0, -0.003], [0, 0, 1, 0.002], [0, 0, 0, 1.0]]))


def fresh_model_input():
    """A seeded synthetic 4-view window at 96x64 for the model pin: images, per-stage intrinsics, cam->world poses."""
    import torch
    torch.manual_seed(0)
    V, H, W = 4, 64, 96
    img = torch.rand(V, 3, H, W)
    img = torch.nn.functional.avg_pool2d(img, 5, 1, 2)
    K3 = torch.tensor([[100.0, 0, 47.5], [0, 100.0, 31.5], [0, 0, 1]])
    Ks = [torch.cat([K3[:2] * s, K3[2:]]) for s in (0.25, 0.5, 1.0)]
    c2w = torch.eye(4).repeat(V, 1, 1)
    c2w[:, 0, 3] = torch.arange(V) * 0.05
    return img, Ks, c2w


TRACKER_CASES = [((120, 160), 1), ((480, 640), 1)]
WARPED_SAMPLE = 20000   # points of the reference's per-point output kept for the tracker pin (seeded sample)


def fusion_setup(n_poses, paired):
    """TSDF scene of the fusion / mesh pins: options, poses (world shifted by +2.56 m), rendered (bgr, depth) frames."""
    from tandem_b200 import DrFusionOptions
    H, W = 120, 160
    intr = dict(fx=80.0, fy=80.0, cx=79.5, cy=59.5)
    opt = DrFusionOptions(height=H, width=W, num_buckets=200003, bucket_size=10, num_blocks=120000, **intr)
    # world shifted by +2.56 m (32 blocks): the reference also integrates its FREE hash entries, all aliased to block (0,0,0);
    # keeping the origin far outside the map keeps that quirk out of the comparison.
    off = np.array([2.56, 2.56, 2.56], np.float32)
    scene = RoomScene(half=1.2, spheres=((0.5, 0.1, 0.4, 0.3), (-0.4, -0.2, 0.6, 0.25), (0.1, 0.4, -0.6, 0.3)))
    poses = circle_trajectory(n_poses, radius=0.3)
    if paired:
        poses = [poses[0], poses[0].copy(), poses[1], poses[1].copy()]
        poses[1][:3, 3] += np.float32(0.03)
        poses[3][:3, 3] -= np.float32(0.02)
    frames = [scene.render(p, H, W, **intr, noise_sigma=0.002, dropout=0.02, seed=k) for k, p in enumerate(poses)]
    for p in poses:
        p[:3, 3] += off
    return opt, poses, frames, off


def tracker_pin_case(size, step):
    h, w = size
    s = w / 640.0
    return tracker_case(H=h, W=w, fx=320.0 * s, fy=320.0 * s, cx=319.5 * s, cy=239.5 * s, step=step)


def warped_sample(n):
    rng = np.random.default_rng(0)
    return np.sort(rng.choice(n, min(n, WARPED_SAMPLE), replace=False))
