"""Option cases of the TSDF engine's option sweep: voxel size, truncation, image size, intrinsics, sensor range, weight
ceiling and hash geometry, each case varying several of them at once.  Shared by tests/test_fusion_options_gpu.py,
tests/test_fusion_options_cpu.py and oracle/gen_reference_pins_fusion_options.py."""
import numpy as np

from tandem_b200.synthetic import RoomScene, circle_trajectory, look_at_pose

_BASE = dict(voxel_size=0.01, truncation_distance=0.04, height=120, width=160, fx=80.0, fy=80.0, cx=79.5, cy=59.5,
             num_buckets=200003, bucket_size=10, num_blocks=120000)

CASES = {
    # the reference's own example configuration (dr_debug_example.cpp: voxel 0.02, truncation 0.1)
    "ref_example": dict(_BASE, voxel_size=0.02, truncation_distance=0.1),
    # fx != fy, an integer principal point (rays exactly parallel to axis planes) and partial 8x8 / 16x16 tiles on both axes
    "aniso_odd": dict(_BASE, height=121, width=163, fx=81.5, fy=77.25, cx=80.0, cy=61.0),
    # 4 cm blocks: eight times the blocks of the default per metre of surface
    "fine": dict(_BASE, voxel_size=0.005, truncation_distance=0.02, height=97, width=131, fx=70.0, fy=90.0, cx=65.5, cy=48.5,
                 num_blocks=400000),
    # tau < 2 voxels: the ray-cast's hits land close to its `sdf < voxel_size` test; portrait image
    "narrow_band": dict(_BASE, voxel_size=0.04, truncation_distance=0.05, height=160, width=120, fx=100.0, fy=95.0,
                        cx=59.5, cy=79.5),
    # a narrow sensor range with depths placed exactly on both limits, at the two ends of the u8 weight
    "range_w1": dict(_BASE, min_sensor_depth=0.5, max_sensor_depth=2.0, max_sdf_weight=1),
    "range_w255": dict(_BASE, min_sensor_depth=0.5, max_sensor_depth=2.0, max_sdf_weight=255),
    # hash geometry: a power-of-two bucket count, and a small prime one with deep buckets
    "hash_pow2": dict(_BASE, num_buckets=65536),
    "hash_1009": dict(_BASE, num_buckets=1009, bucket_size=64),
}

SCENE = RoomScene(half=1.2, spheres=((0.5, 0.1, 0.4, 0.3), (-0.4, -0.2, 0.6, 0.25), (0.1, 0.4, -0.6, 0.3)))
# world shift: no multiple of any case's block size, and the room still spans negative and positive block coordinates
SHIFT = np.float32([0.337, -0.211, 0.129])
N_SCANS = 4


def options(name, **kw):
    from tandem_b200 import DrFusionOptions
    c = dict(CASES[name])
    c.update(kw)
    return DrFusionOptions(**c)


def intrinsics(name):
    c = CASES[name]
    return c["height"], c["width"], c["fx"], c["fy"], c["cx"], c["cy"]


def _axis_pose(R, t):
    T = np.eye(4, dtype=np.float32)
    T[:3, :3] = R
    T[:3, 3] = t
    return T


def scan_poses():
    """Poses 30 degrees apart on an arc (the 90 degree view cones overlap by two thirds), then the first pose again: every
    voxel seen twice is averaged (weights up to N_SCANS), so K6's running mean of sdf and colour and the weight ceiling
    are exercised."""
    arc = circle_trajectory(12, radius=0.3, phase=-np.pi / 3)[:N_SCANS - 1]     # -60, -30, 0 degrees: clear of the spheres
    return arc + [arc[0].copy()]


def scans(name, shift=SHIFT):
    """N_SCANS (bgr, depth, pose) of the room (scan_poses), world shifted by `shift`; each scan has its own noise and
    drop-outs.  The range cases put rows of depths exactly on min_sensor_depth / max_sensor_depth and one float beyond each."""
    H, W, fx, fy, cx, cy = intrinsics(name)
    c = CASES[name]
    out = []
    for k, p in enumerate(scan_poses()):
        bgr, depth = SCENE.render(p, H, W, fx, fy, cx, cy, noise_sigma=0.002, dropout=0.02, seed=k)
        if "min_sensor_depth" in c:
            lo, hi = np.float32(c["min_sensor_depth"]), np.float32(c["max_sensor_depth"])
            depth[10:14] = lo
            depth[14] = np.nextafter(lo, np.float32(0))
            depth[20:24] = hi
            depth[24] = np.nextafter(hi, np.float32(np.inf))
            depth[40:44, ::3] = lo
            depth[50:54, ::3] = hi
        q = p.copy()
        q[:3, 3] += shift
        out.append((bgr, depth, q))
    return out


def views(shift=SHIFT):
    """Render poses besides the scans' own: outside the room looking in, and two axis-aligned ones (identity rotation, from
    behind the wall the scans see, and a 90 degree turn about y, inside the room): with an integer principal point their
    centre column / row is exactly parallel to axis planes."""
    outside = look_at_pose((3.0, 0.2, 0.1), (0.0, 0.0, 0.0))
    outside[:3, 3] += shift
    ident = _axis_pose(np.eye(3, dtype=np.float32), np.float32([0.6, -0.03, -3.0]) + shift)    # behind the z = -1.2 wall
    rot90 = _axis_pose(np.float32([[0, 0, 1], [0, 1, 0], [-1, 0, 0]]), np.float32([-0.1, 0.02, 0.05]) + shift)
    return dict(outside=outside, axis_identity=ident, axis_rot90=rot90)


def mesh_boxes(name, shift=SHIFT):
    """Two boxes per case around the part of the room the scans see: one whose corners are whole multiples of the voxel
    size, one with arbitrary corners that cut blocks.  Sized so that the brute-force oracle visits at most ~1e7 cells."""
    vs = CASES[name]["voxel_size"]
    centre = shift + np.float32([0.55, 0.0, -0.3])
    half = min(1.3, 110 * vs)
    lo = np.round((centre - half) / vs) * vs
    up = np.round((centre + half) / vs) * vs
    aligned = (np.float32(lo), np.float32(up))
    a = min(1.0, 90 * vs)
    corner = shift + np.float32([0.85, 0.0, -0.85])                        # towards the two walls the scans see
    arb = (np.float32(corner + np.float32([-1.2345, -0.777, -1.1111]) * a), np.float32(corner + np.float32([0.9137, 1.0503, 0.8123]) * a))
    return [aligned, arb]
