"""GPU parity of the TSDF path (DrFusion call surface, through the C ABI) against the sequential CPU oracle.
Bar (SURVEY.md §8d config 3): set of allocated block coordinates and block count bit-exact, per-voxel weight and
colour exact, sdf within 1e-5, rendered depth/colour equal."""
import numpy as np
import pytest

from oracle.cpu import TsdfOracle
from tandem_b200 import DrFusion, DrFusionOptions
from tandem_b200.synthetic import RoomScene, circle_trajectory, look_at_pose

pytestmark = pytest.mark.gpu

H, W = 120, 160
INTR = dict(fx=80.0, fy=80.0, cx=79.5, cy=59.5)


def _opts(**kw):
    base = dict(height=H, width=W, num_buckets=200003, bucket_size=10, num_blocks=120000, **INTR)
    base.update(kw)
    return DrFusionOptions(**base)


SCENE = RoomScene(half=1.2, spheres=((0.5, 0.1, 0.4, 0.3), (-0.4, -0.2, 0.6, 0.25), (0.1, 0.4, -0.6, 0.3)))


def _render(poses, seed=0):
    return [SCENE.render(p, H, W, INTR["fx"], INTR["fy"], INTR["cx"], INTR["cy"], noise_sigma=0.002, dropout=0.02,
                         seed=seed + k) for k, p in enumerate(poses)]


def _scene_frames(n, seed=0):
    poses = circle_trajectory(n, radius=0.3)
    return poses, _render(poses, seed)


def _compare_maps(f, o):
    cg, vg = f.dump_blocks()
    co, vo = o.dump_blocks()
    assert cg.shape == co.shape, f"block count {cg.shape[0]} vs oracle {co.shape[0]}"
    assert np.array_equal(cg, co), "allocated block coordinate sets differ"
    assert np.array_equal(vg["weight"], vo["weight"]), "voxel weights differ"
    assert np.array_equal(vg["color"], vo["color"]), "voxel colours differ"
    assert np.max(np.abs(vg["sdf"] - vo["sdf"])) <= 1e-5
    return cg.shape[0], float(np.mean(vg["sdf"] == vo["sdf"]))


def test_integrate_and_render_match_oracle():
    poses, frames = _scene_frames(4)
    poses = [poses[0], poses[0].copy(), poses[1], poses[1].copy()]
    poses[1][:3, 3] += np.float32(0.03)
    poses[3][:3, 3] -= np.float32(0.02)
    frames = _render(poses)
    f = DrFusion(_opts())
    o = TsdfOracle(_opts())
    for k, (pose, (bgr, depth)) in enumerate(zip(poses, frames)):
        f.IntegrateScanAsync(bgr, depth, pose)
        o.integrate(bgr, depth, pose)
        rp = poses[max(k - 1, 0)] if k % 2 else pose   # alternate: the view just integrated / the previous one
        f.RenderAsync([rp])
        (rb,), (rd,) = f.GetRenderResult()
        ob, od = o.render(rp)
        sg, so = f.stats(), o.stats()
        assert sg["allocated_blocks"] == so["allocated_blocks"]
        assert sg["visible_blocks"] == so["visible_blocks"]
        assert sg["dropped_blocks"] == so["dropped_blocks"] == 0
        hit_g, hit_o = rd > 0, od > 0
        assert np.mean(hit_g != hit_o) <= 1e-3
        both = hit_g & hit_o
        assert both.mean() > 0.5
        assert np.mean(np.abs(rd[both] - od[both])) <= 1e-3
        assert np.mean(rd == od) > 0.999, f"rendered depth bit-equality {np.mean(rd == od)}"
        assert np.mean(rb == ob) > 0.999
    nblk, exact = _compare_maps(f, o)
    print(f"blocks {nblk}, sdf bit-exact fraction {exact:.6f}")
    assert exact > 0.9999


def test_negative_coordinates_and_far_plane():
    """camera in the negative octant looking towards -x/-z; depth beyond max_sensor_depth and below min are ignored."""
    scene = RoomScene(half=1.0, spheres=((-0.5, 0.0, -0.5, 0.2),))
    pose = look_at_pose((-0.2, 0.05, -0.1), (-1.0, 0.0, -0.9))
    bgr, depth = scene.render(pose, H, W, **INTR)
    depth[:10] = 25.0   # > max_sensor_depth
    depth[10:20] = 0.05  # < min_sensor_depth
    depth[20:22] = -1.0
    f, o = DrFusion(_opts()), TsdfOracle(_opts())
    f.IntegrateScanAsync(bgr, depth, pose)
    o.integrate(bgr, depth, pose)
    f.RenderAsync([pose])
    f.GetRenderResult()
    _compare_maps(f, o)
    assert (f.dump_blocks(False)[0] < 0).any()


def test_weight_saturates_at_max():
    poses, frames = _scene_frames(1)
    f, o = DrFusion(_opts(max_sdf_weight=3)), TsdfOracle(_opts(max_sdf_weight=3))
    for _ in range(5):
        f.IntegrateScanAsync(frames[0][0], frames[0][1], poses[0])
        o.integrate(frames[0][0], frames[0][1], poses[0])
        f.RenderAsync([poses[0]])
        f.GetRenderResult()
    _compare_maps(f, o)
    assert f.dump_blocks()[1]["weight"].max() == 3


def test_call_order_state_machine():
    """Integrate -> Render -> GetRenderResult is enforced (tsdf_volume.cu:520-525,635-640,703-708)."""
    poses, frames = _scene_frames(1)
    f = DrFusion(_opts())
    with pytest.raises(Exception):
        f.RenderAsync([poses[0]])
    f.IntegrateScanAsync(frames[0][0], frames[0][1], poses[0])
    with pytest.raises(Exception):
        f.IntegrateScanAsync(frames[0][0], frames[0][1], poses[0])
    with pytest.raises(Exception):
        f.RenderAsync([poses[0], poses[0]])   # size must equal num_render_streams (tsdf_volume.cu:643-648)
    f.RenderAsync([poses[0]])
    f.GetRenderResult()
    f.IntegrateScanAsync(frames[0][0], frames[0][1], poses[0])


def test_bucket_overflow_drops_blocks():
    """A full bucket drops the block (hash_table.cu:103-115): never more than bucket capacity, never a crash."""
    poses, frames = _scene_frames(1)
    f = DrFusion(_opts(num_buckets=101, bucket_size=2, num_blocks=1000))
    f.IntegrateScanAsync(frames[0][0], frames[0][1], poses[0])
    f.RenderAsync([poses[0]])
    f.GetRenderResult()
    s = f.stats()
    assert 0 < s["allocated_blocks"] <= 202 and s["dropped_blocks"] > 0
    coords, _ = f.dump_blocks()
    assert len({tuple(c) for c in coords}) == coords.shape[0], "duplicate blocks"


def test_full_size_properties():
    """640x480 frame into the initDr-sized map: idempotent block set on re-integration, render of the integrated
    view reproduces the input depth to ~1 voxel where both are valid."""
    scene = RoomScene()
    pose = look_at_pose((0.3, 0.0, -0.2), (2.5, 0.2, 0.5))
    bgr, depth = scene.render(pose, 480, 640, 320.0, 320.0, 319.5, 239.5)
    f = DrFusion(DrFusionOptions())
    f.IntegrateScanAsync(bgr, depth, pose)
    f.RenderAsync([pose]); f.GetRenderResult()
    n1 = f.stats()["allocated_blocks"]
    f.IntegrateScanAsync(bgr, depth, pose)
    f.RenderAsync([pose])
    (rb,), (rd,) = f.GetRenderResult()
    s = f.stats()
    assert s["allocated_blocks"] == n1 and s["candidate_blocks"] == 0 and s["dropped_blocks"] == 0
    ok = (rd > 0) & (depth > 0.1)
    assert ok.mean() > 0.9
    assert np.median(np.abs(rd[ok] - depth[ok])) < 0.01


def test_config3_shape_matches_oracle():
    """BASELINE.json configs[2] shape (VERDICT r01): 640x480 depth maps of the config-3 scene (5 m room + 3 spheres, camera
    circle r = 1 m, 2 mm noise, 2 % drop-outs) into the initDr-sized map (1 M buckets x 10, 1 M blocks, FullSystem.cpp:259-276):
    block set / count / weights / colours exact, sdf <= 1e-5, render of each integrated view equal to the oracle's."""
    hh, ww = 480, 640
    intr = dict(fx=320.0, fy=320.0, cx=319.5, cy=239.5)
    scene = RoomScene()
    poses = circle_trajectory(3, radius=1.0)
    frames = [scene.render(p, hh, ww, **intr, noise_sigma=0.002, dropout=0.02, seed=k) for k, p in enumerate(poses)]
    for p in poses:
        p[:3, 3] += np.float32(5.12)     # the 5.12 m cube of config 3; keeps block (0,0,0) out of the map (SURVEY Appendix B.2)
    f, o = DrFusion(DrFusionOptions(height=hh, width=ww, **intr)), TsdfOracle(DrFusionOptions(height=hh, width=ww, **intr))
    for k, ((bgr, depth), pose) in enumerate(zip(frames, poses)):
        f.IntegrateScanAsync(bgr, depth, pose)
        o.integrate(bgr, depth, pose)
        f.RenderAsync([pose])
        (rb,), (rd,) = f.GetRenderResult()
        sg, so = f.stats(), o.stats()
        assert sg["allocated_blocks"] == so["allocated_blocks"] and sg["visible_blocks"] == so["visible_blocks"]
        assert sg["dropped_blocks"] == so["dropped_blocks"] == 0
        if k == 0:
            continue                      # the oracle's ray-cast takes ~8 s per 640x480 view: two views are compared
        ob, od = o.render(pose)
        hit_g, hit_o = rd > 0, od > 0
        assert np.mean(hit_g != hit_o) <= 1e-3
        both = hit_g & hit_o
        assert both.mean() > 0.9
        assert np.mean(np.abs(rd[both] - od[both])) <= 1e-3
        assert np.mean(rd == od) > 0.999, f"rendered depth bit-equality {np.mean(rd == od)}"
        assert np.mean(rb == ob) > 0.999
    nblk, exact = _compare_maps(f, o)
    print(f"config-3 shape: {nblk} blocks after 3 frames, sdf bit-exact fraction {exact:.6f}")
    assert nblk > 20000 and exact > 0.9999


def test_raycast_is_bit_identical_to_reference_sampler():
    """Every ray-cast variant must put every sample where the reference's GetInterpolatedVoxel march puts it: the kernel
    that mirrors the reference sampler voxel by voxel (raycast_shared=0: one hash lookup per voxel, IEEE divisions, sgn()) and
    the production kernel (shared per-axis index arithmetic, one lookup per DISTINCT block of a sample, division-free hash,
    select-form rounding), with and without constant-divisor division, render the same volume bit for bit, depth and colour,
    at 160x120 - views from inside the map, from outside looking in and looking away, a pose 100 m from the origin, a Z-slab
    volume - and at the config-3 shape."""
    variants = [{"raycast_shared": 0}, {}, {"fast_div": 1}]

    def run(make, scans, views):
        vols = []
        for opts in variants:
            f = make()
            for k, v in opts.items():
                f.set_option(k, v)
            vols.append(f)
        cover = []
        for k, q in enumerate(views):
            bgr, depth, pose = scans[min(k, len(scans) - 1)]
            ref = None
            for opts, f in zip(variants, vols):
                f.IntegrateScanAsync(bgr, depth, pose)
                f.RenderAsync([q])
                (rb,), (rd,) = f.GetRenderResult()
                if ref is None:
                    ref = (rd.copy(), rb.copy())
                    cover.append(float((rd > 0).mean()))
                else:
                    assert np.array_equal(ref[0].view(np.uint32), rd.view(np.uint32)) and np.array_equal(ref[1], rb), (k, opts)
        return cover

    poses, frames = _scene_frames(3)
    for shift, slab in ((0.0, None), (-7.3, None), (100.0, None), (0.0, (-4, 3))):
        ps = [p.copy() for p in poses]
        for p in ps:
            p[:3, 3] += np.float32(shift)
        outside = look_at_pose((3.0, 0.2, 0.1), (0.0, 0.0, 0.0)); outside[:3, 3] += np.float32(shift)    # outside, looking in
        away = look_at_pose((3.0, 3.0, 3.0), (3.0, 8.0, 4.0)); away[:3, 3] += np.float32(shift)          # outside, looking away

        def make():
            f = DrFusion(_opts())
            if slab:
                f.set_slab(*slab)
            return f
        scans = [(bgr, depth, pose) for (bgr, depth), pose in zip(frames, ps)]
        cover = run(make, scans, [ps[0], ps[1], ps[2], ps[0], outside, away])
        assert slab or min(cover[:4]) > 0.3, cover
        assert cover[5] == 0.0, cover
    hh, ww = 480, 640
    intr = dict(fx=320.0, fy=320.0, cx=319.5, cy=239.5)
    scene = RoomScene()
    ps = circle_trajectory(2, radius=1.0)
    fr = [scene.render(p, hh, ww, **intr, noise_sigma=0.002, dropout=0.02, seed=k) for k, p in enumerate(ps)]
    for p in ps:
        p[:3, 3] += np.float32(5.12)
    scans = [(bgr, depth, pose) for (bgr, depth), pose in zip(fr, ps)]
    cover = run(lambda: DrFusion(DrFusionOptions(height=hh, width=ww, num_buckets=200003, num_blocks=150000, **intr)), scans, [ps[0], ps[1], ps[0]])
    assert min(cover) > 0.3, cover


def test_z_slab_partition_matches_single_volume():
    """SURVEY.md 8e: two Z-slabs (each + 1 halo block) integrated from the same scans reproduce the single-volume map on
    their owned blocks bit-for-bit, and the per-pixel nearest-hit reduction of the two slab renders reproduces the
    single-volume render (same surface; sample positions differ where a ray restarts in another slab)."""
    from tandem_b200.parallel import reduce_nearest_hit, slab_bounds, pack_hits, unpack_hits
    poses, frames = _scene_frames(3)
    full = DrFusion(_opts())
    for (bgr, depth), pose in zip(frames, poses):
        full.IntegrateScanAsync(bgr, depth, pose)
        full.RenderAsync([pose]); full.GetRenderResult()
    cf, vf = full.dump_blocks()
    zmin, zmax = int(cf[:, 2].min()), int(cf[:, 2].max()) + 1
    slabs, renders = [], []
    for r in range(2):
        lo, hi, alo, ahi = slab_bounds(zmin, zmax, r, 2)
        f = DrFusion(_opts())
        f.set_slab(alo, ahi)
        for (bgr, depth), pose in zip(frames, poses):
            f.IntegrateScanAsync(bgr, depth, pose)
            f.RenderAsync([poses[0]])
            (rb,), (rd,) = f.GetRenderResult()
        c, v = f.dump_blocks()
        own = (c[:, 2] >= lo) & (c[:, 2] < hi)
        slabs.append((c[own], v[own]))
        renders.append((rd.copy(), rb.copy()))
    cu = np.concatenate([s[0] for s in slabs]); vu = np.concatenate([s[1] for s in slabs])
    order = np.lexsort((cu[:, 2], cu[:, 1], cu[:, 0]))
    assert np.array_equal(cu[order], cf), "union of owned slab blocks != single volume block set"
    assert np.array_equal(vu[order]["weight"], vf["weight"]) and np.array_equal(vu[order]["sdf"], vf["sdf"])
    full.IntegrateScanAsync(frames[0][0], frames[0][1], poses[0])   # advance the state machine; weights change but not the test
    keys = np.minimum(pack_hits(*renders[0]), pack_hits(*renders[1]))
    dm, bm = unpack_hits(keys)
    f2 = DrFusion(_opts())
    for (bgr, depth), pose in zip(frames, poses):
        f2.IntegrateScanAsync(bgr, depth, pose)
        f2.RenderAsync([poses[0]])
        (fb,), (fd,) = f2.GetRenderResult()
    hit_m, hit_f = dm > 0, fd > 0
    assert np.mean(hit_m != hit_f) < 5e-3
    both = hit_m & hit_f
    assert np.median(np.abs(dm[both] - fd[both])) < 1e-3 and np.quantile(np.abs(dm[both] - fd[both]), 0.99) < 0.02


@pytest.mark.parametrize("world", [2, 3])
def test_pixel_partitioned_raycast_over_peer_slabs_is_bit_identical(world):
    """The fused form of the slab exchange (tdm_fusion_peer_export / peer_attach): each rank integrates only its OWN Z-slab (no
    halo rows), renders only its pixel tiles, but marches them through the whole volume reading every voxel from the owning
    rank's tables.  The MIN-combined render must equal the single-volume render BIT FOR BIT (depth and colour) - occluders in
    other slabs included - which the slab-local ray-cast cannot deliver.  Here the ranks are instances of one process."""
    from tandem_b200.parallel import pack_hits, unpack_hits
    poses, frames = _scene_frames(3)
    full = DrFusion(_opts())
    for (bgr, depth), pose in zip(frames, poses):
        full.IntegrateScanAsync(bgr, depth, pose)
        full.RenderAsync([poses[1]])
        (fb,), (fd,) = full.GetRenderResult()
    cf, _ = full.dump_blocks()
    zmin, zmax = int(cf[:, 2].min()), int(cf[:, 2].max()) + 1
    n = zmax - zmin
    bounds = [zmin + (n * r) // world for r in range(world)] + [zmax]
    bounds[0], bounds[-1] = -(1 << 19), 1 << 19                      # the outer slabs own everything beyond the map
    ranks = []
    for r in range(world):
        f = DrFusion(_opts())
        f.set_slab(bounds[r], bounds[r + 1])
        ranks.append(f)
    blobs = [f.peer_export() for f in ranks]
    for r, f in enumerate(ranks):
        f.peer_attach(blobs, r)
    keys = None
    for k, ((bgr, depth), pose) in enumerate(zip(frames, poses)):
        for f in ranks:
            f.IntegrateScanAsync(bgr, depth, pose)
        for f in ranks:
            f.Synchronize()                                           # the barrier between integration and the peer reads
        rend = []
        for f in ranks:
            f.RenderAsync([poses[1]])
            (rb,), (rd,) = f.GetRenderResult()
            rend.append((rd.copy(), rb.copy()))
    assert sum(f.stats()["allocated_blocks"] for f in ranks) == cf.shape[0], "slabs without halo partition the block set"
    tiles = [(rd > 0).sum() for rd, _ in rend]
    assert all(t > 0 for t in tiles), "every rank must have rendered some of the pixels"
    for rd, rb in rend:
        kk = pack_hits(rd, rb)
        keys = kk if keys is None else np.minimum(keys, kk)
    dm, bm = unpack_hits(keys)
    assert np.array_equal(dm, fd), f"depth differs on {np.mean(dm != fd):.5f} of the pixels"
    assert np.array_equal(bm, fb)


@pytest.mark.parametrize("world,k", [(2, 1), (3, 2), (4, 1)])
def test_interleaved_slab_partition_matches_single_volume(world, k):
    """Interleaved Z-slabs (tdm_fusion_set_interleave: block row z -> rank ((z - z0) div k) mod world, + halo rows): the union of
    the OWNED blocks of all ranks is the single-volume map bit for bit, the slab-clipped ray-cast of each rank equals its own
    unclipped march bit for bit (skipped samples only ever read 'no voxel'), and the nearest-hit MIN over the ranks' renders
    reproduces the single-volume render (same surface; sample positions differ where a ray crosses a foreign slab)."""
    from tandem_b200.parallel import pack_hits, unpack_hits
    poses, frames = _scene_frames(3)
    full = DrFusion(_opts())
    for (bgr, depth), pose in zip(frames, poses):
        full.IntegrateScanAsync(bgr, depth, pose)
        full.RenderAsync([poses[0]])
        (fb,), (fd,) = full.GetRenderResult()
    cf, vf = full.dump_blocks()
    z0 = -3
    owner = lambda z: (np.floor_divide(z - z0, k)) % world
    owned_c, owned_v, keys = [], [], None
    for r in range(world):
        rend = {}
        for clip in (1, 0):
            f = DrFusion(_opts())
            f.set_interleave(r, world, k, z0)
            f.set_option("slab_clip", clip)
            for (bgr, depth), pose in zip(frames, poses):
                f.IntegrateScanAsync(bgr, depth, pose)
                f.RenderAsync([poses[0]])
                (rb,), (rd,) = f.GetRenderResult()
            rend[clip] = (rd.copy(), rb.copy())
        assert np.array_equal(rend[1][0], rend[0][0]) and np.array_equal(rend[1][1], rend[0][1]), "clipped march differs from the unclipped one"
        c, v = f.dump_blocks()
        stored = (owner(c[:, 2]) == r) | (owner(c[:, 2] - 1) == r) | (owner(c[:, 2] + 1) == r)
        assert stored.all(), "a rank stores a block row that is neither its own nor a halo"
        own = owner(c[:, 2]) == r
        owned_c.append(c[own]); owned_v.append(v[own])
        kk = pack_hits(*rend[1])
        keys = kk if keys is None else np.minimum(keys, kk)
    cu, vu = np.concatenate(owned_c), np.concatenate(owned_v)
    order = np.lexsort((cu[:, 2], cu[:, 1], cu[:, 0]))
    assert np.array_equal(cu[order], cf), "union of owned blocks != single volume block set"
    assert np.array_equal(vu[order]["weight"], vf["weight"]) and np.array_equal(vu[order]["sdf"], vf["sdf"])
    assert np.array_equal(vu[order]["color"], vf["color"])
    dm, bm = unpack_hits(keys)
    hit_m, hit_f = dm > 0, fd > 0
    assert np.mean(hit_m != hit_f) < 5e-3
    both = hit_m & hit_f
    err = np.abs(dm[both] - fd[both])
    print(f"interleave world={world} k={k}: hit mismatch {np.mean(hit_m != hit_f):.5f}, depth err median {np.median(err):.2e} p99 {np.quantile(err, 0.99):.2e}, bit-equal {np.mean(dm == fd):.4f}")
    assert np.median(err) < 1e-3 and np.quantile(err, 0.99) < 0.02


# ---------------------------------------------------------------------------------------------------------------------
# marching cubes (SURVEY.md 8f n4): DrFusion::ExtractMeshAsync / GetMeshSync / GetMesh vs the brute-force oracle
def _sorted_tris(vert, cols):
    """Triangle order is unspecified (the reference appends with atomicAdd): compare lexicographically sorted rows."""
    t = np.concatenate([vert.reshape(-1, 9), cols.reshape(-1, 9)], axis=1)
    return t[np.lexsort(t.T[::-1])]


def _mesh_pair(n_frames=3, **kw):
    poses, frames = _scene_frames(n_frames)
    f, o = DrFusion(_opts(**kw)), TsdfOracle(_opts(**kw))
    for (bgr, depth), pose in zip(frames, poses):
        f.IntegrateScanAsync(bgr, depth, pose)
        o.integrate(bgr, depth, pose)
        f.RenderAsync([pose])
        f.GetRenderResult()
    return f, o


@pytest.mark.parametrize("lower,upper", [
    ((-1.28, -1.28, -1.28), (1.28, 1.28, 1.28)),          # voxel-aligned box, negative and positive coordinates
    ((-1.2345, -0.777, -1.1111), (1.3, 0.9137, 1.2501)),  # arbitrary corners: per-axis rounding is whatever fp32 says
    ((0.105, -0.4, -0.3), (1.3, 0.4, 0.7)),               # sub-boxes that cut through blocks
    ((-0.9, -0.6, 0.3), (0.3, 0.5, 1.25)),
])
def test_mesh_matches_oracle_bit_exact(lower, upper):
    f, o = _mesh_pair()
    lo, up = np.float32(lower), np.float32(upper)
    vo, co = o.extract_mesh(lo, up)
    f.ExtractMeshAsync(lo, up)
    vg, cg = f.GetMeshSync()
    print(f"mesh {lower}..{upper}: {len(vg) // 3} triangles (oracle {len(vo) // 3}), device {f.last_mesh_ms():.3f} ms")
    assert len(vo) > 3000, "scene produced no surface - test is vacuous"
    assert len(vg) == len(vo), f"vertex count {len(vg)} vs oracle {len(vo)}"
    assert np.array_equal(_sorted_tris(vg, cg), _sorted_tris(vo, co)), "triangle sets differ"
    # blocking variant (TsdfVolume::ExtractMesh, no call-order requirement) gives the same set
    v2, c2 = f.GetMesh(lo, up)
    assert np.array_equal(_sorted_tris(v2, c2), _sorted_tris(vo, co))


def test_mesh_call_order_capacity_and_regrow(monkeypatch):
    monkeypatch.setenv("TDM_MESH_INIT_TRIS", "64")      # force the grow-and-re-emit path of GetMeshSync
    f, o = _mesh_pair(2)
    lo, up = np.float32([-1.28] * 3), np.float32([1.28] * 3)
    with pytest.raises(Exception):
        f.GetMeshSync()                                  # GetMeshSync without ExtractMeshAsync (tsdf_volume.cu:787-790)
    f.ExtractMeshAsync(lo, up)
    with pytest.raises(Exception):
        f.ExtractMeshAsync(lo, up)                       # twice in a row (tsdf_volume.cu:769-772)
    vg, cg = f.GetMeshSync()
    vo, co = o.extract_mesh(lo, up)
    assert len(vg) == len(vo) > 64 * 3
    assert np.array_equal(_sorted_tris(vg, cg), _sorted_tris(vo, co))
    # only legal where IntegrateScanAsync is legal (tsdf_volume.cu:760-763)
    poses, frames = _scene_frames(1)
    f.IntegrateScanAsync(frames[0][0], frames[0][1], poses[0])
    with pytest.raises(Exception):
        f.ExtractMeshAsync(lo, up)
    f.RenderAsync([poses[0]]); f.GetRenderResult()
    f.ExtractMeshAsync(lo, up)
    import ctypes
    from tandem_b200._lib import lib
    fp = ctypes.POINTER(ctypes.c_float)
    small = np.empty((30, 3), np.float32)
    rc = lib().tdm_fusion_get_mesh(f._h, small.ctypes.data_as(fp), small.ctypes.data_as(fp), 30)
    assert rc < 0 and b"enough storage" in lib().tdm_last_error()   # tsdf_volume.cu:796-799
    # empty boxes
    assert len(f.GetMesh(np.float32([5, 5, 5]), np.float32([5.5, 5.5, 5.5]))[0]) == 0
    assert len(f.GetMesh(lo, np.float32([lo[0], 1, 1]))[0]) == 0


def test_mesh_state_machine_stale_and_blocking_paths(monkeypatch):
    """Advisor r01: (1) scans integrated between ExtractMeshAsync and a GetMeshSync that has to grow its buffers must not be
    classified against stale per-block offsets - the whole extraction is redone on the current volume; (2) the blocking
    ExtractMesh path (GetMesh / SaveMeshToFile) never consumes an ExtractMeshAsync result and never re-uses a count-only
    query for a different box or a changed volume."""
    monkeypatch.setenv("TDM_MESH_INIT_TRIS", "64")
    f, o = _mesh_pair(1)
    lo, up = np.float32([-1.28] * 3), np.float32([1.28] * 3)
    poses, frames = _scene_frames(3)
    f.ExtractMeshAsync(lo, up)
    for k in (1, 2):                                     # a full Integrate -> Render -> GetRenderResult cycle is legal here
        f.IntegrateScanAsync(frames[k][0], frames[k][1], poses[k]); o.integrate(frames[k][0], frames[k][1], poses[k])
        f.RenderAsync([poses[k]]); f.GetRenderResult()
    vg, cg = f.GetMeshSync()                             # count-only query inside, then the grow path: re-extracted
    vo, co = o.extract_mesh(lo, up)
    assert len(vg) == len(vo) > 64 * 3
    assert np.array_equal(_sorted_tris(vg, cg), _sorted_tris(vo, co))
    # blocking path while an asynchronous result is pending: rejected, and the pending result survives
    f.ExtractMeshAsync(lo, up)
    with pytest.raises(Exception):
        f.GetMesh(lo, up)
    v2, c2 = f.GetMeshSync()
    assert np.array_equal(_sorted_tris(v2, c2), _sorted_tris(vo, co))
    # a count-only query of one box followed by a copy call for another box: the second box is what comes back
    import ctypes
    from tandem_b200._lib import lib
    fp = ctypes.POINTER(ctypes.c_float)
    n_full = lib().tdm_fusion_extract_mesh(f._h, lo.ctypes.data_as(fp), up.ctypes.data_as(fp), None, None, 0)
    up2 = np.float32([0.0, 1.28, 1.28])
    vh, ch = f.GetMesh(lo, up2)
    voh, coh = o.extract_mesh(lo, up2)
    assert 0 < len(vh) == len(voh) < n_full
    assert np.array_equal(_sorted_tris(vh, ch), _sorted_tris(voh, coh))


def test_mesh_full_size_properties():
    """640x480 scan into the initDr-sized map, the 10 m box of tandem_backend.cpp:80-81: every vertex lies within a voxel and
    a half of the analytic surface it was fused from; the same call twice gives the same triangle set."""
    scene = RoomScene()
    f = DrFusion(DrFusionOptions())
    for eye in ((0.3, 0.0, -0.2), (0.35, 0.02, -0.15)):
        pose = look_at_pose(eye, (2.5, 0.2, 0.5))
        bgr, depth = scene.render(pose, 480, 640, 320.0, 320.0, 319.5, 239.5)
        f.IntegrateScanAsync(bgr, depth, pose)
        f.RenderAsync([pose]); f.GetRenderResult()
    lo, up = np.float32([-5, -5, -5]), np.float32([5, 5, 5])
    f.ExtractMeshAsync(lo, up)
    v1, c1 = f.GetMeshSync()
    ms = f.last_mesh_ms()
    v2, c2 = f.GetMesh(lo, up)
    print(f"full-size mesh: {len(v1) // 3} triangles from {f.stats()['allocated_blocks']} blocks in {ms:.3f} ms (device)")
    assert len(v1) > 100000 and len(v1) % 3 == 0
    assert np.array_equal(_sorted_tris(v1, c1), _sorted_tris(v2, c2))
    d_walls = np.min(np.abs(np.abs(v1) - scene.half), axis=1)
    d_sph = np.min([np.abs(np.linalg.norm(v1 - np.float32(s[:3]), axis=1) - s[3]) for s in scene.spheres], axis=0)
    assert np.quantile(np.minimum(d_walls, d_sph), 0.995) < 0.015
    assert (c1 >= 0).all() and (c1 <= 1).all()


def test_nearest_hit_keys_roundtrip_on_device():
    """The slab exchange buffers (SURVEY.md 8e): packing a render into int64 keys on the device and unpacking them again is
    the identity, and the device keys equal the host-side packing used by the gloo test (tandem_b200.parallel.pack_hits)."""
    import torch
    from tandem_b200.parallel import _DeviceInt64, pack_hits, reduce_nearest_hit_device
    poses, frames = _scene_frames(2)
    f = DrFusion(_opts())
    for (bgr, depth), pose in zip(frames, poses):
        f.IntegrateScanAsync(bgr, depth, pose)
        f.RenderAsync([poses[0]])
        (rb,), (rd,) = f.GetRenderResult()
    ptr, n = f.render_keys_device(0)
    keys = torch.as_tensor(_DeviceInt64(ptr, n), device="cuda:0").cpu().numpy().reshape(H, W)
    assert np.array_equal(keys, pack_hits(rd, rb))
    dm, bm = reduce_nearest_hit_device(None, f, 0)
    assert np.array_equal(dm, rd) and np.array_equal(bm[rd > 0], rb[rd > 0]) and (rd == 0).any() and (rd > 0).any()
