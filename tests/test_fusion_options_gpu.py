"""The TSDF engine against its CPU oracle (oracle/tsdf_oracle.c) across the options it accepts: voxel size, truncation,
image size, fx != fy, integer and half-pixel principal points, sensor range, weight ceiling and hash geometry (the cases of
oracle/fusion_options.py).  Four scans per case whose views overlap (30 degrees apart, then the first pose again), so most
observed voxels are averaged over two or three scans; world shifted by a non-block offset.

Bars, and why each is what it is:
- block set, block count (allocated / visible / dropped == 0), per-voxel weight and colour: EXACT.  They are integer
  decisions (DDA steps, pixel projections, u8 averages) the kernels take with the oracle's own fp32 expressions.
- sdf: bit-exact, with K6's running mean in play: after the second scan hundreds of thousands of voxels per case have weight
  2 to 4 (asserted, with range_w1 held at weight 1 and range_w255 going past it).  test_fusion_gpu.py allows 1e-5
  (2.5e-4 * tau) on 1e-4 of the voxels, but no voxel of any case here differs, nor in test_fusion_gpu.py's own runs (both
  print 1.000000): K6 evaluates the oracle's expressions in the same order without contraction, each voxel is updated by
  one thread once per scan, and the scans are integrated in the same order.  The bit-exact fraction is printed per scan.
- renders against the oracle, from the scan's pose, the previous scan's pose, outside looking in and two axis-aligned poses
  (identity rotation, 90 degrees about y: with an integer principal point whole pixel rows / columns are exactly parallel
  to axis planes, the parallel-ray branch of the ray-cast's bounding-box clip): hit mismatch <= 1e-3, depth and colour
  bit-equal on >= 0.999 of the pixels (test_fusion_gpu.py's bar; the oracle evaluates the march's expressions on the host,
  where sqrt, floor and the float-to-int conversions are the C library's).
- the production ray-cast, with fast_div 0 and 1, against the reference-shaped comparator (raycast_shared=0): bit for bit on
  every render, since both put every sample where the reference's march puts it.
- the mesh against TsdfOracle.extract_mesh: bit-exact as sorted triangle sets, in a voxel-aligned box and in one that cuts
  blocks.
- slab clipping of an interleaved Z-slab partition (its slack is in voxel units): bit-identical to the unclipped march.
- at two cases, the device and the oracle against the reference's own DrFusion (tests/golden/reference_pins_fusion_options.npz,
  made by oracle/gen_reference_pins_fusion_options.py) with the bars of test_reference_gpu.py in voxel units."""
import os

import numpy as np
import pytest

from oracle import fusion_options as FO
from oracle.cpu import TsdfOracle
from tandem_b200 import DrFusion, DrFusionOptions
from tandem_b200._lib import lib

pytestmark = pytest.mark.gpu

VIEW_NAMES = ("scan", "previous", "outside", "axis_identity", "axis_rot90")
VARIANTS = (("comparator", {"raycast_shared": 0}), ("fast_div", {"fast_div": 1}))


def _compare_maps(f, o, ctx):
    cg, vg = f.dump_blocks()
    co, vo = o.dump_blocks()
    assert cg.shape == co.shape, (ctx, f"block count {cg.shape[0]} vs oracle {co.shape[0]}")
    assert np.array_equal(cg, co), (ctx, "allocated block coordinate sets differ")
    assert np.array_equal(vg["weight"], vo["weight"]), (ctx, "voxel weights differ")
    assert np.array_equal(vg["color"], vo["color"]), (ctx, "voxel colours differ")
    same = vg["sdf"].view(np.uint32) == vo["sdf"].view(np.uint32)
    exact = float(np.mean(same))
    if not same.all():
        d = np.abs(vg["sdf"] - vo["sdf"])[~same]
        print(ctx, f"sdf differs on {int((~same).sum())} voxels: weights {np.bincount(vg['weight'][~same])}, "
                   f"|err| max {d.max():.3e} median {np.median(d):.3e}")
    assert exact == 1.0, (ctx, exact)
    return cg.shape[0], exact, vg["weight"]


def _render_bars(rd, rb, od, ob, ctx):
    hit_g, hit_o = rd > 0, od > 0
    mism = float(np.mean(hit_g != hit_o))
    assert mism <= 1e-3, (ctx, mism)
    assert np.mean(rd.view(np.uint32) == od.view(np.uint32)) >= 0.999, (ctx, float(np.mean(rd == od)))
    assert np.mean(rb == ob) >= 0.999, (ctx, float(np.mean(rb == ob)))
    return float(hit_g.mean())


def _bit_equal(a, b):
    return np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32)) and np.array_equal(a[1], b[1])


@pytest.mark.parametrize("name", list(FO.CASES))
def test_option_case_matches_oracle(name):
    opt = FO.options(name, num_render_streams=len(VIEW_NAMES))
    assert lib().tdm_debug_fast_div_eligible(opt.voxel_size, opt.fx, opt.fy) == 1   # fast_div really runs below
    f = DrFusion(opt)
    others = []
    for _, kv in VARIANTS:
        g = DrFusion(opt)
        for k, v in kv.items():
            g.set_option(k, v)
        others.append(g)
    o = TsdfOracle(opt)
    scans = FO.scans(name)
    extra = FO.views()
    exact = []
    for k, (bgr, depth, pose) in enumerate(scans):
        views = [pose, scans[max(k - 1, 0)][2], extra["outside"], extra["axis_identity"], extra["axis_rot90"]]
        o.integrate(bgr, depth, pose)
        renders = []
        for g in [f] + others:
            g.IntegrateScanAsync(bgr, depth, pose)
            g.RenderAsync(views)
            rb, rd = g.GetRenderResult()
            renders.append([(d.copy(), b.copy()) for d, b in zip(rd, rb)])
        for (label, _), r in zip(VARIANTS, renders[1:]):
            for vn, a, b in zip(VIEW_NAMES, renders[0], r):
                assert _bit_equal(a, b), (name, k, vn, label, "production ray-cast differs from the comparator")
        sg, so = f.stats(), o.stats()
        assert sg["allocated_blocks"] == so["allocated_blocks"], (name, k, sg, so)
        assert sg["visible_blocks"] == so["visible_blocks"], (name, k, sg, so)
        assert sg["dropped_blocks"] == so["dropped_blocks"] == 0, (name, k, sg, so)
        nblk, ex, w = _compare_maps(f, o, (name, k))
        exact.append(ex)
        averaged = int((w > 1).sum())
        # the oracle's ray-cast dominates the run time: the scan's and the previous pose after every scan, all views after the last
        for j in (range(len(VIEW_NAMES)) if k == len(scans) - 1 else (0, 1)):
            ob, od = o.render(views[j])
            cover = _render_bars(*renders[0][j], od, ob, (name, k, VIEW_NAMES[j]))
            if j == 0:
                assert cover > 0.5, (name, k, cover)
        print(f"{name} scan {k}: {nblk} blocks, {averaged} voxels averaged (weight > 1), max weight {int(w.max())}, "
              f"sdf bit-exact fraction {ex:.6f}")
    # the scans overlap: K6's running mean ran on many voxels, and the weight stops at the ceiling
    assert averaged > 1000 if opt.max_sdf_weight > 1 else averaged == 0, (name, averaged)
    assert int(w.max()) == 1 if opt.max_sdf_weight == 1 else int(w.max()) > 1, (name, int(w.max()))
    for lo, up in FO.mesh_boxes(name):
        vo, co = o.extract_mesh(lo, up)
        f.ExtractMeshAsync(lo, up)
        vg, cg = f.GetMeshSync()
        print(f"{name} mesh {lo}..{up}: {len(vg) // 3} triangles (oracle {len(vo) // 3})")
        assert len(vo) >= 150, (name, lo, up, "box holds almost no surface - the comparison is vacuous")
        assert len(vg) == len(vo) and np.array_equal(_sorted_tris(vg, cg), _sorted_tris(vo, co)), (name, lo, up)


def _sorted_tris(vert, cols):
    t = np.concatenate([vert.reshape(-1, 9), cols.reshape(-1, 9)], axis=1)
    return t[np.lexsort(t.T[::-1])]


@pytest.mark.parametrize("name", ["ref_example", "fine"])
def test_slab_clip_is_bit_identical(name):
    """The interleaved partition's ray-cast skips samples whose +-2.5-voxel reach holds no block row of this rank; that slack
    is written in voxel units, so it is checked at a coarse and a fine voxel."""
    opt = FO.options(name, num_render_streams=len(VIEW_NAMES))
    scans, extra = FO.scans(name), FO.views()
    for rank in range(2):
        rend = {}
        for clip in (1, 0):
            f = DrFusion(opt)
            f.set_interleave(rank, 2, 1, -3)
            f.set_option("slab_clip", clip)
            out = []
            for k, (bgr, depth, pose) in enumerate(scans):
                f.IntegrateScanAsync(bgr, depth, pose)
                f.RenderAsync([pose, scans[max(k - 1, 0)][2], extra["outside"], extra["axis_identity"], extra["axis_rot90"]])
                rb, rd = f.GetRenderResult()
                out += [(d.copy(), b.copy()) for d, b in zip(rd, rb)]
            rend[clip] = out
        assert any((d > 0).any() for d, _ in rend[1]), (name, rank, "the slab rendered nothing - the test is vacuous")
        for j, (a, b) in enumerate(zip(rend[1], rend[0])):
            assert _bit_equal(a, b), (name, rank, j)


def test_non_finite_depth_is_ignored():
    """NaN and +-inf depth pixels contribute nothing: K5 and K6 (and the oracle) reject a depth outside
    [min_sensor_depth, max_sensor_depth] in a form NaN fails, so the map equals that of the same scan with those pixels at 0.
    Device and oracle agree on the block set, every voxel and the render.  (Before the fix the device's DDA spun to its
    100000-step guard on every NaN pixel; the count here is kept small so that it would still end.)"""
    name = "hash_pow2"
    opt = FO.options(name)
    (bgr, depth, pose), (bgr2, depth2, pose2) = FO.scans(name)[:2]
    rng = np.random.default_rng(7)
    idx = rng.choice(depth.size, 72, replace=False)
    bad = depth.copy().reshape(-1)
    bad[idx[:40]] = np.nan
    bad[idx[40:56]] = np.inf
    bad[idx[56:]] = -np.inf
    bad = bad.reshape(depth.shape)
    zero = np.where(np.isfinite(bad), bad, np.float32(0))
    f, fz, o = DrFusion(opt), DrFusion(opt), TsdfOracle(opt)
    for g, d in ((f, bad), (fz, zero)):
        g.IntegrateScanAsync(bgr, d, pose)
        g.RenderAsync([pose])
        g.GetRenderResult()
        g.IntegrateScanAsync(bgr2, depth2, pose2)
        g.RenderAsync([pose])
    o.integrate(bgr, bad, pose)
    o.integrate(bgr2, depth2, pose2)
    (rb,), (rd,) = f.GetRenderResult()
    (zb,), (zd,) = fz.GetRenderResult()
    assert f.stats() == fz.stats() and f.stats()["dropped_blocks"] == 0
    cg, vg = f.dump_blocks()
    cz, vz = fz.dump_blocks()
    assert np.array_equal(cg, cz) and np.array_equal(vg.view(np.uint64), vz.view(np.uint64)), "NaN / inf pixels changed the map"
    assert _bit_equal((rd, rb), (zd, zb))
    assert (_compare_maps(f, o, "non-finite")[2] > 1).any()
    ob, od = o.render(pose)
    _render_bars(rd, rb, od, ob, "non-finite")


def test_excluded_divisor_leaves_fast_div_off():
    """fx with an all-ones significand (0x1.fffffep+6): the constant-divisor sequence is not correctly rounded for it, so the
    host keeps the IEEE division and the option fast_div changes nothing."""
    fx = float.fromhex("0x1.fffffep+6")
    assert np.float32(fx).view(np.uint32) & 0x7FFFFF == 0x7FFFFF
    assert lib().tdm_debug_fast_div_eligible(0.01, fx, 80.0) == 0
    opt = DrFusionOptions(height=120, width=160, fx=fx, fy=80.0, cx=79.5, cy=59.5, num_buckets=200003, num_blocks=120000)
    scans = [(b, d, p) for b, d, p in FO.scans("hash_pow2")]
    out = []
    for fast in (0, 1):
        f = DrFusion(opt)
        f.set_option("fast_div", fast)
        for bgr, depth, pose in scans:
            f.IntegrateScanAsync(bgr, depth, pose)
            f.RenderAsync([scans[0][2]])
            (rb,), (rd,) = f.GetRenderResult()
        out.append((rd.copy(), rb.copy()))
    assert (out[0][0] > 0).mean() > 0.5
    assert _bit_equal(out[0], out[1])


@pytest.fixture(scope="module")
def ref_pins():
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_pins_fusion_options.npz"))


def _unobserved(opt, depth, q, scan_poses):
    """Pixels of a render from pose q whose surface point (at `depth`) lies outside the view cone of every scan: no scan's
    ray reached it, so no integration can have put a weighted voxel there."""
    H, W = depth.shape
    v, u = np.mgrid[0:H, 0:W].astype(np.float64)
    pc = np.stack([(u - opt.cx) / opt.fx * depth, (v - opt.cy) / opt.fy * depth, depth.astype(np.float64)], -1)
    q = q.astype(np.float64)
    pw = pc @ q[:3, :3].T + q[:3, 3]
    seen = np.zeros((H, W), bool)
    for T in scan_poses:
        T = T.astype(np.float64)
        c = (pw - T[:3, 3]) @ T[:3, :3]                                    # world -> that scan's camera
        with np.errstate(divide="ignore", invalid="ignore"):
            x, y = opt.fx * c[..., 0] / c[..., 2] + opt.cx, opt.fy * c[..., 1] / c[..., 2] + opt.cy
        seen |= (c[..., 2] > 0) & (x > -1) & (x < W) & (y > -1) & (y < H) & (c[..., 2] <= opt.max_sensor_depth + opt.truncation_distance)
    return ~seen


@pytest.mark.parametrize("name", ["ref_example", "aniso_odd"])
def test_matches_reference_dr_fusion_at_options(ref_pins, name):
    """Device and oracle against the reference's own DrFusion at the reference's example options and at fx != fy with odd
    image sizes, four overlapping scans.  Bars of test_reference_gpu.py::test_fusion_matches_reference_dr_fusion, in voxels
    (hit mismatch <= 3e-3; depth mean-abs <= 0.03 voxel, 99th percentile <= half a voxel: 3e-4 and 5e-3 at its voxel of
    0.01): the reference is FMA-contracted and inverts the pose differently, so "the same surface to a small fraction of a
    voxel" is what can be asked.
    One kind of pixel is left out of the depth bars, and only that kind: the reference hits a surface, ours hits another
    one more than a voxel away, and the reference's surface point lies outside the view cone of every scan.  No scan
    observed that point, so the oracle and the device are right to hold nothing there; the reference holds weighted voxels
    it never integrated (its racy allocation and the integration of its free hash entries, SURVEY.md Appendix B, are the
    known ways).  At most 1e-3 of a render may be such pixels.  A different surface at a point some scan could see counts in
    the depth bars like any other pixel."""
    from oracle.gen_reference_pins_fusion_options import pin_inputs
    opt = FO.options(name)
    sc, rp = pin_inputs(name)
    poses = [p for _, _, p in sc]
    ours, orc = DrFusion(opt), TsdfOracle(opt)
    for k, ((bgr, depth, pose), q) in enumerate(zip(sc, rp)):
        ours.IntegrateScanAsync(bgr, depth, pose)
        orc.integrate(bgr, depth, pose)
        ours.RenderAsync([q])
        (ob,), (od,) = ours.GetRenderResult()
        cb, cd = orc.render(q)
        rd, rb = ref_pins[f"{name}_{k}_depth"], ref_pins[f"{name}_{k}_bgr"]
        assert (rd > 0).mean() > 0.2
        for who, xd, xb in (("cuda", od, ob), ("oracle", cd, cb)):
            hit_r, hit_x = rd > 0, xd > 0
            mism = float(np.mean(hit_r != hit_x))
            ghost = hit_r & hit_x & (np.abs(rd - xd) > opt.voxel_size) & _unobserved(opt, rd, q, poses)
            both = hit_r & hit_x & ~ghost
            err = np.abs(rd[both] - xd[both])
            print(f"{name} scan {k} {who} vs reference: hit mismatch {mism:.5f}, surface no scan saw {int(ghost.sum())} px, "
                  f"depth mean-abs {err.mean():.2e}, q99 {np.quantile(err, 0.99):.2e}, bit-equal {np.mean(rd == xd):.5f}")
            assert mism <= 3e-3, (name, k, who, mism)
            assert ghost.mean() <= 1e-3, (name, k, who, int(ghost.sum()))
            vs = opt.voxel_size                                             # 3e-4 and 5e-3 at voxel 0.01
            assert err.mean() <= 0.03 * vs and np.quantile(err, 0.99) <= 0.5 * vs, (name, k, who)
            assert np.mean(np.abs(rb[both].astype(int) - xb[both].astype(int)) <= 2) > 0.98, (name, k, who)
