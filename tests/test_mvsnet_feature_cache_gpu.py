"""The MVSNet feature cache (tdm_mvsnet_call_async_ids, DrMvsnet.CallAsyncIds): a window submitted by keyframe ids, with
FeatureNet run only for the ids the handle does not hold, must give exactly what tdm_mvsnet_call_async gives for the same
images - the four stage-3 maps, the stage-1/2 outputs and feat1..feat3, bit for bit (NaN-aware) in every precision.
FeatureNet works on each view alone and the tile planners keep each output's fold order whatever the plane count, so
identity is the bar, not a tolerance."""
import os
import subprocess

import numpy as np
import pytest

from tandem_b200 import DrMvsnet, TandemError, default_weights
from tandem_b200.fusion import DrFusion, DrFusionOptions
from tandem_b200.synthetic import RoomScene, circle_trajectory, mvs_plane_window

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WEIGHTS = default_weights("abl03_view_aggregation")
DMIN, DMAX, DISCARD = 0.5, 5.0, 2.5
MAPS = ("depth", "confidence", "depth_dense", "confidence_dense")
_frames_cache = {}


def frames(n, H, W):
    """n keyframes of a room seen from a slow circle (look-out), BGR u8 + cam_to_world, and the full-resolution K."""
    key = (n, H, W)
    if key not in _frames_cache:
        fx = fy = 0.5 * W
        cx, cy = (W - 1) / 2, (H - 1) / 2
        scene = RoomScene()
        poses = circle_trajectory(60, radius=0.4)[:n]
        bgrs = [np.ascontiguousarray(scene.render(p, H, W, fx, fy, cx, cy)[0]) for p in poses]
        K = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float32)
        _frames_cache[key] = (bgrs, [np.asarray(p, np.float32) for p in poses], K)
    return _frames_cache[key]


def collect(m, feats=True):
    """Everything the window produced: GetResult's maps, the stage-1/2 outputs and (optionally) feat1..feat3."""
    r = m.GetResult()
    out = {k: getattr(r, k).copy() for k in MAPS}
    for s in (1, 2):
        for w in ("depth_dense", "confidence_dense"):
            out[f"s{s}.{w}"] = m.stage_output(s, w)
    if feats:
        for f in ("feat1", "feat2", "feat3"):
            out[f] = m.debug_tensor(f)
    return out


def same(a, b, where=""):
    assert a.keys() == b.keys()
    for k in a:
        assert a[k].shape == b[k].shape and np.array_equal(a[k], b[k], equal_nan=True), f"{where}: {k} differs"


class Pair:
    """A cached handle and an uncached one fed the same windows (the uncached one through tdm_mvsnet_call_async, which
    recomputes every view: it is the result a fresh handle gives)."""

    def __init__(self, precision="mixed16", H=256, W=320, n=28):
        self.H, self.W = H, W
        self.bgrs, self.c2ws, self.K = frames(n, H, W)
        self.cached = DrMvsnet(WEIGHTS, precision=precision)
        self.plain = DrMvsnet(WEIGHTS, precision=precision)

    def expect(self, ids, ref):
        self.plain.CallAsync(self.H, self.W, len(ids), ref, [self.bgrs[i] for i in ids], self.K, [self.c2ws[i] for i in ids],
                             DMIN, DMAX, DISCARD)
        return collect(self.plain)

    def submit(self, ids, ref, images):
        """images: the ids whose image is passed; the others get None."""
        self.cached.CallAsyncIds(self.H, self.W, len(ids), ref, ids, [self.bgrs[i] if i in images else None for i in ids], self.K,
                                 [self.c2ws[i] for i in ids], DMIN, DMAX, DISCARD)

    def check(self, ids, ref, images, computed):
        self.submit(ids, ref, images)
        got = collect(self.cached)
        assert self.cached.feature_cache() == (list(ids), computed), (ids, self.cached.feature_cache())
        same(got, self.expect(ids, ref), f"window {ids} ref {ref}")
        return got


@pytest.mark.parametrize("size", [(480, 640), (256, 320)])
@pytest.mark.parametrize("precision", ["mixed16", "fp32", "bf16"])
def test_sliding_window_bit_identical(precision, size):
    """TANDEM's sliding window: 13 keyframes, window 7, reference at V-2; after the first window each call brings only
    the keyframe it adds (the held ids get None) and FeatureNet computes one view."""
    H, W = size
    p = Pair(precision, H, W, n=13)
    V = 7
    for k in range(13 - V + 1):
        ids = list(range(k, k + V))
        p.check(ids, V - 2, images=set(ids) if k == 0 else {k + V - 1}, computed=V if k == 0 else 1)
    # the resident entry re-runs that last window with its newest view recomputed, and the full forward: same maps
    before = p.cached.stage_output(3, "depth_dense")
    ms, launches = p.cached.run_resident_new(1, 3)
    assert ms > 0 and launches > 0
    assert np.array_equal(p.cached.stage_output(3, "depth_dense"), before, equal_nan=True)
    p.cached.run_resident(2)
    assert np.array_equal(p.cached.stage_output(3, "depth_dense"), before, equal_nan=True)


def test_intermediates_hold_the_computed_views():
    """After a cached call the FeatureNet intermediates hold the new views only, in window order; feat1..3 all of them."""
    p = Pair("mixed16")
    p.check(list(range(7)), 5, images=set(range(7)), computed=7)
    full = p.cached.debug_tensor("f.c1")
    assert full.shape[1] == 7
    p.check([1, 2, 3, 4, 5, 6, 7], 5, images={7}, computed=1)
    one = p.cached.debug_tensor("f.c1")
    assert one.shape[1] == 1
    p.plain.CallAsync(p.H, p.W, 7, 5, [p.bgrs[i] for i in range(1, 8)], p.K, [p.c2ws[i] for i in range(1, 8)], DMIN, DMAX, DISCARD)
    p.plain.GetResult()
    # f.c1 of the plain window's view 7 (window position 6, reference-first order: unchanged since 6 > ref)
    assert np.array_equal(one[:, 0], p.plain.debug_tensor("f.c1")[:, 6], equal_nan=True)


@pytest.mark.parametrize("precision", ["mixed16", "fp32"])
def test_window_changes(precision):
    """How DSO's window changes, each against the uncached result, with the computed-view count the cache reports."""
    p = Pair(precision)
    p.check([0, 1, 2, 3, 4, 5, 6], 5, images=set(range(7)), computed=7)
    p.check([0, 1, 2, 4, 5, 6, 7], 5, images={7}, computed=1)                     # a middle keyframe dropped
    p.check([2, 4, 5, 6, 7, 8, 9], 5, images={8, 9, 2}, computed=2)              # two dropped, two added (2's image ignored)
    p.check([9, 2, 7, 4, 5, 6, 8], 1, images=set(), computed=0)                  # same ids permuted, another reference
    p.check([20, 21, 22, 23, 24, 25, 26], 5, images=set(range(20, 27)), computed=7)   # all new
    with pytest.raises(TandemError, match="no image for view id 3"):
        p.submit([21, 22, 23, 24, 25, 26, 3], 5, images=set())                  # an evicted id returns without its image
    p.check([21, 22, 23, 24, 25, 26, 3], 5, images={3}, computed=1)              # ... and with it
    p.check([3, 4, 5, 6, 7], 3, images={3, 4, 5, 6, 7}, computed=5)              # V changes: every view is recomputed
    p.check([4, 5, 6, 7, 8], 3, images={8}, computed=1)


def test_golden_sample_through_the_cache():
    """The shipped 512x320 window with its per-stage K's: the cached path equals tdm_mvsnet_call_async_k, also when the
    second call passes no image at all and moves the reference."""
    g = np.load(os.path.join(ROOT, "tests", "golden", "sample_512x320.npz"))
    nv, gh, gw = g["bgr"].shape[:3]
    bgrs = [np.ascontiguousarray(g["bgr"][v]) for v in range(nv)]
    c2ws = [np.ascontiguousarray(g["c2w"][v]) for v in range(nv)]
    Ks = np.stack([g["K1"], g["K2"], g["K3"]]).astype(np.float32)
    w = default_weights("abl04_fewer_depth_planes")
    a, b = DrMvsnet(w, precision="mixed16"), DrMvsnet(w, precision="mixed16")
    args = (float(g["depth_min"]), float(g["depth_max"]), float(g["discard"]))
    ids = [100 + v for v in range(nv)]
    for ref, imgs in ((int(g["ref_index"]), bgrs), (1, [None] * nv)):
        a.CallAsyncIds(gh, gw, nv, ref, ids, imgs, Ks, c2ws, *args, stage_k=True)
        b.CallAsyncStageK(gh, gw, nv, ref, bgrs, Ks, c2ws, *args)
        same(collect(a), collect(b), f"golden ref {ref}")
    assert a.feature_cache() == (ids, 0)


def test_handoff_reads_the_reference_slot():
    """In cached windows the reference image was passed in an earlier call: tdm_fusion_integrate_mvsnet after GetResult
    still builds the volume the host path builds from that image, in TANDEM's order GetResult(k) -> CallAsync(k+1) ->
    integrate(k)."""
    H, W, V, n = 128, 160, 4, 9
    win = mvs_plane_window(V=n, H=H, W=W, seed=5)
    bgrs, c2ws, K = win["bgrs"], win["c2ws"], win["K"]
    m = DrMvsnet(WEIGHTS, precision="mixed16")
    opts = dict(height=H, width=W, fx=float(K[0, 0]), fy=float(K[1, 1]), cx=float(K[0, 2]), cy=float(K[1, 2]),
                num_buckets=100003, num_blocks=200000)
    host, dev = DrFusion(DrFusionOptions(**opts)), DrFusion(DrFusionOptions(**opts))
    ref = V - 2

    def call(k):
        ids = list(range(k, k + V))
        m.CallAsyncIds(H, W, V, ref, ids, [bgrs[i] if (k == 0 or i == k + V - 1) else None for i in ids], K,
                       c2ws[k:k + V], 0.5, 5.0, 2.5)

    call(0)
    for k in range(n - V + 1):
        r = m.GetResult()
        if k + 1 < n - V + 1:
            call(k + 1)
        host.IntegrateScanAsync(bgrs[k + ref], r.depth, c2ws[k + ref])
        dev.IntegrateScanFromMvsnet(m)
        ca, va = host.dump_blocks()
        cb, vb = dev.dump_blocks()
        assert len(ca) > 0 and np.array_equal(ca, cb) and va.tobytes() == vb.tobytes(), f"keyframe {k}"
        renders = []
        for f in (host, dev):                                    # the call order: integrate -> render -> get render
            f.RenderAsync([np.asarray(c2ws[k + ref], np.float32)])
            b, d = f.GetRenderResult()
            renders.append((b[0].tobytes(), d[0].tobytes()))
        assert renders[0] == renders[1], f"keyframe {k}"


def test_plain_call_empties_the_cache():
    """A plain CallAsync after cached calls gives what it gives today and empties the cache; the next cached call then
    needs every image."""
    p = Pair("mixed16")
    p.check(list(range(7)), 5, images=set(range(7)), computed=7)
    p.check(list(range(1, 8)), 5, images={7}, computed=1)
    ids = list(range(2, 9))
    p.cached.CallAsync(p.H, p.W, 7, 5, [p.bgrs[i] for i in ids], p.K, [p.c2ws[i] for i in ids], DMIN, DMAX, DISCARD)
    same(collect(p.cached), p.expect(ids, 5), "plain call")
    assert p.cached.feature_cache() == ([], 7)
    with pytest.raises(TandemError, match="no image for view id"):
        p.submit(list(range(3, 10)), 5, images={9})
    p.check(list(range(3, 10)), 5, images=set(range(3, 10)), computed=7)
    # an option change empties it too
    p.cached.set_option("fork_fpn", 1)
    with pytest.raises(TandemError, match="no image for view id"):
        p.submit(list(range(4, 11)), 5, images={10})


def test_errors_change_nothing():
    """Each refused call leaves the pools and ids as they were: the next valid call returns what it returns without it."""
    p = Pair("mixed16")
    p.check(list(range(7)), 5, images=set(range(7)), computed=7)
    c = p.cached
    bad = [
        (dict(ids=[1, 2, 3, 4, 5, 6, 7], images=set()), "no image for view id 7"),
        (dict(ids=[1, 2, 3, 4, 5, 6, 6], images={6}), "passed for two views"),
    ]
    for kw, msg in bad:
        with pytest.raises(TandemError, match=msg):
            p.submit(kw["ids"], 5, kw["images"])
        assert c.feature_cache() == (list(range(7)), 7)
    ids = list(range(1, 8))
    poses = [p.c2ws[i] for i in ids]
    for H, W, ref, msg in ((240, 320, 5, "multiples of 32"), (p.H, p.W, 7, "ref_index")):   # bad size, bad ref_index
        with pytest.raises(TandemError, match=msg):
            c.CallAsyncIds(H, W, 7, ref, ids, [None] * 7, p.K, poses, DMIN, DMAX, DISCARD)
        assert c.feature_cache() == (list(range(7)), 7)
    c.set_option("eager_d2h", 1)                                 # not a cache-emptying option
    p.check(ids, 5, images={7}, computed=1)
    c.set_option("filter_all_stages", 0)                         # any other option empties the cache, even at its current value
    p.check(list(range(2, 9)), 5, images=set(range(2, 9)), computed=7)


def test_two_handles_interleaved():
    """Two handles on one device, each with its own sliding sequence (another size, precision and reference), submitted
    before either result is fetched: each equals its solo uncached run."""
    a = Pair("mixed16", 256, 320, n=12)
    b = Pair("bf16", 480, 640, n=12)
    for k in range(5):
        ia, ib = list(range(k, k + 7)), list(range(k, k + 6))
        a.submit(ia, 5, set(ia) if k == 0 else {k + 6})
        b.submit(ib, 2, set(ib) if k == 0 else {k + 5})
        gb = collect(b.cached)                                   # fetched in the other order
        ga = collect(a.cached)
        same(ga, a.expect(ia, 5), f"handle a window {k}")
        same(gb, b.expect(ib, 2), f"handle b window {k}")
        assert a.cached.feature_cache()[1] == (7 if k == 0 else 1) and b.cached.feature_cache()[1] == (6 if k == 0 else 1)


def test_shim_overload(tmp_path):
    """tests/cpp/shim_feature_cache drives DrMvsnet::CallAsync(..., std::vector<long long> const& view_ids, ...) through a
    sliding sequence, passing only the image each window adds: every window's maps equal the uncached result."""
    H, W, V, n = 256, 320, 7, 10
    bgrs, c2ws, K = frames(n, H, W)
    src = tmp_path / "frames.bin"
    with open(src, "wb") as f:
        f.write(b"TDMK0001")
        f.write(np.array([n, V, H, W], np.int32).tobytes())
        f.write(K.astype(np.float32).tobytes())
        f.write(np.array([DMIN, DMAX, DISCARD], np.float32).tobytes())
        for i in range(n):
            f.write(c2ws[i].astype(np.float32).tobytes())
            f.write(bgrs[i].tobytes())
    dst = tmp_path / "maps.bin"
    env = dict(os.environ, TDM_PRECISION="mixed16")
    r = subprocess.run([os.path.join(ROOT, "tests", "cpp", "shim_feature_cache"), WEIGHTS, str(src), str(dst)],
                       capture_output=True, text=True, env=env, timeout=600)
    assert r.returncode == 0, r.stdout + r.stderr
    got = np.fromfile(dst, np.float32).reshape(n - V + 1, 4, H, W)
    m = DrMvsnet(WEIGHTS, precision="mixed16")
    for k in range(n - V + 1):
        m.CallAsync(H, W, V, V - 2, bgrs[k:k + V], K, c2ws[k:k + V], DMIN, DMAX, DISCARD)
        o = m.GetResult()
        for j, name in enumerate(MAPS):
            assert np.array_equal(got[k, j], getattr(o, name), equal_nan=True), (k, name)
