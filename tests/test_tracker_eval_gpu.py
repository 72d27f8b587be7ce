"""The coarse tracker's evaluation kernel (k_tracker<MODE> in tandem_b200/csrc/tracker.cu) per point and per output entry
against the fp64 reference of oracle/tracker_eval.py, at the point counts, borders, thresholds and image values where it
could go wrong: u, v and nid bit-identical, the per-point fetch and residual within the bilinear bound, every count exact
and E, the flow statistics and all 64 + 8 entries of H and b each within its own a-priori bound - for calcRes, calcG,
calcResAndG, calcResBatch and the device LM loop's first evaluation (track with max_iterations = 0).  Also: what calcG
refers to after the calls that write no warped buffers, a refused setReferenceDense, and the dense reference at sizes whose
pixel count is not a multiple of 256.  Run with -s for the worst error / bound of each family."""
import numpy as np
import pytest

from oracle import tracker_eval as te
from oracle.cpu import FrontOracle
from tandem_b200 import CudaCoarseTracker
from tandem_b200.synthetic import RoomScene, look_at_pose, tracker_case

pytestmark = pytest.mark.gpu

WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nworst error / bound per family:")
    for k in sorted(WORST):
        print(f"  {k:24s} {WORST[k]:.3g}")


def _note(family, r, what=""):
    WORST[family] = max(WORST.get(family, 0.0), r)
    assert r <= 1, f"{family} {what}: error / bound = {r}"


@pytest.fixture(scope="module")
def scene640():
    """The 640x480 scene with its points in a fixed random order: every prefix samples the whole frame."""
    c = tracker_case()
    perm = np.random.default_rng(7).permutation(c["n"])
    for k in ("pc_u", "pc_v", "pc_idepth", "pc_color"):
        c[k] = np.ascontiguousarray(c[k][perm])
    return c


@pytest.fixture(scope="module")
def scene160():
    return tracker_case(H=120, W=160, fx=80.0, fy=80.0, cx=79.5, cy=59.5)


def _tracker(c, huber=9.0, n=None, n_max=0, ref_exposure=None, ref_aff=None):
    n = c["n"] if n is None else n
    t = CudaCoarseTracker(c["w"], c["h"], huber, 20.0)
    t.init(n_max)
    t.setK(c["w"], c["h"], c["fx"], c["fy"], c["cx"], c["cy"])
    t.setReference(n, c["pc_u"][:n], c["pc_v"][:n], c["pc_idepth"][:n], c["pc_color"][:n],
                   c["ref_exposure"] if ref_exposure is None else ref_exposure, c["ref_aff"] if ref_aff is None else ref_aff)
    t.setNew(c["dInew"])
    return t


def _check_points(ev, W, label):
    acc = W[6] != 0
    pr = ev.pr
    diff = acc != ev.accepted
    assert not (diff & ~ev.excused).any(), (label, np.nonzero(diff & ~ev.excused)[0][:10])
    assert not (acc & ~ev.finite).any(), label
    for k, name in ((0, "u"), (1, "v"), (4, "nid")):
        assert np.array_equal(W[k][acc], pr[name][acc]), (label, name)
    assert not W[:, ~acc].any(), (label, "points not accepted must be zero in every array")
    _note("point dx, dy", max(te.ratio(W[2][acc], ev.hit[acc, 1], ev.bil[acc, 1]),
                              te.ratio(W[3][acc], ev.hit[acc, 2], ev.bil[acc, 2])), label)
    _note("point res", te.ratio(W[5][acc], ev.res[acc], ev.res_b[acc]), label)
    h = np.float32(ev.P.huber)
    ar = np.abs(W[5][acc])
    with np.errstate(divide="ignore"):
        hw = np.where(ar < h, np.float32(1), h / ar).astype(np.float32)
    assert np.array_equal(W[6][acc], hw), (label, "hw must follow from res")


def _check_res(res, ev, mode, label, maxE_slack=0.0):
    assert res[1] == ev.res6[1], (label, mode, "numTermsInE", res[1], ev.res6[1])
    assert res[3] == 0
    _note(f"{mode} saturated ratio", te.ratio(res[5], ev.res6[5], ev.res6_b[5]), label)
    _note(f"{mode} E", te.ratio(res[0], ev.res6[0], ev.res6_b[0] + ev.nS * maxE_slack), label)
    _note(f"{mode} flow", max(te.ratio(res[2], ev.res6[2], ev.res6_b[2]), te.ratio(res[4], ev.res6[4], ev.res6_b[4])), label)


def _num_warped(res):
    """numTermsInWarped of a res6 (numTermsInE - numSaturated)."""
    if res[1] == 0:
        return 0
    return int(res[1]) - int(round(res[5] * res[1]))


def _evaluate(t, c, n, T, huber, cutoff, new_exposure, new_aff, ref_exposure, ref_aff, label):
    """Every mode on one tracker state, each against the fp64 reference."""
    P = te.Params(c["w"], c["h"], c["fx"], c["fy"], c["cx"], c["cy"], huber, T, cutoff, ref_exposure, new_exposure, ref_aff,
                  new_aff)
    ev = te.Eval(P, c["pc_u"][:n], c["pc_v"][:n], c["pc_idepth"][:n], c["pc_color"][:n], c["dInew"])
    color = c["pc_color"][:n]
    # mode 0
    r0 = t.calcRes(T, new_exposure, new_aff, cutoff)
    W = t.getWarped(n)
    _check_points(ev, W, label)
    _check_res(r0, ev, "calcRes", label)
    nw0 = int(np.count_nonzero(W[6]))
    assert nw0 == _num_warped(r0) and abs(nw0 - ev.nW) <= ev.n_excused, label
    # mode 1: over the device's own warped values
    H1, b1 = t.calcG(new_exposure, new_aff)
    acc, bound = te.g_sums(P, W, color, n)
    Hr, Hb, br, bb = te.pack_hb(acc, bound, nw0)
    _note("calcG H", te.ratio(H1, Hr, Hb), label)
    _note("calcG b", te.ratio(b1, br, bb), label)
    # mode 2: recomputes the fetch, so the bound carries the bilinear error twice (device vs fp64, fp64 vs the warped values)
    r2, H2, b2 = t.calcResAndG(T, new_exposure, new_aff, cutoff)
    _check_res(r2, ev, "calcResAndG", label)
    nw2 = _num_warped(r2)
    assert abs(nw2 - nw0) <= ev.n_excused, label
    pert = (2 * ev.bil[:, 1], 2 * ev.bil[:, 2], 2 * ev.res_b)
    acc2, bound2 = te.g_sums(P, W, color, n, pert=pert, extra=te.excused_g_bound(ev, pert))
    Hr2, Hb2, br2, bb2 = te.pack_hb(acc2, bound2, nw2)
    _note("calcResAndG H", te.ratio(H2, Hr2, Hb2), label)
    _note("calcResAndG b", te.ratio(b2, br2, bb2), label)
    # mode 3, one hypothesis: bit-equal to calcRes
    rb = t.calcResBatch(np.asarray(T)[None], new_exposure, np.asarray(new_aff)[None], cutoff)[0]
    assert np.array_equal(rb, r0, equal_nan=True), (label, rb, r0)
    # calcG still refers to the calcRes above
    H1b, b1b = t.calcG(new_exposure, new_aff)
    assert np.array_equal(H1b, H1, equal_nan=True) and np.array_equal(b1b, b1, equal_nan=True), label
    return ev, r0


def _track_check(t, c, n, T, huber, cutoff, new_exposure, aff, ref_exposure, ref_aff, label):
    """mode 4: track with max_iterations = 0 returns its initial evaluation, at the cutoff after any doubling."""
    r = t.track(T, aff, new_exposure, coarse_cutoff=cutoff, max_iterations=0)
    assert r["iterations"] == 0
    rep = 1.0
    while True:
        P = te.Params(c["w"], c["h"], c["fx"], c["fy"], c["cx"], c["cy"], huber, T, np.float32(cutoff) * np.float32(rep),
                      ref_exposure, new_exposure, ref_aff, aff)
        ev = te.Eval(P, c["pc_u"][:n], c["pc_v"][:n], c["pc_idepth"][:n], c["pc_color"][:n], c["dInew"])
        if ev.res6[5] > 0.6 and rep < 50:
            rep *= 2
            continue
        break
    assert r["cutoff_repeat"] == rep and r["evaluations"] == int(np.log2(rep)) + 1, (label, r["cutoff_repeat"], rep)
    h, cu = float(P.huber), float(P.cutoff)
    _check_res(r["res"], ev, "track", label, maxE_slack=4 * te.U * (2 * h * cu + h * h))   # maxEnergy computed on the device
    return r


@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 255, 256, 257, 67583, 67584, 67585, 135169])
def test_point_counts(scene640, n):
    """n around a warp, the flow-statistics stride, the grid stride (264 x 256 = 67584) and n == n_max."""
    c = scene640
    t = _tracker(c, n=n, n_max=n)
    lab = f"n={n}"
    ev, r0 = _evaluate(t, c, n, c["refToNew"], 9.0, c["cutoffTH"], c["new_exposure"], c["new_aff"], c["ref_exposure"],
                       c["ref_aff"], lab)
    if n == 0:
        assert np.isnan(r0[2]) and np.isnan(r0[4]) and np.isnan(r0[5])
        H, b = t.calcG(c["new_exposure"], c["new_aff"])
        assert np.isnan(H).all() and np.isnan(b).all()
    else:
        assert ev.nW > 0 or n < 31
    aff = np.array([c["ref_aff"][0], c["new_aff"][1]])
    _track_check(t, c, n, c["refToNew"], 9.0, c["cutoffTH"], c["new_exposure"], aff, c["ref_exposure"], c["ref_aff"], lab)
    if n == 67585:   # > 60 % saturated: the loop doubles the cutoff before it takes the evaluation
        r = _track_check(t, c, n, c["refToNew"], 9.0, 1.0, c["new_exposure"], aff, c["ref_exposure"], c["ref_aff"], lab + " cut 1")
        assert r["cutoff_repeat"] > 1
    print(f"{lab}: excused {ev.n_excused}")


@pytest.mark.parametrize("size", [(161, 121), (33, 25), (640, 480)])
@pytest.mark.parametrize("hc", [(9.0, 20.0), (0.5, 0.5), (4.0, 2.0), (1e-3, 1e4)])
def test_exact_scene(size, hc):
    """Borders, idepth signs, points behind / on the camera plane, NaN and inf in the image, |res| at huber and cutoff
    +- 1 ulp: every decision and (at integer positions) every fetch exact."""
    w, h = size
    huber, cutoff = hc
    c = te.exact_scene(w, h, huber, cutoff)
    c.update(ref_exposure=1.0, ref_aff=np.zeros(2))
    n = c["n"]
    t = _tracker(c, huber=huber)
    for translated in (False, True):
        T = te.exact_pose(translated)
        lab = f"exact {w}x{h} huber {huber} cutoff {cutoff} translated {translated}"
        ev, r0 = _evaluate(t, c, n, T, huber, cutoff, 1.0, np.zeros(2), 1.0, np.zeros(2), lab)
        assert ev.n_excused == 0, lab
        if not translated:
            assert ev.nS >= 40 and ev.nW > 0 and (~np.isfinite(ev.hit[ev.pr["inframe"], 0])).sum() >= 15
            if hc == (4.0, 2.0):
                assert ev.P.maxE == 0
        _track_check(t, c, n, T, huber, cutoff, 1.0, np.zeros(2), 1.0, np.zeros(2), lab)
    # exposures: a zero one on either side means none is applied (affa = 1), otherwise affa = new / ref
    for ref_e, new_e in ((0.0, 2.0), (2.0, 0.0), (2.0, 1.0)):
        t.setReference(n, c["pc_u"], c["pc_v"], c["pc_idepth"], c["pc_color"], ref_e, np.zeros(2))
        lab = f"exact {w}x{h} huber {huber} exposures {ref_e} -> {new_e}"
        ev, _ = _evaluate(t, c, n, te.exact_pose(False), huber, cutoff, new_e, np.zeros(2), ref_e, np.zeros(2), lab)
        assert ev.P.affa == (0.5 if new_e == 1.0 else 1.0)
        _track_check(t, c, n, te.exact_pose(False), huber, cutoff, new_e, np.zeros(2), ref_e, np.zeros(2), lab)


@pytest.mark.parametrize("n_hyp", [1, 63, 64])
def test_batch(scene160, n_hyp):
    c = scene160
    t = _tracker(c)
    rng = np.random.default_rng(n_hyp)
    poses, affs = [], []
    for k in range(n_hyp):
        T = np.array(c["refToNew"], np.float64)
        T[:3, 3] += rng.normal(0, 0.01, 3) * (k > 0)
        poses.append(T)
        affs.append(np.array(c["new_aff"]) + (k % 3) * np.array([0.01, 0.5]))
    if n_hyp > 1:
        poses[-1] = poses[-1].copy()
        poses[-1][0, 3] = 1e3                         # this hypothesis sees no point
    batch = t.calcResBatch(np.stack(poses), c["new_exposure"], np.stack(affs), c["cutoffTH"])
    for k in range(n_hyp):
        r = t.calcRes(poses[k], c["new_exposure"], affs[k], c["cutoffTH"])
        assert np.array_equal(batch[k], r, equal_nan=True), k
        P = te.Params(c["w"], c["h"], c["fx"], c["fy"], c["cx"], c["cy"], 9.0, poses[k], c["cutoffTH"], c["ref_exposure"],
                      c["new_exposure"], c["ref_aff"], affs[k])
        ev = te.Eval(P, c["pc_u"], c["pc_v"], c["pc_idepth"], c["pc_color"], c["dInew"])
        _check_res(batch[k], ev, "calcResBatch", f"hypothesis {k} of {n_hyp}")
    if n_hyp > 1:
        assert batch[-1][1] == 0 and np.isnan(batch[-1][5])
    with pytest.raises(Exception):
        t.calcResBatch(np.stack([c["refToNew"]] * 65), c["new_exposure"], np.stack([c["new_aff"]] * 65), c["cutoffTH"])


@pytest.mark.parametrize("call", ["calcResAndG", "track", "calcResBatch"])
def test_calc_g_refers_to_the_last_calc_res(scene160, call):
    """calcResAndG, track and calcResBatch write no warped buffers: calcG after them equals calcG right after calcRes."""
    c = scene160
    t = _tracker(c)
    A = np.array(c["refToNew"])
    B = A.copy()
    B[:3, 3] += 0.02
    rB = t.calcRes(B, c["new_exposure"], c["new_aff"], c["cutoffTH"])
    rA = t.calcRes(A, c["new_exposure"], c["new_aff"], c["cutoffTH"])
    assert _num_warped(rA) != _num_warped(rB), "the two poses must warp different point counts"
    H0, b0 = t.calcG(c["new_exposure"], c["new_aff"])
    if call == "calcResAndG":
        t.calcResAndG(B, c["new_exposure"], c["new_aff"], c["cutoffTH"])
    elif call == "track":
        t.track(B, c["new_aff"], c["new_exposure"], max_iterations=3)
    else:
        t.calcResBatch(B[None], c["new_exposure"], np.asarray(c["new_aff"])[None], c["cutoffTH"])
    H, b = t.calcG(c["new_exposure"], c["new_aff"])
    assert np.array_equal(H, H0) and np.array_equal(b, b0), f"calcG after {call}"
    if call == "calcResAndG":
        fresh = _tracker(c)
        fresh.calcResAndG(A, c["new_exposure"], c["new_aff"], c["cutoffTH"])
        with pytest.raises(Exception):
            fresh.calcG(c["new_exposure"], c["new_aff"])


def _dense_case(h, w):
    f = 160.0 * w / 320.0
    K4 = (f, f, float((w - 1) // 2), float((h - 1) // 2))
    scene = RoomScene()
    pose_d = look_at_pose((0.3, 0.0, -0.2), (2.5, 0.2, 0.5))
    pose_r = look_at_pose((0.34, 0.02, -0.17), (2.5, 0.25, 0.45))
    _, depth = scene.render(pose_d, h, w, *K4, dropout=0.02, seed=1)
    bgr_r, _ = scene.render(pose_r, h, w, *K4)
    gray_r = bgr_r.astype(np.float32) @ np.array([0.114, 0.587, 0.299], np.float32)
    T = np.linalg.inv(pose_r.astype(np.float64)) @ pose_d.astype(np.float64)
    return K4, depth, gray_r, T


@pytest.mark.parametrize("size,step", [((480, 640), 1), ((480, 640), 3), ((121, 161), 1), ((121, 161), 3), ((67, 517), 1)])
def test_dense_reference_sizes(size, step):
    """Bit-exact against FrontOracle where the row chunks of 256 do not divide the row (517: w - 4 = 513, one pixel in the
    third chunk)."""
    h, w = size
    K4, depth, gray, T = _dense_case(h, w)
    n_ref, arrs, _ = FrontOracle().dense_reference(depth, T, K4, step, True, None, None, gray)
    assert n_ref > 100
    t = CudaCoarseTracker(w, h)
    t.init()
    t.setK(w, h, *K4)
    n = t.setReferenceDense(T, 1.0, np.zeros(2), depth=depth, tracking_step=step, ref_gray=gray)
    assert n == n_ref
    got = t.getReference(n + 1)
    for a, b, name in zip(got, arrs, ("u", "v", "idepth", "color")):
        assert np.array_equal(a, b), name
    if size == (121, 161) and step == 1:
        exact = CudaCoarseTracker(w, h)                 # n_max just sufficient: n points + the uncounted last one
        exact.init(n_ref + 1)
        exact.setK(w, h, *K4)
        assert exact.setReferenceDense(T, 1.0, np.zeros(2), depth=depth, tracking_step=step, ref_gray=gray) == n_ref
        assert all(np.array_equal(a, b) for a, b in zip(exact.getReference(n_ref + 1), arrs))
        short = CudaCoarseTracker(w, h)
        short.init(n_ref)
        short.setK(w, h, *K4)
        with pytest.raises(Exception):
            short.setReferenceDense(T, 1.0, np.zeros(2), depth=depth, tracking_step=step, ref_gray=gray)


@pytest.mark.parametrize("with_sparse", [False, True])
def test_refused_set_reference_dense_leaves_the_reference(with_sparse):
    """A setReferenceDense refused for lack of n_max leaves the current reference - and so calcRes - as it was."""
    h, w = 121, 161
    K4, depth, gray, T = _dense_case(h, w)
    n_small, _, _ = FrontOracle().dense_reference(depth, T, K4, 3, True, None, None, gray)
    n_big, _, _ = FrontOracle().dense_reference(depth, T, K4, 1, True, None, None, gray)
    t = CudaCoarseTracker(w, h)
    t.init(n_small + 1 + 50)
    t.setK(w, h, *K4)
    n = t.setReferenceDense(T, 1.0, np.zeros(2), depth=depth, tracking_step=3, ref_gray=gray)
    assert n == n_small and n_big + 1 > n_small + 51
    pts = t.getReference(n + 1)
    t.setReference(n, *[a[1:] for a in pts], 1.0, np.zeros(2))      # point 0 a real point (not the zeroed stale slot)
    rng = np.random.default_rng(2)
    dI = np.stack([gray, rng.normal(0, 4, (h, w)), rng.normal(0, 4, (h, w))], -1).astype(np.float32)
    t.setNew(dI)
    pose = np.eye(4)
    pose[0, 3] = 0.01
    r0 = t.calcRes(pose, 1.0, np.zeros(2), 20.0)
    ref0 = t.getReference(n + 1)
    sparse = None
    if with_sparse:
        sparse = [np.full(21, 7.0, np.float32), np.full(21, 9.0, np.float32), np.full(21, 0.5, np.float32),
                  np.full(21, 100.0, np.float32)]
    with pytest.raises(Exception):
        t.setReferenceDense(T, 1.0, np.zeros(2), depth=depth, tracking_step=1, ref_gray=gray, sparse=sparse, dense_only=not with_sparse)
    ref1 = t.getReference(n + 1)
    assert all(np.array_equal(a, b) for a, b in zip(ref0, ref1)), "the refused call changed the reference"
    r1 = t.calcRes(pose, 1.0, np.zeros(2), 20.0)
    assert np.array_equal(r0, r1)
