"""The fp64 tracker reference with per-output bounds (oracle/tracker_eval.py), checked without a GPU: the C oracle's fp32
evaluation (oracle/tracker_oracle.c) lies within every bound, and errors planted into its H / b that the relative-to-max
tolerance of test_tracker_gpu.py lets through fail the per-entry check."""
import numpy as np
import pytest

from oracle import tracker_eval as te
from oracle.cpu import TrackerOracle
from tandem_b200.synthetic import tracker_case


def _old_rel(a, b):
    return np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-30)


def _oracle(c, huber=9.0):
    o = TrackerOracle(c["w"], c["h"], huber, 20.0)
    o.setK(c["w"], c["h"], c["fx"], c["fy"], c["cx"], c["cy"])
    o.setReference(c["n"], c["pc_u"], c["pc_v"], c["pc_idepth"], c["pc_color"], c["ref_exposure"], c["ref_aff"])
    o.setNew(c["dInew"])
    return o


def _params(c, T, cutoff, huber=9.0, new_exposure=None, new_aff=None):
    return te.Params(c["w"], c["h"], c["fx"], c["fy"], c["cx"], c["cy"], huber, T, cutoff, c["ref_exposure"],
                     c["new_exposure"] if new_exposure is None else new_exposure, c["ref_aff"],
                     c["new_aff"] if new_aff is None else new_aff)


def _check_points(ev, W):
    """The per-point rules of the GPU test, here against the C oracle's warped buffers."""
    acc = W[6] != 0
    pr = ev.pr
    diff = acc != ev.accepted
    assert not (diff & ~ev.excused).any(), np.nonzero(diff & ~ev.excused)[0][:10]
    assert not (acc & ~ev.finite).any()
    for k, name in ((0, "u"), (1, "v"), (4, "nid")):
        assert np.array_equal(W[k][acc], pr[name][acc]), name
    assert not W[:, ~acc].any(), "rejected points must be zero in every array"
    r = [te.ratio(W[2][acc], ev.hit[acc, 1], ev.bil[acc, 1]), te.ratio(W[3][acc], ev.hit[acc, 2], ev.bil[acc, 2]),
         te.ratio(W[5][acc], ev.res[acc], ev.res_b[acc])]
    h = np.float32(ev.P.huber)
    ar = np.abs(W[5][acc])
    with np.errstate(divide="ignore"):
        hw = np.where(ar < h, np.float32(1), h / ar).astype(np.float32)
    assert np.array_equal(W[6][acc], hw), "hw must follow from res"
    return max(r)


@pytest.fixture(scope="module")
def case():
    return tracker_case(H=120, W=160, fx=80.0, fy=80.0, cx=79.5, cy=59.5)


def test_oracle_values_lie_within_the_bounds(case):
    c = case
    o = _oracle(c)
    res = o.calcRes(c["refToNew"], c["new_exposure"], c["new_aff"], c["cutoffTH"])
    H, b = o.calcG(c["new_exposure"], c["new_aff"])
    P = _params(c, c["refToNew"], c["cutoffTH"])
    ev = te.Eval(P, c["pc_u"], c["pc_v"], c["pc_idepth"], c["pc_color"], c["dInew"])
    assert ev.nW > 0.5 * c["n"]
    worst = {"dx/dy/res": _check_points(ev, o.warped)}
    assert res[1] == ev.res6[1]
    worst["E"] = te.ratio(res[0], ev.res6[0], ev.res6_b[0])
    worst["flow"] = max(te.ratio(res[2], ev.res6[2], ev.res6_b[2]), te.ratio(res[4], ev.res6[4], ev.res6_b[4]))
    acc, bound = te.g_sums(P, o.warped, c["pc_color"], c["n"])
    Hr, Hb, br, bb = te.pack_hb(acc, bound, int(o.out7[2]))
    worst["H"], worst["b"] = te.ratio(H, Hr, Hb), te.ratio(b, br, bb)
    print("worst error / bound:", {k: f"{v:.3g}" for k, v in worst.items()})
    assert all(v <= 1 for v in worst.values()), worst
    # the bounds are tight enough to mean something: relative to each entry's own magnitude (not the matrix maximum)
    rel = np.concatenate([(Hb / np.abs(Hr)).ravel(), bb / np.abs(br)])
    assert np.median(rel) < 1e-5 and rel.max() < 1e-3, rel


def test_planted_errors_fail_the_per_entry_check_and_pass_the_old_one(case):
    c = case
    o = _oracle(c)
    o.calcRes(c["refToNew"], c["new_exposure"], c["new_aff"], c["cutoffTH"])
    H, b = o.calcG(c["new_exposure"], c["new_aff"])
    P = _params(c, c["refToNew"], c["cutoffTH"])
    W = o.warped.astype(np.float64)
    nw = int(o.out7[2])
    acc, bound = te.g_sums(P, W, c["pc_color"], c["n"])
    Hr, Hb, br, bb = te.pack_hb(acc, bound, nw)
    assert te.ratio(H, Hr, Hb) <= 1 and te.ratio(b, br, bb) <= 1
    sel = np.nonzero(W[6] != 0)[0]
    planted = {}
    # 1. one accepted point's G contribution dropped (a typical one: its |products| at the median)
    Pp, _ = te.g_terms(P, W[:, sel], np.asarray(c["pc_color"], np.float64)[sel])
    mag = np.abs(Pp).sum(axis=0)
    k = int(np.argsort(mag)[mag.size // 2])
    H1, _, b1, _ = te.pack_hb(acc - Pp[:, k], bound, nw)
    planted["dropped point"] = (H1, b1)
    # 2. the pose rows of H and b scaled by 1 + 1e-3
    H2, b2 = H.copy(), b.copy()
    H2[:6] *= 1 + 1e-3
    b2[:6] *= 1 + 1e-3
    planted["pose rows x (1 + 1e-3)"] = (H2, b2)
    # 3. u and v swapped in J[5] on 0.1 % of the accepted points (on 1 % the relative-to-max check already sees it here)
    rng = np.random.default_rng(0)
    pick = sel[rng.random(sel.size) < 0.001]
    assert pick.size >= 5
    Ws = W[:, pick].copy()
    Ws[[0, 1]] = Ws[[1, 0]]
    Pa, _ = te.g_terms(P, W[:, pick], np.asarray(c["pc_color"], np.float64)[pick])
    Pb_, _ = te.g_terms(P, Ws, np.asarray(c["pc_color"], np.float64)[pick])
    d = np.zeros_like(acc)
    for i, (j1, j2) in enumerate(te.PAIRS):
        if 5 in (j1, j2):
            d[i] = (Pb_[i] - Pa[i]).sum()                 # only the products with J[5] see the swap
    H3, _, b3, _ = te.pack_hb(acc + d, bound, nw)
    planted["u<->v in J[5] on 0.1 %"] = (H3, b3)
    for name, (Hp, bp) in planted.items():
        old = max(_old_rel(Hp, H), _old_rel(bp, b))
        new = max(te.ratio(Hp, Hr, Hb), te.ratio(bp, br, bb))
        print(f"{name}: old relative-to-max {old:.2e} (passes < 1e-4), worst error / bound {new:.3g} (fails > 1)")
        assert old < 1e-4, name
        assert new > 1, name


@pytest.mark.parametrize("size", [(161, 121), (33, 25)])
@pytest.mark.parametrize("hc", [(9.0, 20.0), (0.5, 0.5), (4.0, 2.0), (1e-3, 1e4)])
@pytest.mark.parametrize("translated", [False, True])
def test_exact_scene_against_the_c_oracle(size, hc, translated):
    w, h = size
    c = te.exact_scene(w, h, *hc)
    c.update(ref_exposure=1.0, ref_aff=np.zeros(2), new_exposure=1.0, new_aff=np.zeros(2))
    T = te.exact_pose(translated)
    o = _oracle(c, hc[0])
    res = o.calcRes(T, 1.0, np.zeros(2), hc[1])
    P = _params(c, T, hc[1], huber=hc[0])
    ev = te.Eval(P, c["pc_u"], c["pc_v"], c["pc_idepth"], c["pc_color"], c["dInew"])
    assert ev.n_excused == 0
    _check_points(ev, o.warped)
    assert res[1] == ev.res6[1] and res[5] == ev.res6[5] and int(o.out7[2]) == ev.nW
    for k in (0, 2, 4):
        assert te.ratio(res[k], ev.res6[k], ev.res6_b[k]) <= 1, k
    if not translated:
        # the probes decide as designed
        x, y = c["pc_u"], c["pc_v"]
        for ku, inside in ((2.0, False), (2.0 + 2 ** -8, True), (w - 3.0, False), (w - 3.0 - 2 ** -8, True)):
            at = (x == np.float32(ku)) & (y == np.float32(c["cy"]))
            assert at.sum() == 1 and bool(ev.pr["inframe"][at][0]) == inside, ku
        idp = (x == np.float32(c["cx"] + 1)) & (y == np.float32(c["cy"]))
        assert list(ev.pr["inframe"][idp]) == [False, False, False, True, True, True, True]
        assert ev.nS >= 40 and ev.nW > 0
    else:
        assert (ev.pr["p1"][2] == 0).any() and (ev.pr["p1"][2] < 0).any()
    assert (~np.isfinite(ev.hit[:, 0][ev.pr["inframe"]])).sum() >= (0 if translated else 15)
