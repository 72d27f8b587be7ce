"""GPU parity of tdm_tracker_set_coarse_tracking_ref_nodia: n7 (tdm_tracker_set_coarse_tracking_ref) plus makeCoarseDepthL0's
undilated level-0 cloud pc_*_nodia and get_idepth_quantile over it, the MVSNet depth range of FullSystem::deliverDrFrame.
The cloud (slot pc_n_nodia included) and both quantile values are compared bit for bit with coarse_nodia_oracle /
idepth_quantile_oracle, which tests/test_coarse_nodia_cpu.py pins to the reference's own code; every level's pc_n and arrays
with a plain n7 call on twin trackers."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from oracle import pins_coarse_ref as P
from oracle.coarse_nodia import CoarseNodiaOracle, run_oracle
from tandem_b200 import ImagePyramid, set_coarse_tracking_ref, set_coarse_tracking_ref_nodia
from tandem_b200._lib import CoarseNodiaResult, TandemError, lib
from tandem_b200.tracker import _coarse_ref_call
from test_coarse_ref_gpu import AFF, GOLDEN, H, K0, L, W, fusion_render, room_keyframe, trackers

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def same(a, b):
    """Equal float32 bits, any NaN equal to any NaN."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(a[~np.isnan(a)].view(np.uint32), b[~np.isnan(b)].view(np.uint32))


def nodia_call(ts, points, pyr, fraction, **kw):
    """set_coarse_tracking_ref_nodia with the whole result: (pc_n, pc_n_nodia, idepth_quantile, depth_quantile)."""
    r = CoarseNodiaResult()
    args = dict(depth=None, fusion=None, render_index=0, T_depth_to_ref=None, tracking_step=1, dense_only=False, rgbd_init=False,
                ref_exposure=1.0, ref_aff_g2l=AFF)
    args.update(kw)
    pc_n = _coarse_ref_call(ts, points, pyr, nodia=(fraction, r), **args)
    return pc_n, r.pc_n_nodia, r.idepth_quantile, r.depth_quantile


def assert_levels_equal(ts, twins, pc_n):
    for l, (a, b) in enumerate(zip(ts, twins)):
        for k, (x, y) in enumerate(zip(a.getReference(pc_n[l] + 1), b.getReference(pc_n[l] + 1))):
            assert same(x, y), (l, k)


@pytest.mark.parametrize("name", list(P.CASES))
def test_nodia_matches_pinned_oracle_and_n7(name):
    T = np.load(GOLDEN)[f"{name}_T"]
    (h, w), levels, gray_levels, depth, kfs = P.case_inputs(name)
    expect = run_oracle(name)
    pyr = ImagePyramid(w, h, levels)
    pyr.build(P.gray_image(h, w, 0))
    ts, twins = trackers(w, h, levels, P.K4(h, w)), trackers(w, h, levels, P.K4(h, w))
    for kf, (m, arrs, fr, q) in zip(kfs, expect):
        kw = dict(depth=depth if kf["dense"] else None, T_depth_to_ref=T, tracking_step=kf["step"], dense_only=kf["dense_only"],
                  rgbd_init=kf["rgbd"], ref_exposure=1.25)
        plain = set_coarse_tracking_ref(twins, kf["points"], pyr, ref_aff_g2l=AFF, **kw)
        for f, qf in zip(fr, q):   # the same keyframe again per fraction: the cloud and its slot come out the same
            pc_n, n_nodia, idq, dq = nodia_call(ts, kf["points"], pyr, f, **kw)
            assert pc_n == plain
            assert n_nodia == m
            assert same(idq, qf[0]) and same(dq, qf[1]), (f, idq, dq, qf)
            for k, (a, b) in enumerate(zip(ts[0].getCoarseNodia(m + 1), arrs)):
                assert same(a, b), (f, k, np.flatnonzero(a.view(np.uint32) != b.view(np.uint32))[:10])
        assert_levels_equal(ts, twins, pc_n)


@pytest.fixture(scope="module")
def room():
    gray, pts, T = room_keyframe()
    pyr = ImagePyramid(W, H, L)
    pyr.build(gray)
    gray0 = np.ascontiguousarray(pyr.level(0)[0][..., 0])
    fus, depth = fusion_render()
    return dict(gray=gray, pts=pts, T=T, pyr=pyr, gray0=gray0, fus=fus, depth=depth)


def oracle_nodia(pts, gray0, fraction, o=None):
    o = o or CoarseNodiaOracle(W, H)
    m = o.make(pts, gray0)
    return m, o.result(m + 1), o.quantile(m, fraction)


@pytest.mark.parametrize("source", ["host", "fusion", "none"])
@pytest.mark.parametrize("n", [2000, 8000])
def test_room_keyframe(room, source, n):
    _, pts, _ = room_keyframe(0, n)
    ts, twins = trackers(W, H, L, K0), trackers(W, H, L, K0)
    kw = dict(depth=room["depth"]) if source == "host" else dict(fusion=room["fus"]) if source == "fusion" else {}
    plain = set_coarse_tracking_ref(twins, pts, room["pyr"], T_depth_to_ref=room["T"], ref_aff_g2l=AFF, **kw)
    pc_n, n_nodia, dq = set_coarse_tracking_ref_nodia(ts, pts, room["pyr"], 0.2, T_depth_to_ref=room["T"], ref_aff_g2l=AFF, **kw)
    assert pc_n == plain
    assert_levels_equal(ts, twins, pc_n)
    m, arrs, q = oracle_nodia(pts, room["gray0"], 0.2)
    assert n_nodia == m and m > 0.8 * n
    assert same(dq, q[1]) and np.isfinite(dq) and dq > 0
    assert all(same(a, b) for a, b in zip(ts[0].getCoarseNodia(m + 1), arrs))


def test_two_keyframes_keep_the_stale_slot_and_plain_calls_leave_the_cloud(room):
    ts = trackers(W, H, L, K0)
    o = CoarseNodiaOracle(W, H)
    for seed, n in ((0, 2000), (1, 300)):
        _, pts, _ = room_keyframe(seed, n)
        pts[2][::50] = -pts[2][::50]                      # rejected candidates
        pc_n, n_nodia, idq, dq = nodia_call(ts, pts, room["pyr"], 0.2)
        m, arrs, q = oracle_nodia(pts, room["gray0"], 0.2, o)
        assert n_nodia == m and same(idq, q[0]) and same(dq, q[1])
        assert all(same(a, b) for a, b in zip(ts[0].getCoarseNodia(m + 1), arrs))
    # a plain n7 call with other points rebuilds the levels but leaves the nodia cloud (and slot) as the last _nodia call left it
    before = ts[0].getCoarseNodia(W * H)
    _, other, _ = room_keyframe(2, 1000)
    set_coarse_tracking_ref(ts, other, room["pyr"], depth=room["depth"], T_depth_to_ref=room["T"], ref_aff_g2l=AFF)
    assert all(same(a, b) for a, b in zip(ts[0].getCoarseNodia(W * H), before))


def _raw(ts, n_levels, pts, pyr, fraction, out=True):
    fp = ctypes.POINTER(ctypes.c_float)
    hs = None if ts is None else (ctypes.c_void_p * max(len(ts), 1))(*[t._h for t in ts])
    arrs = [None if a is None else np.ascontiguousarray(a, np.float32) for a in pts]
    n = 0 if arrs[0] is None else len(arrs[0])
    aff = np.zeros(2)
    pc_n = np.zeros(5, np.int32)
    r = CoarseNodiaResult()
    return lib().tdm_tracker_set_coarse_tracking_ref_nodia(
        hs, n_levels, 0, n, *[None if a is None else a.ctypes.data_as(fp) for a in arrs], None if pyr is None else pyr._h,
        None, None, 0, None, 1, 0, 1.0, aff.ctypes.data_as(ctypes.POINTER(ctypes.c_double)), ctypes.c_float(fraction),
        pc_n.ctypes.data_as(ctypes.POINTER(ctypes.c_int)), ctypes.byref(r) if out else None)


def test_errors_launch_nothing_and_a_valid_call_follows(room):
    ts = trackers(W, H, L, K0)
    pts, pyr = room["pts"], room["pyr"]
    with pytest.raises(TandemError):                      # no _nodia call on this tracker yet
        ts[0].getCoarseNodia(1)
    assert lib().tdm_tracker_get_coarse_nodia(None, 0, None, None, None, None) < 0
    for f in (-0.1, 1.0000001, np.nan, np.inf, -np.inf):
        with pytest.raises(TandemError):
            set_coarse_tracking_ref_nodia(ts, pts, pyr, f)
    with pytest.raises(TandemError):                      # the failed calls made no cloud
        ts[0].getCoarseNodia(1)
    m, arrs, q = oracle_nodia(pts, room["gray0"], 0.2)

    def valid():
        pc_n, n_nodia, idq, dq = nodia_call(ts, pts, pyr, 0.2, depth=room["depth"], T_depth_to_ref=room["T"])
        assert n_nodia == m and same(idq, q[0]) and same(dq, q[1])
        assert all(same(a, b) for a, b in zip(ts[0].getCoarseNodia(m + 1), arrs))
        return pc_n

    pc_n = valid()
    levels0 = [t.getReference(n + 1) for t, n in zip(ts, pc_n)]
    _, other, _ = room_keyframe(3, 500)
    cases = [
        lambda: _raw(ts, L, other, pyr, 1.5),                # bad fraction
        lambda: _raw(ts, L, other, pyr, float("nan")),
        lambda: _raw(ts, L, other, pyr, 0.2, out=False),     # null result
        lambda: _raw(None, L, other, pyr, 0.2),              # null levels
        lambda: _raw(ts, L, other, None, 0.2),               # null pyramid
        lambda: _raw(ts, L, (other[0], None, None, None), pyr, 0.2),   # point arrays missing
        lambda: _raw(ts, 0, other, pyr, 0.2),                # n_levels 0
    ]
    for c in cases:
        assert c() < 0
        # nothing ran: the cloud and every level's reference are still the valid call's
        assert all(same(a, b) for a, b in zip(ts[0].getCoarseNodia(m + 1), arrs))
        for t, n, ref in zip(ts, pc_n, levels0):
            assert all(same(a, b) for a, b in zip(t.getReference(n + 1), ref))
    assert valid() == pc_n
    with pytest.raises(TandemError):
        ts[0].getCoarseNodia(W * H + 1)


def test_shim_runs_set_coarse_tracking_ref_with_the_depth_range():
    exe = os.path.join(ROOT, "tests", "cpp", "shim_coarse_nodia")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "shim_coarse_nodia: OK" in r.stdout

