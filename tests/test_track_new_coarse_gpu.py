"""GPU tests of tdm_tracker_track_new_coarse (SURVEY 8f n6): the motion-hypothesis loop of FullSystem::trackNewCoarse
(FullSystem.cpp:538-617) on the device, every try an n5 run.  Levels are set up as in tests/test_track_pyramid_gpu.py: an
ImagePyramid of the new frame (setNewFromPyramid) and a setReferenceDense per level from the reference depth sub-sampled to
that level."""
import os
import subprocess

import numpy as np
import pytest

from oracle import pins_pyramid as P
from oracle import pins_retrack as R
from oracle.cpu import TrackerOracle
from oracle.pyramid_driver import track_pyramid as oracle_track_pyramid
from oracle.retrack_driver import track_new_coarse as host_loop
from tandem_b200 import CudaCoarseTracker, ImagePyramid, track_new_coarse, track_pyramid

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class Levels:
    def __init__(self, h=P.H, w=P.W, levels=P.LEVELS):
        gray_n, gray_r, depth_r, self.T_true = P.scene(h, w)
        K = P.intrinsics(w)
        self.pyr = ImagePyramid(w, h, levels)
        self.pyr.build(gray_n)
        pyr_ref = ImagePyramid(w, h, levels)
        pyr_ref.build(gray_r)
        self.trackers, self.n = [], []
        for l in range(levels):
            t = CudaCoarseTracker(w >> l, h >> l)
            t.init()
            t.setK(w >> l, h >> l, *P.level_K(l, K))
            g = np.ascontiguousarray(pyr_ref.level(l)[0][..., 0])
            self.n.append(t.setReferenceDense(np.eye(4), 1.0, P.REF_AFF, depth=np.ascontiguousarray(depth_r[::2 ** l, ::2 ** l]),
                                              dense_only=True, ref_gray=g))
            t.setNewFromPyramid(self.pyr, l)
            self.trackers.append(t)
        self.K = K

    def oracles(self):
        out = []
        for l, t in enumerate(self.trackers):
            o = TrackerOracle(t.w, t.h)
            o.setK(t.w, t.h, *P.level_K(l, self.K))
            o.setReference(self.n[l], *t.getReference(self.n[l]), 1.0, P.REF_AFF)
            o.setNew(self.pyr.level(l)[0])
            out.append(o)
        return out


def _kw(a):
    return dict(coarse_cutoff=a["coarse_cutoff"], affine_opt_mode_a=a["mode_a"], affine_opt_mode_b=a["mode_b"])


def _device(L, tries, rmse, a):
    return track_new_coarse(L.trackers, tries, P.REF_AFF, a["new_exposure"], rmse, **_kw(a))


def _host_driven(L, tries, rmse, a):
    """The same loop with every try a track_pyramid call from the host (one host wait per try)."""
    def tp(T, aff, min_res):
        return track_pyramid(L.trackers, T, aff, a["new_exposure"], min_res_for_abort=min_res, **_kw(a))
    return host_loop(tp, tries, P.REF_AFF, rmse)


def _pose_err(A, B):
    D = np.linalg.inv(A) @ B
    return np.linalg.norm(D[:3, 3]), np.arccos(np.clip((np.trace(D[:3, :3]) - 1) / 2, -1, 1))


def _same(a, b):
    return np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True)


def _replay_takeover(per_try):
    """achievedRes from the device's own per-try records by the rules of FullSystem.cpp:586-602, and the tries that changed a
    level of it without winning."""
    ach, good, losers_taking_over = np.full(5, np.nan), False, []
    with np.errstate(invalid="ignore", over="ignore"):
        for i, t in enumerate(per_try):
            last = t["last_residuals"]
            won = t["ok"] and np.isfinite(np.float32(last[0])) and not (last[0] >= ach[0])
            good = good or won
            if good:
                before = ach.copy()
                for l in range(5):
                    if not np.isfinite(np.float32(ach[l])) or ach[l] > last[l]:
                        ach[l] = last[l]
                if not won and not _same(before, ach):
                    losers_taking_over.append(i)
    return ach, losers_taking_over


def _assert_bit_identical(d, h):
    for k in ("refToNew", "aff", "flow_vecs", "achieved_res"):
        assert _same(d[k], h[k]), k
    assert d["have_one_good"] == h["have_one_good"] and d["tries"] == h["tries"] and d["winner"] == h["winner"]
    assert len(d["per_try"]) == len(h["per_try"]) == d["tries"]
    for i, (x, y) in enumerate(zip(d["per_try"], h["per_try"])):
        for k in ("ok", "aborted_level", "repeated_level"):
            assert x[k] == y[k], (i, k)
        assert _same(x["last_residuals"], y["last_residuals"]) and _same(x["evaluations"], y["evaluations"]), i


ALL31 = "all31"   # the full list of FullSystem.cpp:437-530 around the far motion of pins_retrack, lastCoarseRMSE 0: every try runs


@pytest.mark.parametrize("case", list(R.CASES) + [ALL31])
@pytest.mark.parametrize("size", [(240, 320), (480, 640)])
def test_track_new_coarse_equals_host_loop_over_track_pyramid(size, case):
    """One track_new_coarse call equals the restated loop driving the device's track_pyramid from the host, bit for bit:
    result, winner pose and every per-try record."""
    L = Levels(*size)
    if case == ALL31:
        tries, rmse, a = R.motion_tries(R.FAR, L.T_true), np.zeros(5), R.DSO
    else:
        tries, rmse, a = R.case_inputs(case)
    d = _device(L, tries, rmse, a)
    h = _host_driven(L, tries, rmse, a)
    print(f"{size} {case}: tries {d['tries']} winner {d['winner']} aborted {[t['aborted_level'] for t in d['per_try']]} "
          f"evaluations {sum(int(t['evaluations'].sum()) for t in d['per_try'])}, {d['device_ms']:.3f} ms on device")
    _assert_bit_identical(d, h)
    assert _same(d["achieved_res"], _replay_takeover(d["per_try"])[0])
    if case == ALL31:
        assert d["tries"] == 31 and any(t["aborted_level"] >= 0 for t in d["per_try"])


@pytest.mark.parametrize("name", list(R.CASES))
def test_track_new_coarse_matches_restatement(name):
    """Parity with oracle/retrack_driver.py over CPU trackers (pinned to the reference) given the same per-level inputs."""
    tries, rmse, a = R.case_inputs(name)
    L = Levels()
    d = _device(L, tries, rmse, a)
    orc = L.oracles()

    def tp(T, aff, min_res):
        return oracle_track_pyramid(orc, T, aff, a["new_exposure"], 1.0, P.REF_AFF, coarse_cutoff=a["coarse_cutoff"],
                                    mode_a=a["mode_a"], mode_b=a["mode_b"], min_res_for_abort=min_res)
    o = host_loop(tp, tries, P.REF_AFF, rmse)
    dt, dr = _pose_err(o["refToNew"], d["refToNew"])
    print(f"{name}: tries {d['tries']} (oracle {o['tries']}) winner {d['winner']} (oracle {o['winner']}), dt {dt:.2e} m, "
          f"dR {dr:.2e} rad, {d['device_ms']:.3f} ms on device")
    assert d["tries"] == o["tries"] and d["winner"] == o["winner"] and d["have_one_good"] == o["have_one_good"]
    for i, (x, y) in enumerate(zip(d["per_try"], o["per_try"])):
        for k in ("ok", "aborted_level", "repeated_level"):
            assert x[k] == y[k], (i, k)
        assert np.array_equal(np.isnan(x["last_residuals"]), np.isnan(y["last_residuals"])), i
    assert dt < 1e-3 and dr < 1e-3                       # SURVEY 8(d) config 4 bar
    assert np.allclose(d["aff"], o["aff"], atol=1e-3 * max(1.0, np.abs(o["aff"]).max()))
    assert np.array_equal(np.isnan(d["achieved_res"]), np.isnan(o["achieved_res"]))
    fin = ~np.isnan(o["achieved_res"])
    assert np.allclose(d["achieved_res"][fin], o["achieved_res"][fin], rtol=1e-3)
    ach, losers = _replay_takeover(d["per_try"])          # the device's takeover, exactly, on its own per-try records
    assert _same(d["achieved_res"], ach)
    if name == "exhaust":                                 # tries that do not win take over levels of achievedRes
        assert losers and all(i > d["winner"] for i in losers)
    if not o["have_one_good"]:
        assert _same(d["refToNew"], tries[0]) and _same(d["flow_vecs"], np.zeros(3)) and _same(d["aff"], P.REF_AFF)


def test_track_new_coarse_errors_launch_nothing():
    L = Levels()
    tries, rmse, a = R.case_inputs("retrack")
    base = _device(L, tries, rmse, a)
    base_p = track_pyramid(L.trackers, np.eye(4), P.REF_AFF, 1.05, **_kw(a))
    base_t = L.trackers[2].track(np.eye(4), P.REF_AFF, 1.05)
    fresh = CudaCoarseTracker(P.W >> 1, P.H >> 1)
    fresh.init()
    with pytest.raises(Exception, match="setK"):
        track_new_coarse([L.trackers[0], fresh] + L.trackers[2:], tries, P.REF_AFF, 1.05, rmse)
    fresh.setK(P.W >> 1, P.H >> 1, *P.level_K(1))
    with pytest.raises(Exception, match="reference"):
        track_new_coarse([L.trackers[0], fresh] + L.trackers[2:], tries, P.REF_AFF, 1.05, rmse)
    fresh.setReference(L.n[1], *L.trackers[1].getReference(L.n[1]), 1.0, P.REF_AFF)
    with pytest.raises(Exception, match="new image"):
        track_new_coarse([L.trackers[0], fresh] + L.trackers[2:], tries, P.REF_AFF, 1.05, rmse)
    with pytest.raises(Exception, match="size"):
        track_new_coarse([L.trackers[0], L.trackers[2], L.trackers[1], L.trackers[3]], tries, P.REF_AFF, 1.05, rmse)
    with pytest.raises(Exception, match="0..4"):
        track_new_coarse(L.trackers + L.trackers[3:] * 2, tries, P.REF_AFF, 1.05, rmse)
    with pytest.raises(Exception, match="0..4"):
        track_new_coarse([], tries, P.REF_AFF, 1.05, rmse)
    with pytest.raises(Exception, match="max_iterations"):
        track_new_coarse(L.trackers, tries, P.REF_AFF, 1.05, rmse, max_iterations=(10, 20, 201, 50))
    with pytest.raises(Exception, match="1..64"):
        track_new_coarse(L.trackers, np.zeros((0, 4, 4)), P.REF_AFF, 1.05, rmse)
    with pytest.raises(Exception, match="1..64"):
        track_new_coarse(L.trackers, np.tile(np.eye(4), (65, 1, 1)), P.REF_AFF, 1.05, rmse)
    again = _device(L, tries, rmse, a)
    _assert_bit_identical(again, base)
    p = track_pyramid(L.trackers, np.eye(4), P.REF_AFF, 1.05, **_kw(a))
    for k in ("refToNew", "aff", "last_residuals", "last_flow_indicators", "evaluations", "iterations"):
        assert _same(p[k], base_p[k]), k
    t = L.trackers[2].track(np.eye(4), P.REF_AFF, 1.05)
    assert _same(t["refToNew"], base_t["refToNew"]) and t["evaluations"] == base_t["evaluations"]


def test_shim_track_new_coarse():
    """CudaCoarseTracker::trackNewCoarse (shims/cuda_coarse_tracker.cpp) through the C++ executable build() links."""
    exe = os.path.join(ROOT, "tests", "cpp", "shim_new_coarse")
    if not os.path.exists(exe):
        pytest.skip("tests/cpp/shim_new_coarse not built (run __graft_entry__.build())")
    p = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    print(p.stdout)
    assert p.returncode == 0, p.stdout + p.stderr
