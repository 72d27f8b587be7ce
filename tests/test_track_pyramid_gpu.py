"""GPU tests of tdm_tracker_track_pyramid (SURVEY 8f n5): the coarse-to-fine loop of CoarseTracker::trackNewestCoarse on the
device.  Levels are set up as tandem_b200/loop.py sets them up: an ImagePyramid of the new frame (setNewFromPyramid) and a
setReferenceDense per level from the reference depth sub-sampled to that level."""
import os
import subprocess

import numpy as np
import pytest

from oracle import pins_pyramid as P
from oracle.cpu import TrackerOracle
from oracle.pyramid_driver import track_pyramid as oracle_track_pyramid
from tandem_b200 import CudaCoarseTracker, ImagePyramid, track_pyramid

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DSO_MODES = dict(affine_opt_mode_a=1e12, affine_opt_mode_b=1e8)   # settings.cpp:109-110


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
        """CPU trackers fed the device's own per-level inputs."""
        out = []
        for l, t in enumerate(self.trackers):
            o = TrackerOracle(t.w, t.h)
            o.setK(t.w, t.h, *P.level_K(l, self.K))
            o.setReference(self.n[l], *t.getReference(self.n[l]), 1.0, P.REF_AFF)
            o.setNew(self.pyr.level(l)[0])
            out.append(o)
        return out


def _pose_err(A, B):
    D = np.linalg.inv(A) @ B
    return np.linalg.norm(D[:3, 3]), np.arccos(np.clip((np.trace(D[:3, :3]) - 1) / 2, -1, 1))


def _same(a, b):
    return np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True)


@pytest.mark.parametrize("size", [(240, 320), (480, 640)])
def test_track_pyramid_equals_host_driven_track_per_level(size):
    """Without repeat or abort, one track_pyramid call equals tdm_tracker_track called level by level from the host, bit for
    bit; a one-level track_pyramid equals track."""
    L = Levels(*size)
    its = (10, 20, 50, 50)
    r = track_pyramid(L.trackers, np.eye(4), P.REF_AFF, 1.05, max_iterations=its, **DSO_MODES)
    assert r["ok"] and r["repeated_level"] == -1 and r["aborted_level"] == -1
    T, aff = np.eye(4), P.REF_AFF
    for l in range(3, -1, -1):
        h = L.trackers[l].track(T, aff, 1.05, max_iterations=its[l])
        T, aff = h["refToNew"], h["aff"]
        assert r["iterations"][l] == h["iterations"] and r["evaluations"][l] == h["evaluations"], l
        assert r["cutoff_repeat"][l] == h["cutoff_repeat"] == 1
        assert r["last_residuals"][l] == float(np.sqrt(np.float32(h["res"][0] / h["res"][1]))), l
    assert _same(r["refToNew"], T) and _same(r["aff"], aff)
    assert _same(r["last_flow_indicators"], h["res"][2:5])
    assert np.isnan(r["last_residuals"][4])
    e0, _ = _pose_err(L.T_true, np.eye(4))
    e1, _ = _pose_err(L.T_true, r["refToNew"])
    print(f"{size}: evaluations {list(r['evaluations'][:4])}, pose error {e0:.4f} -> {e1:.5f} m, {r['device_ms']:.3f} ms on device")
    assert e1 < 0.3 * e0
    one = track_pyramid(L.trackers[:1], np.eye(4), P.REF_AFF, 1.05, max_iterations=(10,), **DSO_MODES)
    h = L.trackers[0].track(np.eye(4), P.REF_AFF, 1.05, max_iterations=10)
    assert _same(one["refToNew"], h["refToNew"]) and _same(one["aff"], h["aff"])
    assert one["iterations"][0] == h["iterations"] and one["evaluations"][0] == h["evaluations"]


@pytest.mark.parametrize("name", list(P.CASES))
def test_track_pyramid_matches_restatement(name):
    """Parity with oracle/pyramid_driver.py (pinned to the reference's body) over CPU trackers given the same per-level inputs."""
    c = P.CASES[name]
    L = Levels()
    r = track_pyramid(L.trackers, np.eye(4), P.REF_AFF, c["new_exposure"], coarse_cutoff=c["coarse_cutoff"],
                      affine_opt_mode_a=c["mode_a"], affine_opt_mode_b=c["mode_b"], min_res_for_abort=c["min_res"])
    o = oracle_track_pyramid(L.oracles(), np.eye(4), P.REF_AFF, c["new_exposure"], 1.0, P.REF_AFF, coarse_cutoff=c["coarse_cutoff"],
                             mode_a=c["mode_a"], mode_b=c["mode_b"], min_res_for_abort=c["min_res"])
    dt, dr = _pose_err(o["refToNew"], r["refToNew"])
    print(f"{name}: ok {r['ok']} aborted {r['aborted_level']} repeated {r['repeated_level']} evaluations {list(r['evaluations'])} "
          f"(oracle {list(o['evaluations'])}), dt {dt:.2e} m, dR {dr:.2e} rad, {r['device_ms']:.3f} ms on device")
    assert r["ok"] == o["ok"] and r["aborted_level"] == o["aborted_level"] and r["repeated_level"] == o["repeated_level"]
    assert list(r["cutoff_repeat"]) == list(o["cutoff_repeat"])
    assert dt < 1e-3 and dr < 1e-3                       # SURVEY 8(d) config 4 bar
    assert np.allclose(r["aff"], o["aff"], atol=1e-3 * max(1.0, np.abs(o["aff"]).max()))
    if r["aborted_level"] >= 0:
        assert _same(r["refToNew"], np.eye(4)) and _same(r["aff"], P.REF_AFF)
    if name == "abort":
        assert r["aborted_level"] == 2
    if name == "repeat":
        assert r["repeated_level"] >= 0
    if name == "affine":
        assert not r["ok"] and r["aborted_level"] == -1
    if c["mode_a"] < 0 and r["ok"]:
        assert r["aff"][0] == 0


def test_track_pyramid_errors_launch_nothing():
    L = Levels()
    base = track_pyramid(L.trackers, np.eye(4), P.REF_AFF, 1.05, **DSO_MODES)
    fresh = CudaCoarseTracker(P.W >> 1, P.H >> 1)
    fresh.init()
    bad = [
        ("setK", lambda: [L.trackers[0], fresh] + L.trackers[2:]),
        ("reference", None),
        ("new image", None),
        ("size", lambda: [L.trackers[0], L.trackers[2], L.trackers[1], L.trackers[3]]),
        ("0..4", lambda: L.trackers + L.trackers[3:] * 2),
        ("0..4", lambda: []),
    ]
    with pytest.raises(Exception, match="setK"):
        track_pyramid(bad[0][1](), np.eye(4), P.REF_AFF, 1.05)
    fresh.setK(P.W >> 1, P.H >> 1, *P.level_K(1))
    with pytest.raises(Exception, match="reference"):
        track_pyramid([L.trackers[0], fresh] + L.trackers[2:], np.eye(4), P.REF_AFF, 1.05)
    fresh.setReference(L.n[1], *L.trackers[1].getReference(L.n[1]), 1.0, P.REF_AFF)
    with pytest.raises(Exception, match="new image"):
        track_pyramid([L.trackers[0], fresh] + L.trackers[2:], np.eye(4), P.REF_AFF, 1.05)
    for what, levels in bad[3:]:
        with pytest.raises(Exception, match=what):
            track_pyramid(levels(), np.eye(4), P.REF_AFF, 1.05)
    with pytest.raises(Exception, match="max_iterations"):
        track_pyramid(L.trackers, np.eye(4), P.REF_AFF, 1.05, max_iterations=(10, 20, 201, 50))
    with pytest.raises(Exception, match="max_iterations"):
        track_pyramid(L.trackers, np.eye(4), P.REF_AFF, 1.05, max_iterations=(10, -1, 50, 50))
    again = track_pyramid(L.trackers, np.eye(4), P.REF_AFF, 1.05, **DSO_MODES)
    for k in ("refToNew", "aff", "last_residuals", "last_flow_indicators", "evaluations", "iterations"):
        assert _same(again[k], base[k]), k
    h = L.trackers[2].track(np.eye(4), P.REF_AFF, 1.05)
    assert h["iterations"] > 0


def test_shim_track_pyramid():
    """CudaCoarseTracker::trackPyramid (shims/cuda_coarse_tracker.cpp) through the C++ executable build() links."""
    exe = os.path.join(ROOT, "tests", "cpp", "shim_pyramid")
    if not os.path.exists(exe):
        pytest.skip("tests/cpp/shim_pyramid not built (run __graft_entry__.build())")
    p = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    print(p.stdout)
    assert p.returncode == 0, p.stdout + p.stderr
