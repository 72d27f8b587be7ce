"""n5 pin (no GPU): the coarse-to-fine restatement oracle/pyramid_driver.py == the reference's own body of
CoarseTracker::trackNewestCoarse (CoarseTracker.cpp:750-936) when both drive the SAME per-level tracker oracles.  The reference's
results are stored in tests/golden/reference_pins_pyramid.npz (oracle/gen_reference_pins_pyramid.py)."""
import os

import numpy as np
import pytest

from oracle import pins_pyramid as P
from oracle.pyramid_driver import track_pyramid

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_pins_pyramid.npz")


@pytest.fixture(scope="module")
def levels():
    return P.level_inputs()


@pytest.mark.parametrize("name", list(P.CASES))
def test_track_pyramid_pinned_to_reference_trackNewestCoarse(levels, name):
    g = np.load(GOLDEN)
    ref = {k: g[f"{name}_{k}"] for k in ("ok", "T", "aff", "last_res", "flow", "counts", "repeated_level")}
    case = P.CASES[name]
    r = track_pyramid(P.oracle_trackers(levels), np.eye(4), P.REF_AFF, case["new_exposure"], 1.0, P.REF_AFF,
                      coarse_cutoff=case["coarse_cutoff"], mode_a=case["mode_a"], mode_b=case["mode_b"],
                      min_res_for_abort=case["min_res"])
    assert r["ok"] == bool(ref["ok"])
    assert list(r["evaluations"]) == list(ref["counts"])            # same accept / reject sequences, doublings, stops, repeat
    assert r["repeated_level"] == int(ref["repeated_level"])
    over = [l for l in range(5) if ref["last_res"][l] > 1.5 * case["min_res"][l]]
    assert r["aborted_level"] == (over[0] if over else -1)
    # The two linear solvers (numpy vs the stand-in LDLT) differ in the last bits; fp32 evaluations amplify that, most in the
    # small-cutoff case where many residuals sit at the cutoff.  The control flow above is compared exactly.
    assert np.abs(r["refToNew"] - ref["T"]).max() < 1e-4
    assert abs(r["aff"][0] - ref["aff"][0]) < 1e-4 and abs(r["aff"][1] - ref["aff"][1]) < 2e-3   # b in grey levels
    assert np.array_equal(np.isnan(r["last_residuals"]), np.isnan(ref["last_res"]))
    fin = ~np.isnan(ref["last_res"])
    assert np.allclose(r["last_residuals"][fin], ref["last_res"][fin], rtol=1e-3, atol=0)
    assert np.allclose(r["last_flow_indicators"], ref["flow"], rtol=1e-3, atol=1e-6)
    # each case exercises what it is named for
    if name == "converge":
        assert r["ok"] and r["repeated_level"] == -1 and all(r["evaluations"][:4] > 0) and np.isfinite(r["last_residuals"][:4]).all()
        _, _, _, T_true = P.scene()
        assert np.linalg.norm((np.linalg.inv(T_true) @ r["refToNew"])[:3, 3]) < 0.3 * np.linalg.norm(T_true[:3, 3])
    elif name == "repeat":
        assert r["repeated_level"] >= 0 and r["cutoff_repeat"].max() > 1 and r["ok"]
    elif name == "abort":
        assert not r["ok"] and r["aborted_level"] == 2 and np.array_equal(r["refToNew"], np.eye(4))
        assert np.array_equal(r["aff"], P.REF_AFF) and r["evaluations"][1] == 0
    elif name == "affine":
        assert not r["ok"] and r["aborted_level"] == -1 and abs(r["aff"][0]) > 1.2
        assert not np.array_equal(r["refToNew"], np.eye(4))                 # rejected after the pose was written (:919-924)
    elif name == "affine_mode0":
        assert r["ok"] and abs(r["aff"][0]) > 1.2
    elif name == "fixed_a":
        assert r["ok"] and r["aff"][0] == 0 and r["aff"][1] != 0
    elif name == "fixed_ab":
        assert r["ok"] and r["aff"][0] == 0 and r["aff"][1] == 0
