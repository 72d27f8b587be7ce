"""n6 pin (no GPU): the motion-hypothesis restatement oracle/retrack_driver.py == the reference's own lines of
FullSystem::trackNewCoarse (FullSystem.cpp:538-617, over its own CoarseTracker::trackNewestCoarse body) when both drive the SAME
per-level tracker oracles.  The reference's results are stored in tests/golden/reference_pins_retrack.npz
(oracle/gen_reference_pins_retrack.py)."""
import os

import numpy as np
import pytest

from oracle import pins_pyramid as P
from oracle import pins_retrack as R
from oracle.pyramid_driver import track_pyramid
from oracle.retrack_driver import track_new_coarse

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_pins_retrack.npz")


@pytest.fixture(scope="module")
def levels():
    return P.level_inputs()


def run_restatement(levels, name):
    tries, rmse, a = R.case_inputs(name)
    trk = P.oracle_trackers(levels)

    def tp(T, aff, min_res):
        return track_pyramid(trk, T, aff, a["new_exposure"], 1.0, P.REF_AFF, coarse_cutoff=a["coarse_cutoff"], mode_a=a["mode_a"],
                             mode_b=a["mode_b"], min_res_for_abort=min_res)
    return track_new_coarse(tp, tries, P.REF_AFF, rmse), tries, rmse


def takeovers(min_res, achieved):
    """(tries, 5) booleans: level l of achievedRes changed after try i, from achievedRes as each try started and the final one."""
    before = np.asarray(min_res, np.float64)
    after = np.concatenate([before[1:], np.asarray(achieved, np.float64)[None]])
    return ~((before == after) | (np.isnan(before) & np.isnan(after)))


@pytest.mark.parametrize("name", list(R.CASES))
def test_track_new_coarse_pinned_to_reference_trackNewCoarse(levels, name):
    g = np.load(GOLDEN)
    ref = {k[len(name) + 1:]: g[k] for k in g.files if k.startswith(name + "_")}
    r, tries, rmse = run_restatement(levels, name)
    # control flow, exactly
    assert r["tries"] == int(ref["tries"]) and r["winner"] == int(ref["winner"]) and r["have_one_good"] == bool(ref["have_one_good"])
    for i, t in enumerate(r["per_try"]):
        over = [l for l in range(5) if ref["try_last_res"][i][l] > 1.5 * ref["try_min_res"][i][l]]
        assert t["ok"] == bool(ref["try_ok"][i]), i
        assert t["aborted_level"] == (over[0] if over else -1), i
        assert t["repeated_level"] == int(ref["try_repeated_level"][i]), i
        assert list(t["evaluations"]) == list(ref["try_counts"][i]), i
        assert np.array_equal(np.isnan(t["last_residuals"]), np.isnan(ref["try_last_res"][i])), i
    # the takeover rule (:595-602), exactly: which levels of achievedRes each try changed
    mine = takeovers([t["min_res"] for t in r["per_try"]], r["achieved_res"])
    theirs = takeovers(ref["try_min_res"], ref["achieved_res"])
    assert np.array_equal(mine, theirs), (mine, theirs)
    # values, within the tolerances of tests/test_track_pyramid_cpu.py (numpy vs the stand-in LDLT differ in the last bits)
    assert np.abs(r["refToNew"] - ref["T"]).max() < 1e-4
    assert abs(r["aff"][0] - ref["aff"][0]) < 1e-4 and abs(r["aff"][1] - ref["aff"][1]) < 2e-3
    assert np.array_equal(np.isnan(r["achieved_res"]), np.isnan(ref["achieved_res"]))
    fin = ~np.isnan(ref["achieved_res"])
    assert np.allclose(r["achieved_res"][fin], ref["achieved_res"][fin], rtol=1e-3, atol=0)
    assert np.allclose(r["flow_vecs"], ref["flow"], rtol=1e-3, atol=1e-6)
    # each case exercises what it is named for
    if name == "first":
        assert r["tries"] == 1 and r["winner"] == 0 and len(tries) == 31
    elif name == "retrack":
        assert r["winner"] > 0 and r["tries"] == r["winner"] + 1 < len(tries)
        assert r["achieved_res"][0] < rmse[0] * 1.5
        aborted = [i for i, t in enumerate(r["per_try"]) if t["aborted_level"] >= 1]
        assert aborted and all(0 < i < r["winner"] for i in aborted)
    elif name == "exhaust":
        assert r["tries"] == len(tries)
        first_win = min(i for i, t in enumerate(r["per_try"]) if t["ok"])
        assert any(t["aborted_level"] >= 0 for t in r["per_try"][first_win + 1:])
        assert np.isnan(r["achieved_res"][4]) and np.isfinite(r["achieved_res"][:4]).all()   # level 4 is never reached
        for l in range(4):   # achievedRes is the level-wise minimum over the tries from the first winner on
            assert r["achieved_res"][l] == np.nanmin([t["last_residuals"][l] for t in r["per_try"][first_win:]])
        # tries that are ok but do not win (lastResiduals[0] >= achievedRes[0]) still take over a level of achievedRes
        losers = [i for i, t in enumerate(r["per_try"]) if t["ok"] and t["last_residuals"][0] >= t["min_res"][0]]
        assert losers and all(i > r["winner"] for i in losers)
        assert any(theirs[i].any() for i in losers)
        assert not any(theirs[i][0] for i in losers)
    elif name == "none_good":
        assert not r["have_one_good"] and r["winner"] == -1 and r["tries"] == len(tries)
        assert np.isnan(r["achieved_res"]).all() and np.array_equal(r["flow_vecs"], np.zeros(3))
        assert np.array_equal(r["refToNew"], tries[0]) and np.array_equal(r["aff"], P.REF_AFF)
    elif name == "single":
        assert len(tries) == 1 and np.array_equal(tries[0], np.eye(4)) and r["tries"] == 1 and r["have_one_good"]
