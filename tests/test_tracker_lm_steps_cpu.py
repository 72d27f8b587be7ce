"""CPU companion of tests/test_tracker_lm_steps_gpu.py: the case list of oracle/lm_cases.py through the pinned host drivers
on the CPU trackers (oracle/tracker_oracle.c).  It checks, without a GPU, that the cases reach every branch of the LM loop
and that the drivers' trace hook changes no result."""
import numpy as np
import pytest

from oracle import lm_cases as C

_RESULT_KEYS = ("refToNew", "aff", "res", "iterations", "evaluations", "cutoff_repeat", "ok", "aborted_level", "repeated_level",
                "last_residuals", "last_flow_indicators", "achieved_res", "flow_vecs", "have_one_good", "tries", "winner")


def _flat(case, trace):
    return [r for t in trace for r in t] if case["entry"] == "new_coarse" else trace


def _run(name):
    case = C.CASES[name]
    trackers, T_true = C.oracle_trackers(case)
    trace = []
    r = C.run_host(case, trackers, T_true, trace=trace)
    n_tries = len(C.new_coarse_inputs(case, T_true)[0]) if case["entry"] == "new_coarse" else None
    return case, trackers, T_true, trace, r, C.branches(case, _flat(case, trace), r, n_tries)


def _same(a, b):
    if isinstance(a, list):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_same(a[k], b[k]) for k in a)
    return np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True)


@pytest.fixture(scope="module")
def runs():
    return {name: _run(name) for name in C.CASES}


def test_cases_reach_every_branch(runs):
    hit = {}
    for name, (_, _, _, _, _, got) in runs.items():
        print(f"{name}: {sorted(got)}")
        for b in got:
            hit.setdefault(b, []).append(name)
    missing = [b for b in C.BRANCHES if b not in hit]
    assert not missing, missing


@pytest.mark.parametrize("name", list(C.CASES))
def test_cases_take_what_they_are_named_for(runs, name):
    case, _, _, trace, r, got = runs[name]
    flat = _flat(case, trace)
    assert flat and all(t["kind"] in ("initial", "cutoff", "candidate") for t in flat)
    evals = r["evaluations"] if case["entry"] != "new_coarse" else sum(int(t["evaluations"].sum()) for t in r["per_try"])
    assert int(np.sum(evals)) == len(flat)                # one record per evaluation
    expect = {"track_max1": "stop_max_iterations_1", "track_max200": "max_iterations_200_runs", "track_limit": "lambda_floor",
              "track_fix_a": "fix_a", "track_fix_b": "fix_b", "track_fix_ab": "fix_ab", "track_no_points": "non_finite_increment",
              "track_flat": "singular_h", "pyr_repeat": "level_repeat", "pyr_abort": "abort", "pyr_affine": "affine_reject_mode",
              "pyr_offset_mode0": "affine_reject_mode0", "pyr_fix_a": "fix_a", "pyr_fix_b": "fix_b", "pyr_fix_ab": "fix_ab",
              "pyr_no_points": "non_finite_increment", "nc_retrack": "early_break"}
    if name in expect:
        assert expect[name] in got, sorted(got)
    if case["flat"]:                                      # the pose cannot move; a and b do, and everything stays finite
        assert _same(r["refToNew"], C.start_pose(case)) and np.all(np.isfinite(r["aff"]))
        assert not np.array_equal(r["aff"], C.P.REF_AFF)
    if case.get("start") == "far":
        assert np.all(np.isfinite(r["refToNew"])) and np.all(np.isfinite(r["aff"]))


@pytest.mark.parametrize("name", list(C.CASES))
def test_trace_hook_changes_no_result(runs, name):
    case, trackers, T_true, _, r, _ = runs[name]
    plain = C.run_host(case, trackers, T_true)
    for k in _RESULT_KEYS:
        if k in r:
            assert _same(plain[k], r[k]), k
    if case["entry"] == "new_coarse":
        assert _same(plain["per_try"], r["per_try"])
