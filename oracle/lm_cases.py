"""Cases of the LM step-by-step check (tests/test_tracker_lm_steps_cpu.py, tests/test_tracker_lm_steps_gpu.py): the device LM
loop (tdm_tracker_track, _track_pyramid, _track_new_coarse) and the pinned host drivers (oracle/lm_driver.py,
oracle/pyramid_driver.py, oracle/retrack_driver.py) run on the same evaluations, and together the cases take every branch
of the loop.  branches() reads the branches a case took from the host driver's trace; BRANCHES lists the ones the case
list as a whole must reach.

A case is a dict: entry ("track": one level of tandem_b200.synthetic.tracker_case, "pyramid": the levels of
oracle/pins_pyramid.py, "new_coarse": those levels with a try list of oracle/pins_retrack.py), size (h, w), and the inputs:
huber / cutoff (the tracker's setting_huberTH and the call's coarse cutoff), new_exposure, start (a pose name, see
start_pose), the call's options, flat (the new image is a constant: no gradients, the pose rows of H are 0) and offset
(added to the new image's intensities)."""
import numpy as np

from oracle import pins_pyramid as P
from oracle import pins_retrack as R
from oracle.lm_driver import se3_exp

DSO_MODES = dict(mode_a=1e12, mode_b=1e8)   # settings.cpp:109-110
FAR = se3_exp([0.0, 0.0, -50.0, 0.0, 0.0, 0.0])   # every point behind the camera: numTermsInE = 0 on every level


def _track(name, size=(240, 320), **kw):
    c = dict(entry="track", size=size, huber=9.0, cutoff=20.0, new_exposure=1.05, start="identity", max_iterations=10,
             limit=0.001, fix_a=False, fix_b=False, flat=False, offset=0.0)
    c.update(kw)
    return name, c


def _pyramid(name, size=(240, 320), **kw):
    c = dict(entry="pyramid", size=size, huber=9.0, cutoff=20.0, new_exposure=1.05, start="identity",
             max_iterations=(10, 20, 50, 50), limit=0.001, min_res=P.NAN5, flat=False, offset=0.0, **DSO_MODES)
    c.update(kw)
    return name, c


def _new_coarse(name, retrack_case, size=(240, 320)):
    a = R.CASES[retrack_case]["args"]
    return name, dict(entry="new_coarse", size=size, huber=9.0, cutoff=a["coarse_cutoff"], new_exposure=a["new_exposure"],
                      mode_a=a["mode_a"], mode_b=a["mode_b"], retrack_case=retrack_case, limit=0.001,
                      max_iterations=(10, 20, 50, 50), flat=False, offset=0.0)


CASES = dict([
    _track("track_320", max_iterations=10),
    _track("track_640", size=(480, 640), max_iterations=10),
    _track("track_max1", max_iterations=1),
    _track("track_max200", max_iterations=200),
    _track("track_limit", limit=0.1),                        # extrapolation from the start, a reject lands on the floor
    _track("track_fix_a", fix_a=True),
    _track("track_fix_b", fix_b=True),
    _track("track_fix_ab", fix_a=True, fix_b=True),
    _track("track_inexact", huber=9.3, cutoff=17.7, new_exposure=1.3),   # huber * cutoff products that round
    _track("track_no_points", start="far"),                  # NaN sums: the increment is not finite and is zeroed
    _track("track_flat", flat=True),                         # singular damped H: only a and b move
    _pyramid("pyr_converge"),
    _pyramid("pyr_converge_640", size=(480, 640)),
    _pyramid("pyr_repeat", cutoff=5.0),                      # cutoff doubling, the one-time level repeat
    _pyramid("pyr_repeat_640", size=(480, 640), cutoff=5.0),
    _pyramid("pyr_abort", min_res=(np.nan, np.nan, 1.0, np.nan, np.nan)),
    _pyramid("pyr_affine", new_exposure=float(np.exp(2.0))),                 # |a| > 1.2 with mode_a != 0
    _pyramid("pyr_affine_mode0", new_exposure=float(np.exp(2.0)), mode_a=0.0, mode_b=0.0),
    _pyramid("pyr_offset_mode0", offset=250.0, mode_a=0.0, mode_b=0.0),      # |b - a * b_ref| > 200 with mode_b == 0
    _pyramid("pyr_fix_a", mode_a=-1.0),
    _pyramid("pyr_fix_b", mode_b=-1.0),
    _pyramid("pyr_fix_ab", mode_a=-1.0, mode_b=-1.0),
    _pyramid("pyr_limit", limit=0.01),
    _pyramid("pyr_inexact", huber=9.3, cutoff=17.7, new_exposure=1.3),
    _pyramid("pyr_no_points", start="far"),
    _new_coarse("nc_retrack", "retrack"),
    _new_coarse("nc_retrack_640", "retrack", size=(480, 640)),
    _new_coarse("nc_exhaust", "exhaust"),
])

# stop_max_iterations_1: a pass stopped by max_iterations = 1; max_iterations_200_runs: a call with the largest bound the
# device accepts (200) ran candidates - it stops on |inc|, no case here stops at 200
BRANCHES = ("accept", "reject", "extrapolation", "lambda_floor", "stop_inc", "stop_max_iterations", "stop_max_iterations_1",
            "max_iterations_200_runs", "cutoff_doubling", "level_repeat", "abort", "affine_reject_mode", "affine_reject_mode0",
            "fix_a", "fix_b", "fix_ab", "non_finite_increment", "singular_h", "several_tries", "winner_not_first",
            "early_break")


def start_pose(case):
    return {"identity": np.eye(4), "far": FAR}[case["start"]]


def new_coarse_inputs(case, T_true):
    """(tries, last_coarse_rmse) of a new_coarse case, around the scene's true pose."""
    rc = R.CASES[case["retrack_case"]]
    return rc["tries"](T_true), np.full(5, rc["last_rmse"])


def new_image(gray, case):
    """The new frame's grey image as a case sees it."""
    g = np.asarray(gray, np.float32)
    if case["flat"]:
        g = np.full_like(g, 100.0)
    return (g + np.float32(case["offset"])).astype(np.float32)


def _level_max_iterations(case, lvl):
    its = case["max_iterations"]
    return its if np.isscalar(its) else its[lvl]


def fixed(case):
    if case["entry"] == "track":
        return case["fix_a"], case["fix_b"]
    return case["mode_a"] < 0, case["mode_b"] < 0


def branches(case, trace, result, n_tries=None):
    """The branches a case took, from the host driver's trace (a list of evaluation records) and its result."""
    got = set()
    cand = [r for r in trace if r["kind"] == "candidate"]
    if any(r["accepted"] for r in cand):
        got.add("accept")
    if any(not r["accepted"] for r in cand):
        got.add("reject")
    if any(r["extrap"] != 1.0 for r in cand):
        got.add("extrapolation")
    if any(not r["accepted"] and np.float32(r["lambda_after"]) != np.float32(r["lambda_before"]) * np.float32(4) for r in cand):
        got.add("lambda_floor")
    for r in trace:
        if r["stop"] is not None:
            got.add("stop_" + r["stop"])
            if r["stop"] == "max_iterations" and _level_max_iterations(case, r["level"]) == 1:
                got.add("stop_max_iterations_1")
    if any(r["kind"] == "cutoff" for r in trace):
        got.add("cutoff_doubling")
    if any(r["pass"] == 1 for r in trace):
        got.add("level_repeat")
    if any(r["zeroed"] for r in cand):
        got.add("non_finite_increment")
    if cand:
        if any(_level_max_iterations(case, r["level"]) == 200 for r in cand):
            got.add("max_iterations_200_runs")
        fa, fb = fixed(case)
        if fa or fb:
            got.add("fix_ab" if fa and fb else ("fix_a" if fa else "fix_b"))
    if case["flat"] and any(r["accepted"] for r in cand):
        got.add("singular_h")
    outcomes = result["per_try"] if case["entry"] == "new_coarse" else [result]
    for o in outcomes:
        if "aborted_level" in o and o["aborted_level"] >= 0:
            got.add("abort")
        if "ok" in o and not o["ok"] and o["aborted_level"] < 0:
            got.add("affine_reject_mode0" if case["mode_a"] == 0 or case["mode_b"] == 0 else "affine_reject_mode")
    if case["entry"] == "new_coarse":
        if result["tries"] > 1:
            got.add("several_tries")
        if result["winner"] > 0:
            got.add("winner_not_first")
        if n_tries is not None and result["tries"] < n_tries:
            got.add("early_break")
    return got


# ---- CPU trackers (oracle/tracker_oracle.c) on the same inputs as the device cases ----
def oracle_levels(case):
    """Per-level TrackerOracle objects of a pyramid / new_coarse case, inputs built with oracle/front_oracle.c (equal to the
    device's pyramid and dense reference bit for bit), and the scene's true pose."""
    from oracle.cpu import FrontOracle, TrackerOracle
    h, w = case["size"]
    f = FrontOracle()
    gray_n, gray_r, depth_r, T_true = P.scene(h, w)
    new_pyr = f.make_images(new_image(gray_n, case), P.LEVELS)
    ref_pyr = f.make_images(gray_r, P.LEVELS)
    K = P.intrinsics(w)
    out = []
    for l in range(P.LEVELS):
        Kl = P.level_K(l, K)
        d = np.ascontiguousarray(depth_r[::2 ** l, ::2 ** l])
        n, arrs, _ = f.dense_reference(d, np.eye(4), Kl, 1, True, None, None, np.ascontiguousarray(ref_pyr[l][0][..., 0]))
        t = TrackerOracle(w >> l, h >> l, case["huber"], case["cutoff"])
        t.setK(w >> l, h >> l, *Kl)
        t.setReference(n, *[a[:n] for a in arrs], 1.0, P.REF_AFF)
        t.setNew(new_pyr[l][0])
        out.append(t)
    return out, T_true


def track_inputs(case):
    """tandem_b200.synthetic.tracker_case at the case's size, the new image as the case sees it."""
    from tandem_b200.synthetic import tracker_case
    h, w = case["size"]
    s = w / 640.0
    c = tracker_case(H=h, W=w, fx=320.0 * s, fy=320.0 * s, cx=319.5 * s, cy=239.5 * s)
    if case["flat"] or case["offset"]:
        dI = c["dInew"].copy()
        dI[..., 0] = new_image(dI[..., 0], case)
        if case["flat"]:
            dI[..., 1:] = 0
        c["dInew"] = dI
    return c


def run_host(case, level_trackers, T_true=None, trace=None):
    """The host driver of the case's entry point over level_trackers (anything with calcRes / calcG; one per level, one for
    "track").  Returns the driver's result; trace (a list) receives its records, for new_coarse one list per try."""
    if case["entry"] == "track":
        from oracle.lm_driver import track_level0
        return track_level0(level_trackers[0], start_pose(case), P.REF_AFF, case["new_exposure"],
                            coarse_cutoff=case["cutoff"], max_iterations=case["max_iterations"],
                            lambda_extrapolation_limit=case["limit"], fix_a=case["fix_a"], fix_b=case["fix_b"], trace=trace)
    from oracle.pyramid_driver import track_pyramid
    kw = dict(coarse_cutoff=case["cutoff"], max_iterations=case["max_iterations"], lambda_extrapolation_limit=case["limit"],
              mode_a=case["mode_a"], mode_b=case["mode_b"])
    if case["entry"] == "pyramid":
        return track_pyramid(level_trackers, start_pose(case), P.REF_AFF, case["new_exposure"], 1.0, P.REF_AFF,
                             min_res_for_abort=case["min_res"], trace=trace, **kw)
    from oracle.retrack_driver import track_new_coarse
    tries, rmse = new_coarse_inputs(case, T_true)

    def tp(T, aff, min_res):
        t = None
        if trace is not None:
            t = []
            trace.append(t)
        return track_pyramid(level_trackers, T, aff, case["new_exposure"], 1.0, P.REF_AFF, min_res_for_abort=min_res, trace=t, **kw)
    return track_new_coarse(tp, tries, P.REF_AFF, rmse)


def oracle_trackers(case):
    """(TrackerOracle objects, one per level of the case, true pose) on the inputs the device case gets."""
    if case["entry"] != "track":
        return oracle_levels(case)
    from oracle.cpu import TrackerOracle
    c = track_inputs(case)
    t = TrackerOracle(c["w"], c["h"], case["huber"], case["cutoff"])
    t.setK(c["w"], c["h"], c["fx"], c["fy"], c["cx"], c["cy"])
    t.setReference(c["n"], c["pc_u"], c["pc_v"], c["pc_idepth"], c["pc_color"], c["ref_exposure"], c["ref_aff"])
    t.setNew(c["dInew"])
    return [t], c["refToNew"]
