"""ORACLE (test infrastructure - never imported by the product).

numpy restatement of the coarse-to-fine body of CoarseTracker::trackNewestCoarse (tandem/src/FullSystem/CoarseTracker.cpp:750-936)
on top of one tracker object per pyramid level with the CudaCoarseTracker call surface (calcRes / calcG).  Each pass over a
level is oracle/lm_driver.track_level0 (the level loop :761-916, already pinned to the reference).  Around it, statement for
statement: lastResiduals[lvl] = sqrtf((float)(E / numTermsInE)) and lastFlowIndicators = resOld[2:5] (:906-907), return false
before the output pose is written when lastResiduals[lvl] > 1.5 * minResForAbort[lvl] (:908), the one-time repeat of a level
whose cutoff had to be raised (:911-915), then the affine checks with the float modes (:923-931) and a / b reported as 0 when
their mode is < 0 (:933-934).  SURVEY.md section 8(f) row n5 moves this loop onto the device (tdm_tracker_track_pyramid).
PINNED: tests/test_track_pyramid_cpu.py compares it with the reference's own body (oracle/ref_wrap_pyramid.cpp), whose results
on the cases of oracle/pins_pyramid.py are stored in tests/golden/reference_pins_pyramid.npz.
"""
import numpy as np

from oracle.lm_driver import track_level0

MAX_ITERATIONS = (10, 20, 50, 50, 50)   # CoarseTracker.cpp:751


def track_pyramid(trackers_per_level, refToNew, aff, new_exposure, ref_exposure, ref_aff, coarse_cutoff=20.0,
                  max_iterations=MAX_ITERATIONS, lambda_extrapolation_limit=0.001, mode_a=0.0, mode_b=0.0,
                  min_res_for_abort=None):
    """trackers_per_level[l] evaluates pyramid level l; len - 1 is the coarsest level.  Returns dict(ok, refToNew, aff,
    last_residuals (5,), last_flow_indicators (3,), aborted_level, repeated_level, iterations (5,), evaluations (5,),
    cutoff_repeat (5,)) - the fields of tdm_track_pyramid_result."""
    T0, a0 = np.array(refToNew, np.float64), np.array(aff, np.float64)
    T, a = T0.copy(), a0.copy()
    min_res = np.full(5, np.nan) if min_res_for_abort is None else np.asarray(min_res_for_abort, np.float64)
    last_res, flow = np.full(5, np.nan), np.full(3, 1000.0)
    its, evs, reps = np.zeros(5, np.int32), np.zeros(5, np.int32), np.ones(5, np.float32)
    out = dict(last_residuals=last_res, iterations=its, evaluations=evs, cutoff_repeat=reps, aborted_level=-1, repeated_level=-1)
    lvl = len(trackers_per_level) - 1
    while lvl >= 0:
        r = track_level0(trackers_per_level[lvl], T, a, new_exposure, coarse_cutoff=coarse_cutoff,
                         max_iterations=max_iterations[lvl], lambda_extrapolation_limit=lambda_extrapolation_limit,
                         fix_a=mode_a < 0, fix_b=mode_b < 0)
        T, a = r["refToNew"], r["aff"]
        its[lvl] += r["iterations"]
        evs[lvl] += r["evaluations"]
        reps[lvl] = max(reps[lvl], r["cutoff_repeat"])
        res = r["res"]
        with np.errstate(invalid="ignore", divide="ignore"):
            last_res[lvl] = float(np.sqrt(np.float32(res[0] / res[1])))
        flow = np.array(res[2:5], np.float64)
        out["last_flow_indicators"] = flow
        if last_res[lvl] > 1.5 * min_res[lvl]:
            out.update(ok=False, refToNew=T0, aff=a0, aborted_level=lvl)
            return out
        if r["cutoff_repeat"] > 1 and out["repeated_level"] < 0:
            out["repeated_level"] = lvl
            continue
        lvl -= 1
    out["last_flow_indicators"] = flow
    ok = not ((mode_a != 0 and float(abs(np.float32(a[0]))) > 1.2) or (mode_b != 0 and float(abs(np.float32(a[1]))) > 200))
    if ok:
        eF, eT = np.float32(ref_exposure), np.float32(new_exposure)
        if eF == 0 or eT == 0:
            eF = eT = np.float32(1)
        ra = np.exp(a[0] - ref_aff[0]) * float(eT) / float(eF)
        rb = a[1] - ra * ref_aff[1]
        with np.errstate(divide="ignore", invalid="ignore"):
            l0 = float(abs(np.log(np.float32(ra))))
        ok = not ((mode_a == 0 and l0 > 1.5) or (mode_b == 0 and float(abs(np.float32(rb))) > 200))
    if ok:
        a = a.copy()
        if mode_a < 0:
            a[0] = 0
        if mode_b < 0:
            a[1] = 0
    out.update(ok=ok, refToNew=T, aff=a)
    return out
