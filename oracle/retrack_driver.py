"""ORACLE (test infrastructure - never imported by the product).

numpy restatement of the motion-hypothesis loop of FullSystem::trackNewCoarse (tandem/src/FullSystem/FullSystem.cpp:538-617),
monocular path (rgbd_flag == false), on top of any callable with the call surface of trackNewestCoarse.  The same code drives
oracle.pyramid_driver.track_pyramid over CPU tracker oracles and tandem_b200.track_pyramid on the GPU (the host-driven
baseline of tdm_tracker_track_new_coarse, SURVEY.md section 8(f) row n6).  Statement for statement: every try starts from
lastF_2_fh_tries[i] and aff_last_2_l with minResForAbort = achievedRes as it stands (:553-559); a try wins when it is ok,
lastResiduals[0] is finite as a float and not >= achievedRes[0] (:586-592); once one has won, every level takes over the try's
lastResiduals where achievedRes is not finite (as a float) or larger (:595-602); the loop ends when achievedRes[0] <
lastCoarseRMSE[0] * setting_reTrackThreshold (:605); without a winner the pose is tries[0], aff is aff_last_2_l and the flow
(0, 0, 0) (:610-615).
PINNED: tests/test_track_new_coarse_cpu.py compares it with the reference's own lines (oracle/ref_wrap_retrack.cpp), whose
results on the cases of oracle/pins_retrack.py are stored in tests/golden/reference_pins_retrack.npz.
"""
import numpy as np


def track_new_coarse(track_pyramid, tries, aff_last_2_l, last_coarse_rmse, retrack_threshold=1.5):
    """track_pyramid(refToNew (4,4), aff (2,), min_res_for_abort (5,)) -> dict with ok, refToNew, aff, last_residuals,
    last_flow_indicators, aborted_level, repeated_level, evaluations (the fields of track_pyramid).
    tries: (n, 4, 4) lastF_2_fh_tries.  Returns dict(refToNew, aff, flow_vecs (3,), achieved_res (5,) - the caller's new
    lastCoarseRMSE -, have_one_good, tries (tryIterations), winner (index of the last winner, -1: none), per_try (list of dicts
    ok, aborted_level, repeated_level, last_residuals (5,), evaluations (5,), min_res (5,): achievedRes as the try started))."""
    tries = np.asarray(tries, np.float64).reshape(-1, 4, 4)
    aff_last_2_l = np.array(aff_last_2_l, np.float64)
    achieved = np.full(5, np.nan)
    flow, T_best, aff_best = np.full(3, 100.0), np.eye(4), np.zeros(2)
    have_one_good, winner, per_try = False, -1, []
    thresh = float(np.float32(retrack_threshold))            # setting_reTrackThreshold is a float
    for i in range(len(tries)):
        r = track_pyramid(tries[i].copy(), aff_last_2_l.copy(), achieved.copy())
        last = np.asarray(r["last_residuals"], np.float64)
        per_try.append(dict(ok=bool(r["ok"]), aborted_level=int(r["aborted_level"]), repeated_level=int(r["repeated_level"]),
                            last_residuals=last.copy(), evaluations=np.asarray(r["evaluations"], np.int32).copy(),
                            min_res=achieved.copy()))
        with np.errstate(invalid="ignore", over="ignore"):
            if r["ok"] and np.isfinite(np.float32(last[0])) and not (last[0] >= achieved[0]):
                flow = np.array(r["last_flow_indicators"], np.float64)
                aff_best, T_best = np.array(r["aff"], np.float64), np.array(r["refToNew"], np.float64)
                have_one_good, winner = True, i
            if have_one_good:
                for l in range(5):
                    if not np.isfinite(np.float32(achieved[l])) or achieved[l] > last[l]:
                        achieved[l] = last[l]
            if have_one_good and achieved[0] < float(last_coarse_rmse[0]) * thresh:
                break
    if not have_one_good:
        flow, aff_best, T_best = np.zeros(3), aff_last_2_l.copy(), tries[0].copy()
    return dict(refToNew=T_best, aff=aff_best, flow_vecs=flow, achieved_res=achieved, have_one_good=have_one_good,
                tries=len(per_try), winner=winner, per_try=per_try)
