"""Runs the reference's own motion-hypothesis loop (FullSystem.cpp:538-617 over CoarseTracker.cpp:750-936, built by
oracle/ref_build_retrack.mk) on the cases of oracle/pins_retrack.py, every level evaluated by the CPU tracker oracle, and stores
what it computed in tests/golden/reference_pins_retrack.npz for tests/test_track_new_coarse_cpu.py.  CPU only.

    make -C oracle -f ref_build_retrack.mk REFERENCE=REFERENCE_DIR
    python oracle/gen_reference_pins_retrack.py
"""
import ctypes
import os
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from oracle import pins_pyramid as P  # noqa: E402
from oracle import pins_retrack as R  # noqa: E402
from oracle.gen_reference_pins_pyramid import G, RES, dp  # noqa: E402

ip = ctypes.POINTER(ctypes.c_int)


def run_reference(trackers, tries, last_rmse, args, threshold=1.5):
    l = ctypes.CDLL(os.path.join(REPO, "oracle", "_ref", "libretrack_ref.so"))
    l.ref_track_new_coarse.restype = ctypes.c_int

    def res_cb(_, lvl, T16, expo, aff2, cut, out6):
        r = trackers[lvl].calcRes(np.array([T16[i] for i in range(16)]).reshape(4, 4), expo, np.array([aff2[0], aff2[1]]), cut)
        for i in range(6):
            out6[i] = r[i]

    def g_cb(_, lvl, T16, expo, aff2, H64, b8):
        H, b = trackers[lvl].calcG(expo, np.array([aff2[0], aff2[1]]))
        for i in range(8):
            b8[i] = b[i]
            for j in range(8):
                H64[8 * i + j] = H[i, j]
    n = len(tries)
    tr = np.ascontiguousarray(tries, np.float64).reshape(n, 16)
    rmse = np.ascontiguousarray(last_rmse, np.float64).copy()
    T, aff, flow = np.zeros(16), np.zeros(2), np.zeros(3)
    good, winner = ctypes.c_int(0), ctypes.c_int(-1)
    t_ok, t_rep, t_counts = np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros((n, 5), np.int32)
    t_T, t_aff, t_min, t_last = np.zeros((n, 16)), np.zeros((n, 2)), np.zeros((n, 5)), np.zeros((n, 5))
    cb_res, cb_g = RES(res_cb), G(g_cb)
    k = l.ref_track_new_coarse(None, cb_res, cb_g, len(trackers) - 1, tr.ctypes.data_as(dp), n, P.REF_AFF.ctypes.data_as(dp),
                               ctypes.c_float(args["new_exposure"]), ctypes.c_float(1.0), P.REF_AFF.ctypes.data_as(dp),
                               ctypes.c_float(args["coarse_cutoff"]), ctypes.c_float(args["mode_a"]), ctypes.c_float(args["mode_b"]),
                               rmse.ctypes.data_as(dp), ctypes.c_float(threshold), T.ctypes.data_as(dp), aff.ctypes.data_as(dp),
                               flow.ctypes.data_as(dp), ctypes.byref(good), ctypes.byref(winner), t_ok.ctypes.data_as(ip),
                               t_T.ctypes.data_as(dp), t_aff.ctypes.data_as(dp), t_min.ctypes.data_as(dp), t_last.ctypes.data_as(dp),
                               t_counts.ctypes.data_as(ip), t_rep.ctypes.data_as(ip))
    return dict(tries=k, achieved_res=rmse, T=T.reshape(4, 4), aff=aff, flow=flow, have_one_good=good.value, winner=winner.value,
                try_ok=t_ok[:k], try_T=t_T[:k].reshape(k, 4, 4), try_aff=t_aff[:k], try_min_res=t_min[:k], try_last_res=t_last[:k],
                try_counts=t_counts[:k], try_repeated_level=t_rep[:k])


def main():
    levels = P.level_inputs()
    out = {}
    for name in R.CASES:
        tries, rmse, args = R.case_inputs(name)
        r = run_reference(P.oracle_trackers(levels), tries, rmse, args)
        for k, v in r.items():
            out[f"{name}_{k}"] = np.asarray(v)
        print(name, {k: r[k] for k in ("tries", "winner", "have_one_good")}, "achievedRes", np.round(r["achieved_res"], 4).tolist(),
              "per-try ok", r["try_ok"].tolist())
    np.savez_compressed(os.path.join(REPO, "tests", "golden", "reference_pins_retrack.npz"), **out)


if __name__ == "__main__":
    main()
