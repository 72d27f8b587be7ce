"""Runs the reference's own coarse-to-fine body (CoarseTracker.cpp:750-936, built by oracle/ref_build_pyramid.mk) on the cases
of oracle/pins_pyramid.py, every level evaluated by the CPU tracker oracle, and stores what it computed in
tests/golden/reference_pins_pyramid.npz for tests/test_track_pyramid_cpu.py.  CPU only.

    make -C oracle -f ref_build_pyramid.mk REFERENCE=REFERENCE_DIR
    python oracle/gen_reference_pins_pyramid.py
"""
import ctypes
import os
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from oracle import pins_pyramid as P  # noqa: E402

dp = ctypes.POINTER(ctypes.c_double)
RES = ctypes.CFUNCTYPE(None, ctypes.c_void_p, ctypes.c_int, dp, ctypes.c_float, dp, ctypes.c_float, dp)
G = ctypes.CFUNCTYPE(None, ctypes.c_void_p, ctypes.c_int, dp, ctypes.c_float, dp, dp, dp)


def run_reference(trackers, case, T0, aff0):
    l = ctypes.CDLL(os.path.join(REPO, "oracle", "_ref", "libpyramid_ref.so"))
    l.ref_track_pyramid.restype = ctypes.c_int

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
    T = np.ascontiguousarray(T0, np.float64).copy()
    aff = np.array(aff0, np.float64).copy()
    last_res, flow = np.zeros(5), np.zeros(3)
    counts = np.zeros(5, np.int32)
    rep = ctypes.c_int(-1)
    min_res = np.ascontiguousarray(case["min_res"], np.float64)
    ok = l.ref_track_pyramid(None, RES(res_cb), G(g_cb), len(trackers) - 1, T.ctypes.data_as(dp), aff.ctypes.data_as(dp),
                             ctypes.c_float(case["new_exposure"]), ctypes.c_float(1.0), P.REF_AFF.ctypes.data_as(dp),
                             ctypes.c_float(case["coarse_cutoff"]), ctypes.c_float(case["mode_a"]), ctypes.c_float(case["mode_b"]),
                             min_res.ctypes.data_as(dp), last_res.ctypes.data_as(dp), flow.ctypes.data_as(dp),
                             counts.ctypes.data_as(ctypes.POINTER(ctypes.c_int)), ctypes.byref(rep))
    return dict(ok=ok, T=T, aff=aff, last_res=last_res, flow=flow, counts=counts, repeated_level=rep.value)


def main():
    levels = P.level_inputs()
    out = {}
    for name, case in P.CASES.items():
        r = run_reference(P.oracle_trackers(levels), case, np.eye(4), P.REF_AFF)
        for k, v in r.items():
            out[f"{name}_{k}"] = np.asarray(v)
        print(name, {k: (v if np.ndim(v) == 0 else np.round(np.asarray(v, np.float64), 4).tolist()) for k, v in r.items() if k != "T"})
    np.savez_compressed(os.path.join(REPO, "tests", "golden", "reference_pins_pyramid.npz"), **out)


if __name__ == "__main__":
    main()
