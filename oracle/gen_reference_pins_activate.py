"""Runs the reference's own optimizeImmaturePoint and linearizeResidual (FullSystemOptPoint.cpp:51-205,
ImmaturePoint.cpp:476-543, built with n8's cut of the constructor and traceOn by oracle/ref_build_activate.mk) on the cases
of oracle/activate.py: every host's points are added and traced by the reference, the fresh ones added behind them, and every
variant's candidates activated.  Stores per variant the candidates and, per candidate, the return, the PointHessian's
idepth (NaN where none is made) and every residual's state_state, state_energy, state_NewState and state_NewEnergy
(n_cand x n_frames, the host's column -1 / NaN) in tests/golden/reference_pins_activate.npz for tests/test_activate_cpu.py.
Every energy the reference holds as a double is a float value, which is checked before it is stored as one.  CPU only.

    make -C oracle -f ref_build_activate.mk REFERENCE=REFERENCE_DIR
    python oracle/gen_reference_pins_activate.py
"""
import ctypes
import os
import sys

import numpy as np

REPO = os.path.dirname(os.path.abspath(os.path.dirname(__file__)))
sys.path.insert(0, REPO)
from oracle import activate as A  # noqa: E402
from oracle import trace as T  # noqa: E402

_fp = ctypes.POINTER(ctypes.c_float)
_ip = ctypes.POINTER(ctypes.c_int)
_dp = ctypes.POINTER(ctypes.c_double)


def p(a, t=_fp):
    return a.ctypes.data_as(t)


def main():
    lib = ctypes.CDLL(os.path.join(REPO, "oracle", "_ref", "libactivate_ref.so"))
    s = T.settings_array(T.DEFAULT_SETTINGS)
    out = {}
    for name in A.CASES:
        c = A.case_inputs(name)
        w, h, n = c["w"], c["h"], len(c["frames"])
        lib.ref_act_reset()
        hosts = [f for f in c["frames"] if f["slot"] >= 0]
        for f in hosts:
            dI = np.ascontiguousarray(f["dI"], np.float32)
            lib.ref_act_add(w, h, p(dI), p(s), f["slot"], len(f["u"]), p(f["u"], _ip), p(f["v"], _ip), p(f["type"]))
        for t in c["traces"]:
            dI = np.ascontiguousarray(t["dI"], np.float32)
            for slot, (K, Kt, aff) in t["params"].items():
                K, Kt, aff = (np.ascontiguousarray(a, np.float32) for a in (K, Kt, aff))
                lib.ref_act_trace(w, h, p(dI), p(s), slot, p(K), p(Kt), p(aff))
        for f in hosts:
            dI = np.ascontiguousarray(f["dI"], np.float32)
            one = np.ones(len(f["u2"]), np.float32)
            lib.ref_act_add(w, h, p(dI), p(s), f["slot"], len(f["u2"]), p(f["u2"], _ip), p(f["v2"], _ip), p(one))
        # the candidates are chosen on the C oracle's points, which tests/test_trace_cpu.py pins to the reference's
        o = A.build_points(c)
        for f in hosts:
            assert lib.ref_act_count(f["slot"]) == len(o.pts[f["slot"]]["u"])
        dIs = [np.ascontiguousarray(f["dI"], np.float32) for f in c["frames"]]
        arr = (_fp * n)(*[p(d) for d in dIs])
        slots = np.array([f["slot"] for f in c["frames"]], np.int32)
        pc = np.ascontiguousarray(c["precalc"], np.float32)
        for v, (sover, which) in enumerate(c["variants"]):
            st = dict(A.DEFAULTS, **sover)
            cf, ci = A.candidates(c, o.pts, which)
            k = len(cf)
            r = dict(result=np.zeros(k, np.int32), idepth=np.zeros(k, np.float32), state=np.zeros((k, n), np.int32),
                     energy=np.zeros((k, n)), new_state=np.zeros((k, n), np.int32), new_energy=np.zeros((k, n)))
            lib.ref_act_activate(w, h, n, arr, p(slots, _ip), p(pc), p(c["calib4"]), ctypes.c_float(T.DEFAULT_SETTINGS["huber_th"]),
                                 ctypes.c_float(st["min_idepth_h_act"]), int(st["gn_iterations"]), k, p(cf, _ip), p(ci, _ip),
                                 int(st["min_obs"]), p(r["result"], _ip), p(r["idepth"]), p(r["state"], _ip), p(r["energy"], _dp),
                                 p(r["new_state"], _ip), p(r["new_energy"], _dp))
            assert np.isin(r["result"], [-1, 0, 1]).all()
            for key in ("energy", "new_energy"):
                e = r[key]
                assert np.array_equal(np.isnan(e), np.isnan(e.astype(np.float32))), key
                fin = ~np.isnan(e)
                assert (e[fin].astype(np.float32).astype(np.float64) == e[fin]).all(), key
                r[key] = e.astype(np.float32)
            pre = f"{name}_v{v}_"
            out[pre + "cand_frame"], out[pre + "cand_index"] = cf.astype(np.int8), ci.astype(np.int16)
            out[pre + "result"] = r["result"].astype(np.int8)
            out[pre + "idepth"] = r["idepth"]
            for key in ("state", "new_state"):
                out[pre + key] = r[key].astype(np.int8)
            for key in ("energy", "new_energy"):
                out[pre + key] = r[key]
            print(name, v, k, np.unique(r["result"], return_counts=True))
    lib.ref_act_reset()
    np.savez_compressed(os.path.join(REPO, "tests", "golden", "reference_pins_activate.npz"), **out)


if __name__ == "__main__":
    main()
