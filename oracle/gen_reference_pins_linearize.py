"""Runs the reference's own linearizeAll, PointFrameResidual::linearize, applyRes, applyRes_Reductor and setNewFrameEnergyTH
(Residuals.cpp:78-274, 306-328, FullSystemOptimize.cpp:52-210, built by oracle/ref_build_linearize.mk) on every variant of
oracle/linearize.py's "room" window - the points n9 activates on room_640x480_8f, with their IN residuals - as the
optimize()-shaped sequence of oracle/linearize.py's steps.  Stores per variant and step the energy, the newest frame's
frameEnergyTH, every residual's state_NewState, state_NewEnergy, state_NewEnergyWithOutlier, centerProjectedTo (NaN where
linearize does not set it), and with fixLinearization the applied state_state, the removed flags and every point's maxRelBaseline
and numGoodResiduals, in tests/golden/reference_pins_linearize.npz for tests/test_linearize_cpu.py, in the form of
oracle/linearize.py's pin_record: the float arrays (the Jacobian records of the residuals that are not OOB, the energies,
the centres, maxRelBaseline) as SHA-256 digests of their bytes, so the file stays small.  Every energy the reference holds as a double is a float value, which is checked before it is stored as one.
CPU only.

    make -C oracle -f ref_build_linearize.mk REFERENCE=REFERENCE_DIR
    python oracle/gen_reference_pins_linearize.py
"""
import ctypes
import os
import sys

import numpy as np

REPO = os.path.dirname(os.path.abspath(os.path.dirname(__file__)))
sys.path.insert(0, REPO)
from oracle import linearize as L  # noqa: E402

_fp = ctypes.POINTER(ctypes.c_float)
_ip = ctypes.POINTER(ctypes.c_int)
_dp = ctypes.POINTER(ctypes.c_double)


def p(a, t=_fp):
    return a.ctypes.data_as(t)


def run_reference(lib, win):
    """The reference over steps(win): [dict of outputs per step] with the keys of LinearizeOracle.linearize."""
    seq = L.steps(win)
    n, npt, m, S = win["n_frames"], len(win["host"]), len(win["res_point"]), len(seq)
    dI = [np.ascontiguousarray(d, np.float32) for d in win["dI"]]
    arr = (_fp * n)(*[p(d) for d in dI])
    fix = np.array([s["fix"] for s in seq], np.int32)
    apply = np.array([s["apply"] for s in seq], np.int32)
    ids = np.ascontiguousarray(np.stack([s["idepth_scaled"] for s in seq]), np.float32)
    idz = np.ascontiguousarray(np.stack([s["idepth_zero_scaled"] for s in seq]), np.float32)
    pc = np.ascontiguousarray(np.stack([s["precalc"] for s in seq]), np.float32)
    o = dict(energy=np.zeros(S), new_th=np.zeros(S, np.float32), new_state=np.zeros((S, m), np.int32),
             new_energy=np.zeros((S, m)), new_energy_wo=np.zeros((S, m)), center=np.zeros((S, m, 3), np.float32),
             J=np.zeros((S, m, L.JACOBIAN_FLOATS), np.float32), state=np.zeros((S, m), np.int32), removed=np.zeros((S, m), np.int32),
             mrb=np.zeros((S, npt), np.float32), ngood=np.zeros((S, npt), np.int32))
    s8 = L.settings_array(win["settings"])
    lib.ref_lin_run(win["w"], win["h"], n, arr, p(win["calib4"]), p(s8), npt, p(win["host"], _ip), p(win["u"]), p(win["v"]),
                    p(win["color"]), p(win["weights"]), p(win["max_rel_baseline"]), p(win["num_good"], _ip), m,
                    p(win["res_point"], _ip), p(win["res_target"], _ip), S, p(fix, _ip), p(apply, _ip), p(ids), p(idz), p(pc),
                    p(win["frame_th"]), p(o["energy"], _dp), p(o["new_th"]), p(o["new_state"], _ip), p(o["new_energy"], _dp),
                    p(o["new_energy_wo"], _dp), p(o["center"]), p(o["J"]), p(o["state"], _ip), p(o["removed"], _ip), p(o["mrb"]),
                    p(o["ngood"], _ip))
    out = []
    for s in range(S):
        for k in ("new_energy", "new_energy_wo"):
            e = o[k][s]
            assert (e.astype(np.float32).astype(np.float64) == e).all(), k
        r = dict(energy=float(o["energy"][s]), new_frame_energy_th=float(o["new_th"][s]), new_state=o["new_state"][s].astype(np.int8),
                 new_energy=o["new_energy"][s].astype(np.float32), new_energy_with_outlier=o["new_energy_wo"][s].astype(np.float32),
                 center_projected_to=o["center"][s], jacobians=o["J"][s])
        if fix[s]:
            r.update(state=o["state"][s].astype(np.int8), removed=o["removed"][s].astype(np.uint8), max_rel_baseline=o["mrb"][s], num_good_residuals=o["ngood"][s])
        out.append(r)
    return out


def main():
    lib = ctypes.CDLL(os.path.join(REPO, "oracle", "_ref", "liblinearize_ref.so"))
    out = {}
    for variant in L.VARIANTS:
        win = L.window("room", variant)
        for k, r in enumerate(run_reference(lib, win)):
            pre = f"{variant}_s{k}_"
            for key, a in L.pin_record(r).items():
                out[pre + key] = a
            print(variant, k, r["energy"], r["new_frame_energy_th"], np.bincount(r["new_state"], minlength=3))
    np.savez_compressed(os.path.join(REPO, "tests", "golden", "reference_pins_linearize.npz"), **out)


if __name__ == "__main__":
    main()
