"""Runs the reference's own takeDataF, accumulateAF_MT, accumulateLF_MT, accumulateSCF_MT and resubstituteF_MT (single-thread
branches, built by oracle/ref_build_accumulate.mk) on every case of oracle/accumulate.py as the optimize()-shaped sequence of
accumulate.pin_sequence, and stores per case and accumulate H_top = HA_top + HL_top, b_top, H_sc, b_sc, every point's HdiF
and idepth_hessian, resInA and the resubstituted steps, in tests/golden/reference_pins_accumulate.npz for
tests/test_accumulate_cpu.py, as SHA-256 digests of the arrays' bytes (accumulate.pin_record).  The Jacobians the reference
takes are those of oracle/linearize_oracle.c, itself pinned to the reference's linearize by tests/test_linearize_cpu.py.
CPU only.

    make -C oracle -f ref_build_accumulate.mk REFERENCE=REFERENCE_DIR
    python oracle/gen_reference_pins_accumulate.py
"""
import ctypes
import os
import sys

import numpy as np

REPO = os.path.dirname(os.path.abspath(os.path.dirname(__file__)))
sys.path.insert(0, REPO)
from oracle import accumulate as A  # noqa: E402

_fp = ctypes.POINTER(ctypes.c_float)
_ip = ctypes.POINTER(ctypes.c_int)
_dp = ctypes.POINTER(ctypes.c_double)


def p(a, t=_fp):
    return a.ctypes.data_as(t)


class Reference:
    """The reference's accumulate / resubstitute over an AccumulateOracle's taken data."""

    def __init__(self, lib, o, inp):
        self.lib, self.o, self.inp = lib, o, inp
        self.x = None

    def run(self, x):
        W, inp = self.o.win, self.inp
        n, npt, m = W["n_frames"], len(W["host"]), len(W["res_point"])
        dim = 8 * n + 4
        out = {k: np.zeros((dim, dim)) for k in ("HA", "HL", "H_sc")}
        out.update({k: np.zeros(dim) for k in ("bA", "bL", "b_sc")})
        out.update(hdi=np.zeros(npt, np.float32), idepth_hessian=np.zeros(npt, np.float32), step=np.zeros(npt, np.float32))
        mrb = np.ascontiguousarray(W["max_rel_baseline"], np.float32).copy()
        f64 = lambda a: np.ascontiguousarray(a, np.float64)
        na = self.lib.ref_acc_run(n, npt, p(W["host"], _ip), m, p(W["res_point"], _ip), p(W["res_target"], _ip), p(self.o.Jt),
                                  p(np.ascontiguousarray(self.o.active, np.int32), _ip), p(A._c_layout(inp["ad_host"], n), _dp),
                                  p(A._c_layout(inp["ad_target"], n), _dp), p(f64(inp["frame_prior"]), _dp),
                                  p(f64(inp["frame_delta_prior"]), _dp), p(f64(inp["c_prior"]), _dp),
                                  p(np.ascontiguousarray(inp["c_delta"], np.float32)), p(np.ascontiguousarray(inp["point_prior"], np.float32)),
                                  p(np.ascontiguousarray(inp["point_delta"], np.float32)), p(f64(x), _dp), p(out["HA"], _dp),
                                  p(out["bA"], _dp), p(out["HL"], _dp), p(out["bL"], _dp), p(out["H_sc"], _dp), p(out["b_sc"], _dp),
                                  p(out["hdi"]), p(out["idepth_hessian"]), p(mrb), p(out["step"]))
        return dict(H_top=out["HA"] + out["HL"], b_top=out["bA"] + out["bL"], H_sc=out["H_sc"], b_sc=out["b_sc"], hdi=out["hdi"],
                    idepth_hessian=out["idepth_hessian"], n_active=na, step=out["step"])

    def accumulate(self):
        self.last = self.run(np.zeros(8 * self.o.win["n_frames"] + 4))
        return {k: v for k, v in self.last.items() if k != "step"}

    def resubstitute(self, x):
        return self.run(x)["step"]   # the accumulators of the same taken data, then resubstituteF_MT(x)


def main():
    lib = ctypes.CDLL(os.path.join(REPO, "oracle", "_ref", "libaccumulate_ref.so"))
    out = {}
    for name in A.CASES:
        win = A.case(name)
        o = A.AccumulateOracle(win)
        inp = A.inputs(win)
        ref = Reference(lib, o, inp)
        for k, r in enumerate(A.pin_sequence(o, inp, ref.accumulate, ref.resubstitute)):
            for key, v in A.pin_record(r).items():
                out[f"{name}_a{k}_{key}"] = v
    np.savez_compressed(os.path.join(REPO, "tests", "golden", "reference_pins_accumulate.npz"), **out)
    print(len(out), "arrays")


if __name__ == "__main__":
    main()
