"""Runs the reference's own ImmaturePoint constructor and traceOn (ImmaturePoint.cpp:32-61, 75-414, built by
oracle/ref_build_trace.mk) on the cases of oracle/trace.py: every host's points are added, then every frame is traced from
every host in turn.  Stores the count each add leaves and digests (oracle.trace.digest) of the point fields and of the full trace state after
every trace in tests/golden/reference_pins_trace.npz for tests/test_trace_cpu.py.  CPU only.

    make -C oracle -f ref_build_trace.mk REFERENCE=REFERENCE_DIR
    python oracle/gen_reference_pins_trace.py
"""
import ctypes
import os
import sys

import numpy as np

REPO = os.path.dirname(os.path.abspath(os.path.dirname(__file__)))
sys.path.insert(0, REPO)
from oracle import trace as T  # noqa: E402

_fp = ctypes.POINTER(ctypes.c_float)
_ip = ctypes.POINTER(ctypes.c_int)


def p(a, t=_fp):
    return a.ctypes.data_as(t)


def get(lib, slot):
    n = lib.ref_trace_count(slot)
    f = dict(u=(n,), v=(n,), type=(n,), energy_th=(n,), color=(n, 8), weights=(n, 8), grad_h=(n, 4), idepth_min=(n,),
             idepth_max=(n,), quality=(n,), uv=(n, 2), interval=(n,))
    o = {k: np.zeros(s, np.float32) for k, s in f.items()}
    o["status"] = np.zeros(n, np.int32)
    lib.ref_trace_get(slot, p(o["u"]), p(o["v"]), p(o["type"]), p(o["energy_th"]), p(o["color"]), p(o["weights"]),
                      p(o["grad_h"]), p(o["idepth_min"]), p(o["idepth_max"]), p(o["quality"]), p(o["status"], _ip), p(o["uv"]),
                      p(o["interval"]))
    return o


def main():
    lib = ctypes.CDLL(os.path.join(REPO, "oracle", "_ref", "libtrace_ref.so"))
    out = {}
    for name in T.CASES:
        c = T.case_inputs(name)
        s = T.settings_array(c["settings"])
        lib.ref_trace_reset()
        for hh in c["hosts"]:
            dI = np.ascontiguousarray(hh["dI"], np.float32)
            m = lib.ref_trace_add(c["w"], c["h"], p(dI), p(s), hh["slot"], len(hh["u"]), p(hh["u"], _ip), p(hh["v"], _ip),
                                  p(hh["type"]))
            out[f"{name}_add{hh['slot']}_n"] = np.int32(m)
            o = get(lib, hh["slot"])
            for k in T.POINT:
                out[f"{name}_add{hh['slot']}_{k}"] = np.array(T.digest(o[k]))
        for j, f in enumerate(c["frames"]):
            dI = np.ascontiguousarray(f["dI"], np.float32)
            for slot, (K, Kt, aff) in f["params"].items():
                K, Kt, aff = (np.ascontiguousarray(a, np.float32) for a in (K, Kt, aff))
                lib.ref_trace_trace(c["w"], c["h"], p(dI), p(s), slot, p(K), p(Kt), p(aff))
                o = get(lib, slot)
                for k in T.STATE:
                    out[f"{name}_t{j}_{slot}_{k}"] = np.array(T.digest(o[k]))
            print(name, j, {slot: np.bincount(get(lib, slot)["status"], minlength=6).tolist() for slot in f["params"]})
    lib.ref_trace_reset()
    np.savez_compressed(os.path.join(REPO, "tests", "golden", "reference_pins_trace.npz"), **out)


if __name__ == "__main__":
    main()
