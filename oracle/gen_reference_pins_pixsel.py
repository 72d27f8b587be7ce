"""Runs the reference's own PixelSelector (PixelSelector2.cpp:41-438, built by oracle/ref_build_pixsel.mk with the real
srand / rand) on the cases of oracle/pixsel.py: one selector per case, every call's makeMaps in order on the pinned pyramid of
its image.  Stores per call the selected pixels (flat indices in raster order) and their types, makeMaps' return value, the
last select's n2 / n3 / n4 and potential, whether it re-selected and currentPotential after the call; per image size a
digest and the first oracle.pixsel.PATTERN_PREFIX bytes of the selector's random pattern.  Output:
tests/golden/reference_pins_pixsel.npz for tests/test_pixsel_cpu.py and tests/test_pixsel_gpu.py.  CPU only.

    make -C oracle -f ref_build_pixsel.mk REFERENCE=REFERENCE_DIR
    python oracle/gen_reference_pins_pixsel.py
"""
import ctypes
import os
import sys

import numpy as np

REPO = os.path.dirname(os.path.abspath(os.path.dirname(__file__)))
sys.path.insert(0, REPO)
from oracle import pixsel as P  # noqa: E402
from oracle import trace as T  # noqa: E402

_fp = ctypes.POINTER(ctypes.c_float)
_ip = ctypes.POINTER(ctypes.c_int)


def p(a, t=_fp):
    return a.ctypes.data_as(t)


def main():
    lib = ctypes.CDLL(os.path.join(REPO, "oracle", "_ref", "libpixsel_ref.so"))
    lib.ref_pixsel_create.restype = ctypes.c_void_p
    for f in ("ref_pixsel_destroy", "ref_pixsel_pattern", "ref_pixsel_get_potential", "ref_pixsel_set_potential",
              "ref_pixsel_make_maps"):
        getattr(lib, f).argtypes = None
    out = {}
    sizes = set()
    for name, ((h, w), calls) in P.CASES.items():
        sel = ctypes.c_void_p(lib.ref_pixsel_create(w, h))
        if (h, w) not in sizes:
            sizes.add((h, w))
            rp = np.zeros(w * h, np.uint8)
            lib.ref_pixsel_pattern(sel, w * h, rp.ctypes.data_as(ctypes.c_void_p))
            out[f"pattern_{w}x{h}_digest"] = np.array(T.digest(rp))
            out[f"pattern_{w}x{h}_prefix"] = rp[:P.PATTERN_PREFIX].copy()
        for i, (c, g) in enumerate(zip(calls, P.case_images(name))):
            if c["pot"] is not None:
                lib.ref_pixsel_set_potential(sel, c["pot"])
            s = P.settings_array(dict(P.DEFAULTS, **c["settings"]))
            dI, ag = P.levels(g)
            dI = np.ascontiguousarray(dI, np.float32)
            ag = [np.ascontiguousarray(a, np.float32) for a in ag]
            m = np.zeros((h, w), np.float32)
            info = np.zeros(5, np.int32)
            ret = lib.ref_pixsel_make_maps(sel, w, h, p(dI), p(ag[0]), p(ag[1]), p(ag[2]), p(s), ctypes.c_float(c["density"]),
                                           int(c["rec"]), ctypes.c_float(c["th"]), p(m), p(info, _ip))
            idx, typ = P.selected(m)
            pre = f"{name}_{i}_"
            out[pre + "index"], out[pre + "type"] = idx, typ
            out[pre + "ret"] = np.int32(ret)
            out[pre + "n"] = info[:3].copy()
            out[pre + "pot_used"] = np.int32(info[3])
            out[pre + "reselected"] = np.int32(info[4] > 1)
            out[pre + "pot_after"] = np.int32(lib.ref_pixsel_get_potential(sel))
        lib.ref_pixsel_destroy(sel)
    path = os.path.join(REPO, "tests", "golden", "reference_pins_pixsel.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, len(out), "arrays")


if __name__ == "__main__":
    main()
