"""Runs the reference's own photometric undistortion, remap, BGR remap, setGammaFunction and makeImages (built by
oracle/ref_build_undistort.mk) on the cases of oracle/undistort.py, and the reference's own PixelSelector (built by
oracle/ref_build_pixsel.mk) on the gamma-weighted pyramids of the cases with `select`.  Stores per case: valid, getG(), the
Binv sequence given to setGammaFunction and B after it; per frame: exposure_time, the undistorted image, the BGR remap and
the digests (oracle.trace.digest) of every pyramid level's (I, dx, dy) and absSquaredGrad - the image and the BGR remap as
full arrays for small cases, as digests for the others; per selected frame the selected pixels and types of makeMaps (density 1500, one recursion, thFactor 1, a new selector).
Output: tests/golden/reference_pins_undistort.npz for tests/test_undistort_cpu.py and tests/test_undistort_gpu.py.  CPU only.

    make -C oracle -f ref_build_undistort.mk REFERENCE=REFERENCE_DIR CXX=g++
    make -C oracle -f ref_build_pixsel.mk REFERENCE=REFERENCE_DIR
    python oracle/gen_reference_pins_undistort.py
"""
import ctypes
import os
import sys
import tempfile

import numpy as np

REPO = os.path.dirname(os.path.abspath(os.path.dirname(__file__)))
sys.path.insert(0, REPO)
from oracle import pixsel as P  # noqa: E402
from oracle import undistort as U  # noqa: E402

_fp = ctypes.POINTER(ctypes.c_float)
_ip = ctypes.POINTER(ctypes.c_int)
_up = ctypes.POINTER(ctypes.c_ubyte)
_sp = ctypes.POINTER(ctypes.c_ushort)
SELECT = dict(density=1500.0, rec=1, th=1.0)


def p(a, t=_fp):
    return None if a is None else a.ctypes.data_as(t)


def store(out, key, a, full):
    if full:
        out[key] = np.asarray(a).copy()
    else:
        out[key + "_digest"] = np.array(U.digest(a))


def select(lib, w, h, levels):
    sel = ctypes.c_void_p(lib.ref_pixsel_create(w, h))
    dI = np.ascontiguousarray(levels[0][0], np.float32)
    ag = [np.ascontiguousarray(levels[l][1], np.float32) for l in range(3)]
    m = np.zeros((h, w), np.float32)
    info = np.zeros(5, np.int32)
    ret = lib.ref_pixsel_make_maps(sel, w, h, p(dI), p(ag[0]), p(ag[1]), p(ag[2]), p(P.settings_array(P.DEFAULTS)),
                                   ctypes.c_float(SELECT["density"]), SELECT["rec"], ctypes.c_float(SELECT["th"]), p(m),
                                   p(info, _ip))
    lib.ref_pixsel_destroy(sel)
    return ret, m


def main():
    lib = ctypes.CDLL(os.path.join(REPO, "oracle", "_ref", "libundistort_ref.so"))
    lib.ref_und_create.restype = ctypes.c_void_p
    for f in ("ref_und_destroy", "ref_und_get_gamma", "ref_und_set_gamma", "ref_und_frame"):
        getattr(lib, f).argtypes = None
    pix = ctypes.CDLL(os.path.join(REPO, "oracle", "_ref", "libpixsel_ref.so"))
    pix.ref_pixsel_create.restype = ctypes.c_void_p
    out = {}
    tmp = tempfile.mkdtemp()
    for name, c in U.CASES.items():
        cam = U.camera(name)
        full = U.full(name)
        r, v = cam["response"], cam["vignette"]
        u = ctypes.c_void_p(lib.ref_und_create(c["w_org"], c["h_org"], c["w"], c["h"], p(cam["remap_x"]), p(cam["remap_y"]), p(r),
                                               0 if r is None else r.size, p(v, _sp), 8 if c["vig"] == "v8" else 16, c["mode"],
                                               c["use_exposure"], c["gamma_weights"],
                                               os.path.join(tmp, name + ".txt").encode()))
        G = np.zeros(256, np.float32)
        G_member = np.zeros(256, np.float32)
        valid = lib.ref_und_get_gamma(u, p(G), p(G_member))
        out[f"{name}_valid"] = np.int32(valid)
        if valid:
            out[f"{name}_G"] = G
        B = np.arange(256, dtype=np.float32)
        for k, kind in enumerate(c["gammas"]):
            b = U.binv(kind, G_member)
            lib.ref_und_set_gamma(u, p(b), p(B))
            out[f"{name}_binv{k}"] = b
        out[f"{name}_B"] = B.copy()
        for k, (exposure, factor, _) in enumerate(c["frames"]):
            gray, bgr = U.frame_inputs(name, k)
            levels = c["levels"]
            tot = sum((c["w"] >> l) * (c["h"] >> l) for l in range(levels))
            img = np.zeros((c["h"], c["w"]), np.float32)
            t = np.zeros(1, np.float32)
            bo = np.zeros((c["h"], c["w"], 3), np.uint8)
            dI = np.zeros(3 * tot, np.float32)
            ag = np.zeros(tot, np.float32)
            lib.ref_und_frame(u, p(gray, _up), ctypes.c_float(exposure), ctypes.c_float(factor), p(bgr, _up), levels, p(img), p(t),
                              p(bo, _up), p(dI), p(ag))
            pre = f"{name}_f{k}_"
            out[pre + "exposure_time"] = t[0]
            store(out, pre + "image", img, full)
            store(out, pre + "bgr", bo, full)
            off = 0
            lv = []
            for l in range(levels):
                wl, hl = c["w"] >> l, c["h"] >> l
                d, a = dI[3 * off:3 * (off + wl * hl)].reshape(hl, wl, 3), ag[off:off + wl * hl].reshape(hl, wl)
                store(out, pre + f"dI{l}", d, False)
                store(out, pre + f"ag{l}", a, False)
                lv.append((d, a))
                off += wl * hl
            if c["select"] and k == 0:
                ret, m = select(pix, c["w"], c["h"], lv)
                idx, typ = P.selected(m)
                out[pre + "select_ret"] = np.int32(ret)
                out[pre + "select_index"], out[pre + "select_type"] = idx, typ
        lib.ref_und_destroy(u)
    path = os.path.join(REPO, "tests", "golden", "reference_pins_undistort.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, len(out), "arrays")


if __name__ == "__main__":
    main()
