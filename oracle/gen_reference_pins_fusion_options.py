"""Runs the reference's own DrFusion (built into oracle/_ref/ by oracle/ref_build.mk) at two of the option cases of
oracle/fusion_options.py - the reference's example configuration and the anisotropic, odd-sized one - and stores its renders
under tests/golden/, so that tests/test_fusion_options_gpu.py can pin the CPU oracle and the device at those options on
any checkout.  Needs a CUDA device (the stored file was made on an H100).

    make -C oracle -f ref_build.mk REFERENCE=REFERENCE_DIR
    python oracle/gen_reference_pins_fusion_options.py [OUT.npz]   # default tests/golden/reference_pins_fusion_options.npz

The reference is never given NaN depth: its allocation DDA has no step guard and does not return on a NaN pixel.
"""
import ctypes
import os
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from oracle import fusion_options as FO  # noqa: E402

REF_DIR = os.path.join(REPO, "oracle", "_ref")
OUT = os.path.join(REPO, "tests", "golden", "reference_pins_fusion_options.npz")
PIN_CASES = ("ref_example", "aniso_odd")
# The reference also integrates its FREE hash entries, all aliased to block (0,0,0) (oracle/pins.py::fusion_setup): this
# shift keeps the origin far outside the map, and is no multiple of either case's block size.
PIN_SHIFT = np.float32([2.537, 2.489, 2.529])


def pin_inputs(name):
    """(scans, render pose after each scan): the first scan's pose after the first two scans (the second overlaps it), the
    second scan's pose after the third, the 90-degree axis-aligned view after the last."""
    sc = FO.scans(name, PIN_SHIFT)
    rp = [sc[0][2], sc[0][2], sc[1][2], FO.views(PIN_SHIFT)["axis_rot90"]]
    assert len(rp) == len(sc)
    return sc, rp


def main(out=OUT):
    _fp = ctypes.POINTER(ctypes.c_float)
    l = ctypes.CDLL(os.path.join(REF_DIR, "libdr_fusion_ref.so"))
    l.ref_fusion_create.restype = ctypes.c_void_p
    res = {}
    for name in PIN_CASES:
        opt = FO.options(name)
        H, W = opt.height, opt.width
        sc, rp = pin_inputs(name)
        ref = ctypes.c_void_p(l.ref_fusion_create(ctypes.byref(opt)))
        for k, ((bgr, depth, pose), q) in enumerate(zip(sc, rp)):
            assert np.isfinite(depth).all()
            b, d = np.ascontiguousarray(bgr), np.ascontiguousarray(depth)
            l.ref_fusion_integrate(ref, ctypes.c_void_p(b.ctypes.data), d.ctypes.data_as(_fp), np.ascontiguousarray(pose).ctypes.data_as(_fp))
            rb = np.zeros((H, W, 3), np.uint8)
            rd = np.zeros((H, W), np.float32)
            q = np.ascontiguousarray(q, np.float32)
            l.ref_fusion_render(ref, q.ctypes.data_as(_fp), ctypes.c_void_p(rb.ctypes.data), rd.ctypes.data_as(_fp), H * W)
            res[f"{name}_{k}_depth"], res[f"{name}_{k}_bgr"] = rd, rb
            print(f"{name} scan {k}: reference render covers {np.mean(rd > 0):.3f} of the pixels")
        l.ref_fusion_destroy(ref)
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
    np.savez_compressed(out, **res)


if __name__ == "__main__":
    main(*sys.argv[1:2])
