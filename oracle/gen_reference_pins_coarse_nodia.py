"""Runs the reference's own makeCoarseDepthL0 body (CoarseTracker.cpp:148-374) with its pc_*_nodia arrays kept across a case's
keyframes, and its get_idepth_quantile (tandem_backend.cpp:354-361), both built by oracle/ref_build_coarse_nodia.mk, on the cases
of oracle/pins_coarse_ref.py.  Stores pc_n_nodia, a digest of the four nodia arrays (slot pc_n_nodia included) and the
quantile at the fractions of oracle.coarse_nodia.fractions in tests/golden/reference_pins_coarse_nodia.npz for
tests/test_coarse_nodia_cpu.py.  CPU only.

    make -C oracle -f ref_build_coarse_nodia.mk REFERENCE=REFERENCE_DIR
    python oracle/gen_reference_pins_coarse_nodia.py
"""
import os
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from oracle import pins_coarse_ref as P  # noqa: E402
from oracle.coarse_nodia import CoarseNodiaRef, fractions  # noqa: E402


def main():
    out = {}
    for name in P.CASES:
        (h, w), levels, gray_levels, _, kfs = P.case_inputs(name)
        r = CoarseNodiaRef(w, h, levels)
        for j, kf in enumerate(kfs):
            m = r.make(kf["points"], gray_levels, kf["rgbd"])
            fr = fractions(m)
            q = np.stack([r.quantile(m, f) for f in fr])
            out[f"{name}_{j}_n"] = np.array(m, np.int32)
            out[f"{name}_{j}_arrays"] = np.array(P.digest(*r.result(m + 1)))
            out[f"{name}_{j}_fractions"] = fr
            out[f"{name}_{j}_quantile"] = q
            print(name, j, m, q.tolist())
    np.savez_compressed(os.path.join(REPO, "tests", "golden", "reference_pins_coarse_nodia.npz"), **out)


if __name__ == "__main__":
    main()
