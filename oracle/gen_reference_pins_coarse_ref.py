"""Runs the reference's own makeCoarseDepthL0 body (CoarseTracker.cpp:148-374, built by oracle/ref_build_coarse_ref.mk), chained
with its dense block (:655-725, oracle/ref_build.mk), on the cases of oracle/pins_coarse_ref.py and stores what it computed in
tests/golden/reference_pins_coarse_ref.npz for tests/test_coarse_ref_cpu.py.  CPU only.

    make -C oracle -f ref_build.mk REFERENCE=REFERENCE_DIR
    make -C oracle -f ref_build_coarse_ref.mk REFERENCE=REFERENCE_DIR
    python oracle/gen_reference_pins_coarse_ref.py
"""
import os
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
from oracle import pins_coarse_ref as P  # noqa: E402
from oracle.coarse_ref import CoarseRefRef  # noqa: E402


def main():
    out = {}
    for name in P.CASES:
        (h, w), levels, gray_levels, depth, kfs = P.case_inputs(name)
        r = CoarseRefRef(w, h, levels)
        T_all = np.eye(4)
        for j, kf in enumerate(kfs):
            pc_n, T = r.set_coarse_tracking_ref(kf["points"], gray_levels, kf["rgbd"], depth if kf["dense"] else None,
                                                P.POSE_D.astype(np.float32), P.POSE_R.astype(np.float64), P.K4(h, w), kf["step"],
                                                kf["dense_only"])
            if T is not None:
                T_all = T
            res = r.result(pc_n)
            out[f"{name}_{j}_pc_n"] = np.array(pc_n, np.int32)
            for l in range(levels):
                out[f"{name}_{j}_l{l}"] = np.array(P.digest(*res[l]))
            print(name, j, pc_n)
        out[f"{name}_T"] = np.asarray(T_all, np.float64)
    np.savez_compressed(os.path.join(REPO, "tests", "golden", "reference_pins_coarse_ref.npz"), **out)


if __name__ == "__main__":
    main()
