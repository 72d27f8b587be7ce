"""Pins against the REAL reference: the reference's own dr_fusion class and tracker kernels, compiled unmodified
(oracle/ref_build.mk) and run on an H100 by oracle/gen_reference_pins.py, computed what tests/golden/reference_pins_gpu.npz
stores; ours and the CPU oracles are compared with it here.  (The reference's DrFusion::GetMesh does not return in
minutes on an H100, so the mesh is pinned only against the CPU marching-cubes oracle, tests/test_fusion_gpu.py.)  These tests are what lifts the TSDF / tracker oracles from
"parity unpinned" to "pinned against the reference's CUDA code" (modulo the reference's documented races, SURVEY.md
Appendix B)."""
import os

import numpy as np
import pytest

from oracle import pins
from oracle.cpu import TrackerOracle, TsdfOracle
from tandem_b200 import CudaCoarseTracker, DrFusion

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ref():
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_pins_gpu.npz"))


def test_fusion_matches_reference_dr_fusion(ref):
    opt, poses, frames, _ = pins.fusion_setup(2, True)
    ours, orc = DrFusion(opt), TsdfOracle(opt)
    for k, (pose, (bgr, depth)) in enumerate(zip(poses, frames)):
        ours.IntegrateScanAsync(bgr, depth, pose)
        orc.integrate(bgr, depth, pose)
        rp = poses[max(k - 1, 0)] if k % 2 else pose
        rd, rb = ref[f"fusion_{k}_depth"], ref[f"fusion_{k}_bgr"]
        ours.RenderAsync([rp])
        (ob,), (od,) = ours.GetRenderResult()
        cb, cd = orc.render(rp)
        for name, xd, xb in (("cuda", od, ob), ("oracle", cd, cb)):
            hit_r, hit_x = rd > 0, xd > 0
            mism = float(np.mean(hit_r != hit_x))
            both = hit_r & hit_x
            err = np.abs(rd[both] - xd[both])
            print(f"frame {k} {name} vs reference: hit mismatch {mism:.5f}, depth mean-abs {err.mean():.2e}, "
                  f"max {err.max():.2e}, bit-equal {np.mean(rd == xd):.5f}, colour equal {np.mean(rb == xb):.5f}")
            # the reference itself is FMA-contracted, uses a different 4x4 inverse and sphere-traces, so "same
            # surface to a small fraction of a voxel" is the strongest statement available (voxel = 1e-2 m)
            assert mism <= 3e-3
            assert err.mean() <= 3e-4 and np.quantile(err, 0.99) <= 5e-3
            assert np.mean(np.abs(rb[both].astype(int) - xb[both].astype(int)) <= 2) > 0.98


@pytest.mark.parametrize("size,step", pins.TRACKER_CASES)
def test_tracker_matches_reference_kernels(ref, size, step):
    h, w = size
    c = pins.tracker_pin_case(size, step)
    n = c["n"]
    orc = TrackerOracle(w, h)
    orc.setK(w, h, c["fx"], c["fy"], c["cx"], c["cy"])
    orc.setReference(n, c["pc_u"], c["pc_v"], c["pc_idepth"], c["pc_color"], c["ref_exposure"], c["ref_aff"])
    orc.setNew(c["dInew"])
    ro = orc.calcRes(c["refToNew"], c["new_exposure"], c["new_aff"], c["cutoffTH"])
    Ho, bo = orc.calcG(c["new_exposure"], c["new_aff"])
    k = f"tracker_{h}x{w}_{step}"
    o7, o45 = ref[k + "_o7"], ref[k + "_o45"]
    # reference host post-processing (cuda_coarse_tracker.cpp:264-272, 335-355)
    rr = np.array([o7[0], o7[1], o7[4] / o7[6], 0, o7[5] / o7[6], o7[3] / o7[1]], np.float64)
    scale = np.array([1, 1, 1, .5, .5, .5, 10, 1000.0])
    tri = lambda r, q: min(r, q) * 9 + max(r, q) - min(r, q) * (min(r, q) + 1) // 2
    Hr = np.array([[o45[tri(r, q)] for q in range(8)] for r in range(8)], np.float64) / o7[2] * np.outer(scale, scale)
    br = np.array([o45[tri(r, 8)] for r in range(8)], np.float64) / o7[2] * scale
    g = CudaCoarseTracker(w, h)
    g.init()
    g.setK(w, h, c["fx"], c["fy"], c["cx"], c["cy"])
    g.setReference(n, c["pc_u"], c["pc_v"], c["pc_idepth"], c["pc_color"], c["ref_exposure"], c["ref_aff"])
    g.setNew(c["dInew"])
    rg, Hg, bg = g.calcResAndG(c["refToNew"], c["new_exposure"], c["new_aff"], c["cutoffTH"])
    rel = lambda a, b: np.max(np.abs(a - b)) / np.max(np.abs(b))
    for name, (r_, H_, b_) in (("cuda", (rg, Hg, bg)), ("oracle", (ro, Ho, bo))):
        print(f"{name} vs reference kernels: dE/E {abs(r_[0] - rr[0]) / rr[0]:.2e}, numE {r_[1]} vs {rr[1]}, "
              f"H rel {rel(H_, Hr):.2e}, b rel {rel(b_, br):.2e}")
        assert abs(r_[1] - rr[1]) <= 2          # the reference's own FMA contraction may flip a border point
        assert abs(r_[0] - rr[0]) <= 2e-4 * rr[0]
        assert abs(r_[2] - rr[2]) <= 1e-3 * rr[2] and abs(r_[4] - rr[4]) <= 1e-3 * rr[4]
        assert abs(r_[5] - rr[5]) <= 1e-4
        assert rel(H_, Hr) < 2e-3 and rel(b_, br) < 2e-3   # reference sums 3e5 fp32 terms with float atomics
    # per-point output on the stored seeded sample of the points
    idx = pins.warped_sample(n)
    w5, w6 = ref[k + "_warped5"], ref[k + "_warped6"]
    wo = orc.warped[:, idx]
    same = (w6 != 0) == (wo[6] != 0)
    assert same.mean() > 0.9999
    m = (w6 != 0) & (wo[6] != 0)
    assert np.quantile(np.abs(w5[m] - wo[5][m]), 0.999) < 5e-3 and np.max(np.abs(w5[m] - wo[5][m])) < 5e-2
