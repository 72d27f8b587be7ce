"""n12 without a GPU: the C oracle of DSO's linearizeAll (oracle/linearize_oracle.c: PointFrameResidual::linearize,
applyRes, applyRes_Reductor, the reductor's fix branch and setNewFrameEnergyTH) equals the reference's own statements
(Residuals.cpp:78-274, 306-328, FullSystemOptimize.cpp:52-210, compiled unmodified by oracle/ref_build_linearize.mk) bit for
bit at every step of the optimize()-shaped sequence of oracle/linearize.py, on every variant of the window of points n9
activates on room_640x480_8f: every residual's state_NewState, state_NewEnergy, state_NewEnergyWithOutlier,
centerProjectedTo, the Jacobian records of the residuals that are not OOB, the newest frame's
frameEnergyTH, and with fixLinearization the applied states, the removed flags and the points' maxRelBaseline and numGoodResiduals; the energy to
the last bit of the reference's sequential sum.  The reference's results are in tests/golden/reference_pins_linearize.npz
(oracle/gen_reference_pins_linearize.py; float arrays as SHA-256 digests of their bytes)."""
import functools
import os

import numpy as np
import pytest

from oracle import linearize as L

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_pins_linearize.npz")


@functools.lru_cache(maxsize=None)
def run(variant):
    win = L.window("room", variant)
    o = L.LinearizeOracle(win)
    seq = L.run_sequence(o, win)
    return win, seq


def pins(g, variant, k):
    pre = f"{variant}_s{k}_"
    return {key[len(pre):]: g[key] for key in g.files if key.startswith(pre)}


@pytest.mark.parametrize("variant", list(L.VARIANTS))
def test_linearize_oracle_pinned_to_reference(variant):
    g = np.load(GOLDEN)
    win, seq = run(variant)
    assert not any(k.startswith(f"{variant}_s{len(seq)}_") for k in g.files)
    for k, (st, r, th) in enumerate(seq):
        p = pins(g, variant, k)
        assert p, k
        bad = L.compare_pins(r, p, exact_energy=True)
        assert bad == [], (k, bad)


def test_pins_reach_every_case():
    """Every variant does what it is there for: outliers and IN residuals in every step, OOB from projections and from NaN
    pixels, OOB residuals that stay OOB after apply calls, removed residuals, a newest frame without residuals (12*12*8)
    and one with them, and JabF zeroed under affine mode -1."""
    g = np.load(GOLDEN)
    _, base = run("base")
    for st, r, th in base:
        c = np.bincount(r["new_state"], minlength=3)
        assert c[L.IN] > 1000 and c[L.OUTLIER] > 100
    assert base[-1][1]["removed"].sum() > 100 and base[-1][1]["num_good_residuals"].sum() > 1000
    assert (base[-1][1]["max_rel_baseline"] > 0).sum() > 100
    assert all(r["new_frame_energy_th"] != 12 * 12 * 8 for _, r, _ in base)
    assert all(r["new_frame_energy_th"] == 12 * 12 * 8 for _, r, _ in run("no_newest")[1])
    _, sticky = run("sticky_oob")
    oob = sticky[1][1]["new_state"] == L.OOB
    assert oob.sum() > 20 and (sticky[2][1]["new_state"][oob] == L.OOB).all()
    assert (sticky[3][1]["state"][oob] == L.OOB).all() and sticky[3][1]["removed"][oob].all()
    _, nan = run("nan_pixels")
    assert (nan[0][1]["new_state"] == L.OOB).sum() > 5
    _, aff = run("affine_off")
    live = aff[0][1]["new_state"] != L.OOB
    assert (aff[0][1]["jacobians"][live][:, 46:62] == 0).all()
    assert (base[0][1]["jacobians"][live][:, 46:62] != 0).any()
    assert len(g.files) > 0
