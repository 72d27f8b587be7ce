"""n13's oracle on the CPU: its float-tier mode equals the reference's own compiled accumulators (tests/golden/
reference_pins_accumulate.npz) bit for bit; the reference's float tiers and the double sums the device is held to agree within the float
worst case, the bound the device is held to is not vacuous (the two modes differ), the LF part of the top system is the
priors alone, and the stitch is symmetric where the reference makes it so."""
import os

import numpy as np
import pytest

from oracle import accumulate as A
from oracle import linearize as L


def applied(name):
    win = A.case(name)
    o = A.AccumulateOracle(win)
    st = L.steps(win)[0]
    o.linearize(st["idepth_scaled"], st["idepth_zero_scaled"], A.precalc(win), win["frame_th"], 0)
    o.apply_res()
    return win, o, A.inputs(win)


@pytest.mark.parametrize("name", ["room", "seeded_n2", "seeded_clamp"])
def test_tiers_and_double_agree_within_the_float_bound(name):
    win, o, inp = applied(name)
    t, d, ab = o.accumulate(inp, A.TIERS), o.accumulate(inp, A.DOUBLE), o.accumulate(inp, A.ABS)
    for k in ("top", "acc_e", "acc_eb", "acc_d", "hcc", "bc"):
        n = ab["raw"]["top_num"].max() if k != "acc_d" else ab["raw"]["d_num"].max()
        n = max(n, ab["raw"]["n_points_active"])
        assert (np.abs(t["raw"][k] - d["raw"][k]) <= n * 2.0 ** -24 * ab["raw"][k]).all(), k
    # the float tiers differ from the double sum, the double bound is far tighter than their difference
    diff = np.abs(t["raw"]["top"] - d["raw"]["top"])
    assert diff.max() > 0
    bar = A.summation_bars(ab["raw"])["top"]
    assert (diff > bar).any()
    # per-point values do not depend on the mode
    for k in ("hdi", "idepth_hessian", "bd_sum", "hcd"):
        assert L.same_bits(t[k], d[k]), k
    assert t["n_active"] == d["n_active"] == int(o.active.sum())


def test_lf_part_is_the_priors_alone():
    win, o, inp = applied("room")
    d = o.accumulate(inp, A.DOUBLE)
    zero = {k: np.zeros_like(v) for k, v in d["raw"].items() if isinstance(v, np.ndarray)}
    zero["n_points_active"] = 0
    s = A.stitch(zero, inp, win["n_frames"])
    dim = 8 * win["n_frames"] + 4
    H = np.zeros((dim, dim))
    H[np.arange(4), np.arange(4)] = inp["c_prior"]
    H[np.arange(4, dim), np.arange(4, dim)] = inp["frame_prior"].ravel()
    b = np.concatenate([inp["c_prior"] * inp["c_delta"].astype(np.float64), (inp["frame_prior"] * inp["frame_delta_prior"]).ravel()])
    assert np.array_equal(s["H_top"], H) and np.array_equal(s["b_top"], b)
    assert not s["H_sc"].any() and not s["b_sc"].any()


def test_points_without_active_residuals_and_the_clamp():
    win, o, inp = applied("seeded_clamp")
    d = o.accumulate(inp, A.DOUBLE)
    assert (d["hdi"] == 0).sum() > 0 and (d["idepth_hessian"] == np.float32(1e-10)).sum() > 0
    assert (d["hdi"][d["idepth_hessian"] == np.float32(1e-10)] == np.float32(1.0 / np.float32(1e-10))).all()
    # the transposed copies: every off-diagonal frame block and the calibration rows equal their mirror bit for bit
    H, n = d["H_top"], win["n_frames"]
    assert np.array_equal(H[:4, 4:], H[4:, :4].T)
    for a in range(n):
        for b in range(a + 1, n):
            assert np.array_equal(H[4 + 8 * a:12 + 8 * a, 4 + 8 * b:12 + 8 * b], H[4 + 8 * b:12 + 8 * b, 4 + 8 * a:12 + 8 * a].T)


GOLDEN = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden", "reference_pins_accumulate.npz")


@pytest.mark.parametrize("name", list(A.CASES))
def test_tiers_mode_equals_the_reference_pins(name):
    """The oracle's TIERS mode gives the reference's own accumulateAF/LF/SCF_MT and resubstituteF_MT outputs bit for bit
    (oracle/gen_reference_pins_accumulate.py) at every accumulate of the pinned sequence."""
    g = np.load(GOLDEN)
    win = A.case(name)
    o = A.AccumulateOracle(win)
    inp = A.inputs(win)
    recs = A.pin_sequence(o, inp, lambda: o.accumulate(inp, A.TIERS), o.resubstitute)
    assert len(recs) == 4
    for k, r in enumerate(recs):
        pre = f"{name}_a{k}_"
        pins = {key[len(pre):]: g[key] for key in g.files if key.startswith(pre)}
        got = A.pin_record(r)
        assert set(got) == set(pins), (k, set(got) ^ set(pins))
        bad = [key for key in pins if not np.array_equal(got[key], pins[key])]
        assert bad == [], (k, bad)
