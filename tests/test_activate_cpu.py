"""n9 without a GPU: the C oracle of DSO's activation solve (oracle/activate_oracle.c: optimizeImmaturePoint and
linearizeResidual) equals the reference's own statements (FullSystemOptPoint.cpp:51-205, ImmaturePoint.cpp:476-543,
ResidualProjections.h:36-87, compiled unmodified by oracle/ref_build_activate.mk on points the reference itself made and
traced) bit for bit on every variant of every case of oracle/activate.py: the return, the PointHessian's idepth where one is
made, and every residual's state_state, state_energy, state_NewState and state_NewEnergy (NaN equal to NaN).  The
reference's results are in tests/golden/reference_pins_activate.npz (oracle/gen_reference_pins_activate.py).

Two return paths cannot be reached, and the coverage test does not ask for them:
- the in-loop `!isfinite(lastEnergy)` (FullSystemOptPoint.cpp:113): lastEnergy is finite once the initial test passes, and it
  is only replaced by a newEnergy with newEnergy < lastEnergy.  Every residual energy is a sum of non-negative terms
  (hw <= 1, so 2 - hw >= 1) or NaN, so such a newEnergy is finite.
- a non-finite energyTH (:175): PointHessian copies the point's energyTH, and a set keeps only points whose energyTH is
  finite (n8's add, as makeNewTraces does).  The oracle and the kernel still test it."""
import collections
import functools
import os

import numpy as np
import pytest

from oracle import activate as A

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_pins_activate.npz")


def same_bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape:
        return False
    if a.dtype.kind == "f":
        na, nb = np.isnan(a), np.isnan(b)
        return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))
    return np.array_equal(a, b)


@functools.lru_cache(maxsize=None)
def run(name):
    return A.run_oracle(A.case_inputs(name))


@pytest.mark.parametrize("name", list(A.CASES))
def test_activate_oracle_pinned_to_reference(name):
    g = np.load(GOLDEN)
    for v, (s, cf, ci, r) in enumerate(run(name)):
        pre = f"{name}_v{v}_"
        assert np.array_equal(cf, g[pre + "cand_frame"]) and np.array_equal(ci, g[pre + "cand_index"]), v
        assert np.array_equal(r["result"], g[pre + "result"]), v
        made = r["result"] == 1
        assert same_bits(np.where(made, r["idepth"], np.nan), g[pre + "idepth"]), v
        for k in ("state", "new_state"):
            assert np.array_equal(r[k], g[pre + k]), (v, k)
        for k in ("energy", "new_energy"):
            assert same_bits(r[k], g[pre + k]), (v, k)


def test_pins_reach_every_reachable_path():
    paths, flags = collections.Counter(), collections.Counter()
    min_obs2 = no_its = 0
    for name in A.CASES:
        for s, cf, ci, r in run(name):
            paths.update(r["path"].tolist())
            for bit in A.FLAGS:
                flags[bit] += int(((r["flags"] & bit) != 0).sum())
            if s["min_obs"] == 2:
                min_obs2 += int((r["path"] == 6).sum())
            if s["gn_iterations"] == 0:
                no_its += len(cf)
                assert not (r["flags"] & (1 | 2 | 4 | 8)).any()
    missing = [A.PATHS[p] for p in A.PATHS if p not in (4, 7) and paths[p] == 0]
    assert not missing, missing
    missing = [A.FLAGS[b] for b in A.FLAGS if flags[b] == 0]
    assert not missing, missing
    assert min_obs2 > 0 and no_its > 0
