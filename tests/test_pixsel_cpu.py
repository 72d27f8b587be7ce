"""n10 without a GPU: the C oracle of DSO's pixel selection (oracle/pixsel_oracle.c: the constructor's random pattern,
makeHists, select and makeMaps) equals the reference's own statements (PixelSelector2.cpp:41-438, compiled unmodified with the
real srand / rand by oracle/ref_build_pixsel.mk) bit for bit on every call of every case of oracle/pixsel.py: the selected
pixels and their types, the return value, the last select's n2 / n3 / n4 and potential, whether the call re-selected and
currentPotential after it.  The restated glibc generator equals the pinned pattern of every image size.  The reference's
results are in tests/golden/reference_pins_pixsel.npz (oracle/gen_reference_pins_pixsel.py)."""
import collections
import functools
import os

import numpy as np
import pytest

from oracle import pixsel as P
from oracle import trace as T

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_pins_pixsel.npz")


@functools.lru_cache(maxsize=None)
def run(name):
    return P.run_oracle(name)


@pytest.mark.parametrize("name", list(P.CASES))
def test_pixsel_oracle_pinned_to_reference(name):
    g = np.load(GOLDEN)
    for i, r in enumerate(run(name)):
        pre = f"{name}_{i}_"
        idx, typ = P.selected(r["map"])
        assert np.array_equal(idx, g[pre + "index"]) and np.array_equal(typ, g[pre + "type"]), i
        assert r["ret"] == int(g[pre + "ret"]), i
        assert np.array_equal(r["n"], g[pre + "n"]), i
        assert r["pot_used"] == int(g[pre + "pot_used"]) and r["pot_after"] == int(g[pre + "pot_after"]), i
        assert r["reselected"] == int(g[pre + "reselected"]), i
        assert r["ret"] == len(idx)


@pytest.mark.parametrize("hw", sorted({c[0] for c in P.CASES.values()}))
def test_glibc_pattern_restated(hw):
    h, w = hw
    g = np.load(GOLDEN)
    rp = P.pattern(w * h)
    assert T.digest(rp) == str(g[f"pattern_{w}x{h}_digest"])
    assert np.array_equal(rp[:P.PATTERN_PREFIX], g[f"pattern_{w}x{h}_prefix"])


def test_pins_reach_every_path():
    seen = collections.Counter()
    sizes = set()
    for name, ((h, w), calls) in P.CASES.items():
        sizes.add((w, h))
        prev_after = None
        for c, r in zip(calls, run(name)):
            have = int(r["n"].sum())
            q = np.float32(c["density"]) / np.float32(have) if have else (np.inf if c["density"] > 0 else np.nan)
            seen["keep"] += not r["reselected"]
            seen["re-select down"] += r["reselected"] and r["pot_used"] < r["pot_before"]
            seen["re-select up"] += r["reselected"] and r["pot_used"] > r["pot_before"]
            seen["pot 1 floor"] += c["rec"] > r["selects"] - 1 and r["pot_used"] == 1 and q > 1.25
            seen["recursions 0"] += c["rec"] == 0
            seen["recursions 2"] += c["rec"] == 2
            seen["subsample"] += bool(q < 0.95) and r["ret"] < have
            seen["no subsample"] += not q < 0.95 and have > 0
            seen["thFactor 2 at potential 3"] += c["th"] == 2.0 and r["pot_used"] == 3
            seen["direction distribution off"] += c["settings"].get("select_direction_distribution", 1) == 0 and have > 0
            seen["direction-dependent cells"] += r["nonuniform"] > 0
            seen["tied maxima"] += r["ties"] > 0
            seen["flat image"] += c["img"][0] == "flat"
            seen["numHave 0"] += have == 0
            seen["NaN pixels"] += "nan" in c["img"][0] and have > 0
            seen["density 0"] += c["density"] == 0 and have > 0
            seen["NaN quotia"] += bool(np.isnan(q))
            seen["partial blocks"] += have > 0 and (w % (4 * r["pot_used"]) != 0 or h % (4 * r["pot_used"]) != 0)
            if c["pot"] is None and prev_after is not None:
                assert r["pot_before"] == prev_after
                seen["potential carried"] += 1
            prev_after = r["pot_after"]
    missing = [k for k in ("keep", "re-select down", "re-select up", "pot 1 floor", "recursions 0", "recursions 2", "subsample",
                           "no subsample", "thFactor 2 at potential 3", "direction distribution off", "direction-dependent cells",
                           "tied maxima", "flat image", "numHave 0", "NaN pixels", "density 0", "NaN quotia", "partial blocks",
                           "potential carried") if seen[k] == 0]
    assert not missing, missing
    assert {(640, 480), (752, 480), (331, 247)} <= sizes
    # both tail reads: level 2's last row is read at every size; thsSmoothed beyond w32 * h32 iff w % 32 >= 6 or h % 32 >= 4
    assert 752 % 32 >= 6 and 331 % 32 >= 6 and 247 % 32 >= 4 and not (640 % 32 >= 6 or 480 % 32 >= 4)
    assert len(P.CASES["room_640x480_sequence"][1]) >= 5
