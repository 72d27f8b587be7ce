"""n11 without a GPU: the C oracle of DSO's per-frame input (oracle/undistort_oracle.c: PhotometricUndistorter's constructor
and processFrame, Undistort::undistort's remap, the BGR remap, setGammaFunction and the gamma-weighted makeImages) equals the
reference's own statements (compiled unmodified by oracle/ref_build_undistort.mk) bit for bit on every frame of every case of
oracle/undistort.py: getG and valid, B after the case's setGammaFunction calls, exposure_time, the image, the BGR remap and
every pyramid level's (I, dx, dy) and absSquaredGrad.  The oracle's gamma-weighted pyramids, fed to the pixel-selection
oracle (oracle/pixsel_oracle.c), select what the reference's PixelSelector selects on the reference's pyramids.  The
reference's results are in tests/golden/reference_pins_undistort.npz (oracle/gen_reference_pins_undistort.py)."""
import functools
import os

import numpy as np
import pytest

from oracle import pixsel as P
from oracle import undistort as U

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_pins_undistort.npz")


@functools.lru_cache(maxsize=None)
def run(name):
    return U.run_oracle(name)


@pytest.mark.parametrize("name", list(U.CASES))
def test_undistort_oracle_pinned_to_reference(name):
    g = np.load(GOLDEN)
    r = run(name)
    assert r["valid"] == bool(g[f"{name}_valid"])
    if r["valid"]:
        assert np.array_equal(r["G"], g[f"{name}_G"])
    assert len(r["binv"]) == len(U.CASES[name]["gammas"])
    for k, b in enumerate(r["binv"]):
        assert np.array_equal(b, g[f"{name}_binv{k}"])
    assert np.array_equal(r["B"], g[f"{name}_B"], equal_nan=True)
    for k, f in enumerate(r["frames"]):
        assert U.frame_mismatches(g, name, k, f["exposure_time"], f["image"], f["bgr"], f["levels"]) == [], k


@pytest.mark.parametrize("name", [n for n, c in U.CASES.items() if c["select"]])
def test_selection_on_gamma_weighted_pyramid_pinned(name):
    g = np.load(GOLDEN)
    c = U.CASES[name]
    lv = run(name)["frames"][0]["levels"]
    o = P.PixelSelectorOracle(c["w"], c["h"])
    r = o.make_maps_on(lv[0][0], [lv[l][1] for l in range(3)], 1500.0, 1, 1.0)
    assert r["ret"] == int(g[f"{name}_f0_select_ret"])
    assert np.array_equal(r["map"], U.pinned_selection_map(g, name, c["w"], c["h"]))
    # the weights matter: the unweighted pyramid of the same image selects differently
    plain = U.make_images(run(name)["frames"][0]["image"], 3, None)
    r0 = P.PixelSelectorOracle(c["w"], c["h"]).make_maps_on(plain[0][0], [plain[l][1] for l in range(3)], 1500.0, 1, 1.0)
    assert not np.array_equal(r0["map"], r["map"])


def test_cases_reach_every_path():
    seen = set()
    for name, c in U.CASES.items():
        r = run(name)
        seen.add(f"mode {c['mode']}")
        seen.add("valid" if r["valid"] else "invalid")
        seen.add("passthrough" if not c["remap"] else ("w_org > w" if c["w_org"] > c["w"] else "w_org < w" if c["w_org"] < c["w"]
                                                       else "w_org == w"))
        if c["resp"] == "long":
            seen.add("response > 256")
        if c["vig"]:
            seen.add(c["vig"])
        if len(c["gammas"]) > 1:
            seen.add("two set_gamma")
        if not c["use_exposure"]:
            seen.add("use_exposure off")
        for k, (exposure, factor, _) in enumerate(c["frames"]):
            if exposure <= 0:
                seen.add("exposure <= 0")
            if factor != 1:
                seen.add("factor != 1")
            img = r["frames"][k]["image"]
            if np.isnan(img).any():
                seen.add("NaN grey")
            if np.isinf(img).any():
                seen.add("inf grey")
        if "plateau" in c["gammas"]:
            seen.add("plateau Binv")   # test_set_gamma_keeps_unfound_entries shows what it leaves unfound
        if (c["w"] % 2 or c["h"] % 2):
            seen.add("odd size")
    for want in ("mode 0", "mode 1", "mode 2", "valid", "invalid", "passthrough", "w_org > w", "w_org < w", "response > 256",
                 "v8", "v16", "v16_zero", "two set_gamma", "use_exposure off", "exposure <= 0", "factor != 1", "NaN grey",
                 "inf grey", "plateau Binv", "odd size"):
        assert want in seen, want


def test_set_gamma_keeps_unfound_entries():
    G = U.create("down_97x75to91x67_mode0")[1]
    B1 = U.set_gamma(U.binv("G", G), np.arange(256, dtype=np.float32))
    B2 = U.set_gamma(U.binv("plateau", G), B1)
    assert np.array_equal(B2[200:255], B1[200:255])          # Binv <= 191 everywhere: no s found for these i
    B3 = U.set_gamma(U.binv("plateau", G), np.arange(256, dtype=np.float32))
    assert np.array_equal(B3[200:255], np.arange(200, 255, dtype=np.float32))
    assert not np.array_equal(B2[10:100], B1[10:100])
