"""Host-side checks (no GPU) behind the TSDF option sweep of tests/test_fusion_options_gpu.py: the constant-divisor division
of the ray-cast is correctly rounded for every divisor the sweep uses, a divisor it is not proven correct for leaves fast_div off,
options whose rays could reach the ray-cast's step guard are refused, and the mesh extractor's per-axis tables match a
float32 restatement for every box and voxel size of the sweep."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from oracle import fusion_options as FO
from tandem_b200 import DrFusionOptions
from tandem_b200._lib import lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VOXEL_SIZES = sorted({c["voxel_size"] for c in FO.CASES.values()} - {0.01})          # 0.01 is covered by test_abi.py
FOCALS = sorted({c[k] for c in FO.CASES.values() for k in ("fx", "fy")})
EXCLUDED = float.fromhex("0x1.fffffep+6")                                               # 127.99999, all-ones significand


@pytest.fixture(scope="module")
def cdiv(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("cdiv") / "libcdiv_check.so")
    subprocess.run(["gcc", "-O2", "-mfma", "-ffp-contract=off", "-fno-fast-math", "-shared", "-fPIC", "-o", so,
                    os.path.join(ROOT, "tests", "cpp", "cdiv_check.c"), "-lm"], check=True)
    l = ctypes.CDLL(so)
    l.cdiv_check_exhaustive.restype = ctypes.c_long
    l.cdiv_check_exhaustive.argtypes = [ctypes.c_float, ctypes.c_float, ctypes.c_float]
    l.cdiv_check_random_x.restype = ctypes.c_long
    l.cdiv_check_random_x.argtypes = [ctypes.c_float, ctypes.c_uint64, ctypes.c_long]
    return l


@pytest.mark.parametrize("d", VOXEL_SIZES)
def test_constant_division_by_voxel_size_is_correctly_rounded(cdiv, d):
    """cdiv_ divides world coordinates by voxel_size: every float of |x| in [1e-6, 4096] (and its negation), as for 0.01 in
    test_abi.py, and 1e7 random x over 80 binades."""
    assert cdiv.cdiv_check_exhaustive(d, 1e-6, 4096.0) == 0
    assert cdiv.cdiv_check_random_x(d, 11, 10_000_000) == 0


@pytest.mark.parametrize("d", FOCALS)
def test_constant_division_by_focal_length_is_correctly_rounded(cdiv, d):
    """cdiv_ divides (u - cx) * depth by fx and (v - cy) * depth by fy: every float of |x| in [1e-3, 16384] covers pixel offsets
    from 0.5 to 200 at ray depths from 0.005 to 80, plus 1e7 random x."""
    assert cdiv.cdiv_check_exhaustive(d, 1e-3, 16384.0) == 0
    assert cdiv.cdiv_check_random_x(d, 12, 10_000_000) == 0


def test_excluded_divisor_leaves_fast_div_off(cdiv):
    """The host turns fast_div on only where Markstein's theorem proves the sequence correctly rounded, so never for a divisor
    with an all-ones significand, in any of the three divisor slots, and always for the sweep's divisors.  The theorem does
    not cover an all-ones significand; for 0x1.fffffep+6 every quotient over the ray-cast's range of a focal-length division
    is in fact correctly rounded (checked exhaustively here), so the exclusion is conservative there."""
    assert cdiv.cdiv_check_exhaustive(EXCLUDED, 1e-3, 16384.0) == 0
    l = lib()
    for vs, fx, fy in [(0.01, EXCLUDED, 80.0), (0.01, 80.0, EXCLUDED), (EXCLUDED / 8192, 80.0, 80.0)]:
        assert l.tdm_debug_fast_div_eligible(vs, fx, fy) == 0, (vs, fx, fy)
    for c in FO.CASES.values():
        assert l.tdm_debug_fast_div_eligible(c["voxel_size"], c["fx"], c["fy"]) == 1, c


def _create(**kw):
    h = ctypes.c_void_p()
    rc = lib().tdm_fusion_create(ctypes.byref(DrFusionOptions(**kw)), 0, ctypes.byref(h))
    if rc == 0:
        lib().tdm_fusion_destroy(h)
    return rc, lib().tdm_last_error().decode()


def test_options_that_could_reach_the_march_guard_are_refused():
    """Every ray-cast step that does not end a ray adds at least min(truncation_distance, voxel_size), and the production
    kernel does not count the steps of a ray's clipped prefix against the 100000-step guard the comparator and the oracle
    count.  Options allowing more than 50000 steps are refused before anything is allocated (with or without a GPU), so the
    three can never end a ray differently; 50000 itself is accepted.  Non-positive or non-finite sizes are refused too."""
    for kw in [dict(truncation_distance=1e-4), dict(voxel_size=1e-4, truncation_distance=1e-4), dict(max_sensor_depth=600.0),
               dict(voxel_size=1.9e-4)]:
        rc, err = _create(**kw)
        assert rc != 0 and "must not exceed 50000" in err, (kw, err)
    for kw in [dict(voxel_size=0.0), dict(voxel_size=-0.01), dict(voxel_size=float("nan")), dict(truncation_distance=0.0),
               dict(truncation_distance=float("inf")), dict(max_sensor_depth=float("nan"))]:
        rc, err = _create(**kw)
        assert rc != 0 and ("must be positive and finite" in err or "must be finite" in err), (kw, err)
    rc, err = _create(max_sensor_depth=500.0)                       # 500 / 0.01 = 50000: the limit itself
    assert "50000" not in err, err
    assert rc == 0 or "no CPU fallback" in err, err


def _boxes():
    out = []
    for name in FO.CASES:
        for lo, up in FO.mesh_boxes(name):
            out.append((name, FO.CASES[name]["voxel_size"], lo, up))
    return out


@pytest.mark.parametrize("name,s,lower,upper", _boxes())
def test_mesh_axis_tables_at_the_sweep_boxes(name, s, lower, upper):
    """The mesh extractor's per-axis cell table (host logic) against a float32 restatement of mesh_extractor.cu:248-261 and
    WorldToGlobalVoxel, for every cell of every axis of the boxes tests/test_fusion_options_gpu.py meshes."""
    f32 = np.float32
    vs = f32(s)
    h = vs / f32(2)

    def w2g(x):
        x = f32(x)
        sg = f32(int(x > 0) - int(x < 0))
        return int(f32(f32(x / vs) + f32(sg * f32(0.5))))

    ip, fp = ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_float)
    for a in range(3):
        lo, up = f32(lower[a]), f32(upper[a])
        cap = 4096
        ints = np.zeros((cap, 5), np.int32); flts = np.zeros((cap, 4), np.float32); rng = np.zeros((cap, 2), np.int32)
        bm = np.zeros(2, np.int32)
        n = lib().tdm_debug_mesh_axis_table(float(lo), float(up), float(vs), ints.ctypes.data_as(ip), flts.ctypes.data_as(fp),
                                            rng.ctypes.data_as(ip), bm.ctypes.data_as(ip), cap)
        assert n == int(f32(abs(lo - up)) / vs) and 0 < n <= cap, (name, a, n)
        for i in range(n):
            pos = f32(np.longdouble(i) * np.longdouble(vs) + np.longdouble(lo))   # one rounding, as the fma
            cM, cP = f32(pos + (-h)), f32(pos + h)
            exp = []
            for c in (cM, cP):
                pd = f32(c - h)
                exp += [w2g(f32(pd + f32(0))), w2g(f32(pd + vs))]
            exp.append(w2g(pos))
            assert list(ints[i]) == exp, (name, a, i, list(ints[i]), exp)
            vpM, vpP = f32(cM / vs), f32(cP / vs)
            assert flts[i, 0] == f32(vpM - np.floor(vpM)) and flts[i, 1] == f32(vpP - np.floor(vpP)), (name, a, i)
            assert flts[i, 2] == cM and flts[i, 3] == cP, (name, a, i)
        first, nb, covered = int(bm[0]), int(bm[1]), 0
        for b in range(nb):
            s0, c = int(rng[b, 0]), int(rng[b, 1])
            if c == 0:
                continue
            assert s0 == covered
            covered += c
            g = ints[s0:s0 + c]
            assert (g[:, 0] >> 3 == first + b).all() and g.min() >= 8 * (first + b) and g.max() < 8 * (first + b) + 12
        assert covered == n, (name, a)
