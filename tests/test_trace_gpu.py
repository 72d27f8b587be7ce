"""n8 on the device: ImmaturePoints (tdm_immature_*) equals the C oracle of DSO's ImmaturePoint constructor and traceOn
(oracle/trace_oracle.c, itself pinned to the reference by tests/test_trace_cpu.py) bit for bit - every state field after every
trace of every pin case (and the pins' digests), and seeded random sequences of 7 hosts - plus the compaction of
activatePointsMT, the ordering against pyramid rebuilds, the out-of-image rule and the rejection of invalid input."""
import os
import subprocess

import numpy as np
import pytest

from oracle import trace as T
from oracle.pins_coarse_ref import K4
from tandem_b200 import ImagePyramid, ImmaturePoints, TandemError

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "reference_pins_trace.npz")
STATE_KEYS = {"idepth_min": "idepth_min", "idepth_max": "idepth_max", "quality": "quality", "status": "status", "uv": "uv",
              "interval": "interval"}


def same_bits(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape:
        return False
    if a.dtype.kind == "f":
        na, nb = np.isnan(a), np.isnan(b)
        return np.array_equal(na, nb) and np.array_equal(a[~na].view(np.uint32), b[~nb].view(np.uint32))
    return np.array_equal(a, b)


def pyramid(gray):
    h, w = gray.shape
    p = ImagePyramid(w, h, 1)
    p.build(gray)
    return p


def run_device(c, frames_gray=None):
    """Adds every host, traces every frame (one call for all hosts); returns (adds {slot: (m, fields)}, [state per slot])."""
    d = ImmaturePoints(c["w"], c["h"], 4096, **c["settings"])
    hp = [pyramid(hh["gray"]) for hh in c["hosts"]]
    adds = {}
    for hh, p in zip(c["hosts"], hp):
        m = d.add(hh["slot"], p, hh["u"], hh["v"], hh["type"])
        adds[hh["slot"]] = (m, d.get(hh["slot"]))
    frame = ImagePyramid(c["w"], c["h"], 1)
    states = []
    for f in c["frames"]:
        frame.build(f["gray"])
        slots = sorted(f["params"])
        d.trace(frame, slots, [f["params"][s][0] for s in slots], [f["params"][s][1] for s in slots],
                [f["params"][s][2] for s in slots], host_pyramids=[hp[[h["slot"] for h in c["hosts"]].index(s)] for s in slots])
        states.append({s: d.get(s) for s in slots})
    return adds, states


@pytest.mark.parametrize("name", list(T.CASES))
def test_trace_equals_oracle_and_pins(name):
    c = T.case_inputs(name)
    g = np.load(GOLDEN)
    oadds, otraces = T.run_oracle(c)
    for hh in c["hosts"]:
        assert same_bits(pyramid(hh["gray"]).level(0)[0], hh["dI"])          # the pinned pyramid definition
    adds, states = run_device(c)
    for slot, (m, fields) in adds.items():
        assert m == oadds[slot][0] == int(g[f"{name}_add{slot}_n"])
        for k in T.POINT:
            assert same_bits(fields[k], oadds[slot][1][k]), (slot, k)
            assert T.digest(fields[k]) == str(g[f"{name}_add{slot}_{k}"]), (slot, k)
    for j, (st, ot) in enumerate(zip(states, otraces)):
        for slot in st:
            for k in T.STATE:
                assert same_bits(st[slot][k], ot[slot][0][k]), (j, slot, k)
                assert T.digest(st[slot][k]) == str(g[f"{name}_t{j}_{slot}_{k}"]), (j, slot, k)


def random_case(seed, n_hosts=7, npts=700, h=480, w=640, frames=4):
    from oracle.cpu import FrontOracle
    rng = np.random.default_rng(seed)
    front = FrontOracle()
    hosts = []
    for j in range(n_hosts):
        p = T.pose(rng.uniform(-2, 6), jitter=rng.uniform(-0.05, 0.05))
        g = T.gray(p, h, w).astype(np.float32)
        dI = T.level0(g, front)
        u, v = T.select(dI, npts, rng)
        hosts.append(dict(slot=j, pose=p, gray=g, dI=dI, u=u, v=v, type=np.ones(len(u), np.float32)))
    fr = []
    for k in range(frames):
        c2w = T.pose(rng.uniform(-2, 8), jitter=rng.uniform(-0.05, 0.05))
        g = T.gray(c2w, h, w).astype(np.float32)
        params = {}
        for hh in hosts:
            K, Kt, aff = T.frame_params("real", c2w, hh["pose"], K4(h, w))
            params[hh["slot"]] = (K, Kt, np.array([rng.uniform(0.9, 1.1), rng.uniform(-5, 5)], np.float32))
        fr.append(dict(gray=g, dI=T.level0(g, front), params=params))
    return dict(w=w, h=h, settings=dict(T.DEFAULT_SETTINGS), hosts=hosts, frames=fr)


@pytest.mark.parametrize("seed", [11, 12])
def test_trace_random_sequences_of_seven_hosts(seed):
    c = random_case(seed)
    oadds, otraces = T.run_oracle(c)
    adds, states = run_device(c)
    assert sum(m for m, _ in adds.values()) >= 4000
    statuses = np.zeros(6, int)
    for st, ot in zip(states, otraces):
        for slot in st:
            assert not ot[slot][3].any()
            for k in T.STATE:
                assert same_bits(st[slot][k], ot[slot][0][k]), (slot, k)
            statuses += np.bincount(st[slot]["status"], minlength=6)
    assert statuses[0] > 1000, statuses   # most traces find a real match


def test_remove_and_drop_host_follow_activate_points_compaction():
    c = T.case_inputs("room_160x120_nan_hosts")
    d = ImmaturePoints(c["w"], c["h"], 1024)
    hp = pyramid(c["hosts"][0]["gray"])
    m = d.add(5, hp, c["hosts"][0]["u"], c["hosts"][0]["v"], c["hosts"][0]["type"])
    ref = d.get(5)
    ids = list(range(m))
    rng = np.random.default_rng(3)
    for removed in (rng.choice(m, 40, replace=False), [m - 41, 0, m - 42], [], list(range(m - 43))):
        null = set(int(i) for i in removed)
        # FullSystem.cpp:849-856
        vec = [None if i in null else ids[i] for i in range(len(ids))]
        i = 0
        while i < len(vec):
            if vec[i] is None:
                vec[i] = vec[-1]
                vec.pop()
                i -= 1
            i += 1
        d.remove(5, np.array(sorted(null) if len(null) % 2 else list(null), np.int32))
        ids = vec
        got = d.get(5)
        assert len(got["u"]) == len(ids)
        for k in got:
            assert same_bits(got[k], ref[k][ids]), k
    d.drop_host(5)
    assert d.count(5) == 0
    assert d.add(5, hp, c["hosts"][0]["u"][:10], c["hosts"][0]["v"][:10]) == 10


def test_rebuilding_the_frame_pyramid_right_after_a_trace_keeps_the_old_image():
    c = T.case_inputs("room_320x240_3hosts")
    hh = c["hosts"][0]
    f0, f1 = c["frames"][0], c["frames"][3]
    K, Kt, aff = f0["params"][hh["slot"]]
    results = []
    for rebuild in (False, True):
        d = ImmaturePoints(c["w"], c["h"], 1024)
        hp = pyramid(hh["gray"])
        d.add(0, hp, hh["u"], hh["v"], hh["type"])
        frame = pyramid(f0["gray"])
        d.trace(frame, [0], [K], [Kt], [aff], host_pyramids=[hp])
        if rebuild:
            frame.build(f1["gray"])
            hp.build(f1["gray"])
            del frame
        results.append(d.get(0))
    for k in results[0]:
        assert same_bits(results[0][k], results[1][k]), k


def test_out_of_image_samples_stay_in_bounds_and_count_as_non_finite():
    c = T.case_inputs("room_160x120_no_search")
    hh = c["hosts"][0]
    s = dict(T.DEFAULT_SETTINGS)
    o = T.TraceOracle(c["w"], c["h"], s)
    d = ImmaturePoints(c["w"], c["h"], 1024)
    hp = pyramid(hh["gray"])
    assert o.add(0, hh["dI"], hh["u"], hh["v"], hh["type"]) == d.add(0, hp, hh["u"], hh["v"], hh["type"])
    # a 4x magnification about the image centre: the rotated pattern spans +-8 pixels, so near the border samples leave the
    # image although uMin / uMax pass the 4-pixel margin test
    cx, cy = (c["w"] - 1) / 2.0, (c["h"] - 1) / 2.0
    K = np.array([[4, 0, -3 * cx], [0, 4, -3 * cy], [0, 0, 1]], np.float32)
    Kt = np.array([8.0, 0.0, 0.0], np.float32)
    aff = np.array([1.0, 0.0], np.float32)
    frame = pyramid(c["frames"][0]["gray"])
    diag = o.trace(c["frames"][0]["dI"], {0: (K, Kt, aff)})
    d.trace(frame, [0], [K], [Kt], [aff])
    assert diag[0][2].sum() > 0                                  # some samples left the image
    got = d.get(0)
    for k in T.STATE:
        assert same_bits(got[k], o.pts[0][k]), k


def test_invalid_input_is_an_error_and_launches_nothing():
    c = T.case_inputs("room_160x120_no_search")
    hh = c["hosts"][0]
    d = ImmaturePoints(c["w"], c["h"], 300)
    hp = pyramid(hh["gray"])
    m = d.add(1, hp, hh["u"], hh["v"])
    before = d.get(1)
    other = ImagePyramid(c["w"] + 2, c["h"], 1)
    other.build(np.zeros((c["h"], c["w"] + 2), np.float32))
    frame = pyramid(c["frames"][0]["gray"])
    K, Kt, aff = c["frames"][0]["params"][0]
    bad = [
        lambda: d.add(8, hp, hh["u"][:3], hh["v"][:3]),
        lambda: d.add(-1, hp, hh["u"][:3], hh["v"][:3]),
        lambda: d.add(2, other, hh["u"][:3], hh["v"][:3]),
        lambda: d.add(1, hp, hh["u"], hh["v"]),                          # 300 - m free, 200 candidates
        lambda: d.add(2, hp, [1], [50]),                                 # pattern leaves the image
        lambda: d.add(2, hp, [50], [c["h"] - 3]),
        lambda: d.trace(other, [1], [K], [Kt], [aff]),
        lambda: d.trace(frame, [8], [K], [Kt], [aff]),
        lambda: d.trace(frame, [1, 1], [K, K], [Kt, Kt], [aff, aff]),
        lambda: d.trace(frame, [1], [K], [Kt], [aff], host_pyramids=[other]),
        lambda: d.remove(1, [0, 0]),
        lambda: d.remove(1, [m]),
        lambda: d.remove(1, [-1]),
        lambda: d.get(1, first=m, n=1),
        lambda: d.drop_host(9),
    ]
    for f in bad:
        with pytest.raises(TandemError):
            f()
    with pytest.raises(TandemError):
        ImmaturePoints(c["w"], c["h"], 0)
    after = d.get(1)
    assert d.count(1) == m and all(same_bits(before[k], after[k]) for k in before)
    assert d.count(2) == 0


def test_shim_traces_a_shifted_frame():
    exe = os.path.join(ROOT, "tests", "cpp", "shim_trace")
    r = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "shim_trace: OK" in r.stdout
