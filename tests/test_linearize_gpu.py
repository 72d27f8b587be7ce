"""n12 on the device: ActivePoints (tdm_active_*) equals the C oracle of DSO's linearizeAll (oracle/linearize_oracle.c, itself
pinned to the reference by tests/test_linearize_cpu.py) bit for bit on every per-residual output, the Jacobians of every
residual that is not OOB, the new frameEnergyTH, the applied states, the removed flags and the points' maxRelBaseline and
numGoodResiduals, at every step of an optimize()-shaped sequence, on every variant of the activated-points window and of a
seeded 2000-point window at 640x480 (and on the pins themselves).  The energy is within 1e-12 relative of the oracle's
sequential sum and the same on every call.  The file also covers sticky OOB across apply calls, zero residuals, the
empty-threshold case, invalid input, the ordering against asynchronous pyramid builds and the C++ shim."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from oracle import linearize as L
from tandem_b200 import ActivePoints, ImagePyramid, TandemError
from tandem_b200._lib import lib

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "reference_pins_linearize.npz")
CASES = [(s, v) for s in ("room", "seeded") for v in L.VARIANTS]


def pyramids(win):
    out = []
    for g in win["gray"]:
        p = ImagePyramid(win["w"], win["h"], 1)
        p.build(np.ascontiguousarray(g, np.float32))
        out.append(p)
    return out


class Device:
    """ActivePoints over one window with the oracle's call signature."""

    def __init__(self, win, fp=None, capacity=None):
        self.win = win
        self.fp = fp or pyramids(win)
        self.d = ActivePoints(win["w"], win["h"], capacity or max(len(win["host"]), 1), **win["settings"])
        self.load()

    def load(self):
        W = self.win
        self.d.load(W["n_frames"], W["host"], W["u"], W["v"], W["color"], W["weights"], W["res_point"], W["res_target"],
                    W["max_rel_baseline"], W["num_good"])

    def linearize(self, ids, idz, precalc, frame_th, fix):
        return self.d.linearize(self.fp, precalc, frame_th, self.win["calib4"], ids, idz, fix=fix)

    def apply_res(self):
        self.d.apply_res()


@pytest.mark.parametrize("source,variant", CASES)
def test_linearize_sequence_equals_oracle(source, variant):
    win = L.window(source, variant)
    o, d = L.LinearizeOracle(win), Device(win)
    ro, rd = L.run_sequence(o, win), L.run_sequence(d, win)
    for k, ((st, a, tha), (_, b, thb)) in enumerate(zip(ro, rd)):
        assert np.array_equal(tha, thb), k
        assert L.compare(b, a, exact_energy=False) == [], (k, L.compare(b, a, exact_energy=False))
    # the states the device holds after the sequence are the oracle's
    s = d.d.get_state()
    assert np.array_equal(s["state"], o.state.astype(np.int8))
    assert L.same_bits(s["energy"], o.energy.astype(np.float32))
    if variant == "sticky_oob":
        # residuals OOB after the applied perturbed step stay OOB through the rejected step and the fix call
        oob1 = ro[1][1]["new_state"] == L.OOB
        assert oob1.sum() > 20
        assert (ro[2][1]["new_state"][oob1] == L.OOB).all() and (rd[3][1]["state"][oob1] == L.OOB).all()
        assert rd[3][1]["removed"][oob1].all()


@pytest.mark.skipif(not os.path.exists(GOLDEN), reason="no pins")
@pytest.mark.parametrize("variant", list(L.VARIANTS))
def test_linearize_equals_pins(variant):
    g = np.load(GOLDEN)
    win = L.window("room", variant)
    for k, (st, r, th) in enumerate(L.run_sequence(Device(win), win)):
        pre = f"{variant}_s{k}_"
        pins = {key[len(pre):]: g[key] for key in g.files if key.startswith(pre)}
        assert L.compare_pins(r, pins, exact_energy=False) == [], (k, L.compare_pins(r, pins, exact_energy=False))


@pytest.mark.parametrize("seed", [1, 2])
def test_seeded_windows_and_repeated_calls(seed):
    win = L.window("seeded", "base", seed=seed, n_points=2200)
    o, d = L.LinearizeOracle(win), Device(win, capacity=4000)
    st = L.steps(win)[1]
    a = o.linearize(st["idepth_scaled"], st["idepth_zero_scaled"], st["precalc"], win["frame_th"], 0)
    b = [d.linearize(st["idepth_scaled"], st["idepth_zero_scaled"], st["precalc"], win["frame_th"], 0) for _ in range(3)]
    for r in b:
        assert L.compare(r, a, exact_energy=False) == []
        assert np.float64(r["energy"]).tobytes() == np.float64(b[0]["energy"]).tobytes()
    assert abs(b[0]["energy"] - a["energy"]) <= 1e-12 * abs(a["energy"])


def test_zero_residuals_and_the_empty_threshold():
    win = L.window("room", "base")
    fp = pyramids(win)
    d = ActivePoints(win["w"], win["h"], 16)
    pc = L.steps(win)[0]["precalc"]
    n = win["n_frames"]
    for npt in (0, 3):
        d.load(n, win["host"][:npt], win["u"][:npt], win["v"][:npt], win["color"][:npt], win["weights"][:npt], [], [])
        for fix in (0, 1):
            r = d.linearize(fp, pc, win["frame_th"], win["calib4"], win["idepth"][:npt], win["idepth"][:npt], fix=fix)
            assert r["energy"] == 0.0 and r["new_frame_energy_th"] == 12 * 12 * 8
            assert all(len(r[k]) == 0 for k in ("new_state", "jacobians"))
        d.apply_res()
    # residuals, none to the newest frame: 12*12*8 as well
    win2 = L.window("room", "no_newest")
    r = Device(win2, fp=fp).linearize(win2["idepth"], win2["idepth"], pc, win2["frame_th"], 0)
    assert r["new_frame_energy_th"] == 12 * 12 * 8 and r["energy"] > 0


def test_invalid_input_is_an_error_and_launches_nothing():
    win = L.window("room", "base")
    fp = pyramids(win)
    n, m = win["n_frames"], len(win["res_point"])
    d = ActivePoints(win["w"], win["h"], len(win["host"]))
    st = L.steps(win)[0]
    with pytest.raises(TandemError):   # linearize before load
        d.linearize(fp[:0], np.zeros(0, np.float32), np.zeros(0, np.float32), win["calib4"], np.zeros(0, np.float32),
                    np.zeros(0, np.float32))

    def load(n_frames=n, host=win["host"], rp=win["res_point"], rt=win["res_target"], k=len(win["host"])):
        d.load(n_frames, host[:k], win["u"][:k], win["v"][:k], win["color"][:k], win["weights"][:k], rp, rt)

    bad_host = win["host"].copy()
    bad_host[5] = n
    same = win["res_target"].copy()
    same[7] = win["host"][win["res_point"][7]]
    bad = [
        lambda: load(n_frames=1),
        lambda: load(n_frames=9),
        lambda: load(host=bad_host),
        lambda: load(rp=np.where(np.arange(m) == 3, len(win["host"]), win["res_point"])),
        lambda: load(rp=np.where(np.arange(m) == 3, -1, win["res_point"])),
        lambda: load(rt=np.where(np.arange(m) == 3, n, win["res_target"])),
        lambda: load(rt=same),                                                           # host == target
        lambda: ActivePoints(win["w"], win["h"], 10).load(n, win["host"], win["u"], win["v"], win["color"], win["weights"],
                                                          [], []),                     # capacity (points)
        lambda: ActivePoints(win["w"], win["h"], 1).load(n, win["host"][:1], win["u"][:1], win["v"][:1], win["color"][:1],
                                                         win["weights"][:1], [0] * 9, [(win["host"][0] + 1) % n] * 9),
    ]
    for f in bad:
        with pytest.raises(TandemError):
            f()
    assert lib().tdm_active_load(None, n, 0, None, None, None, None, None, None, None, 0, None, None) < 0
    assert lib().tdm_active_apply_res(None) < 0
    load()
    other = ImagePyramid(win["w"] + 2, win["h"], 1)
    other.build(np.zeros((win["h"], win["w"] + 2), np.float32))
    with pytest.raises(TandemError):
        d.linearize([other] + fp[1:], st["precalc"], win["frame_th"], win["calib4"], win["idepth"], win["idepth"])
    assert lib().tdm_active_linearize(d._h, None, None, None, None, None, None, 0, *([None] * 11)) < 0
    # nothing ran: the state is resetOOB's, and a full sequence still equals the oracle
    s = d.get_state()
    assert (s["state"] == L.IN).all() and (s["energy"] == 0).all()
    o = L.LinearizeOracle(win)
    a = o.linearize(st["idepth_scaled"], st["idepth_zero_scaled"], st["precalc"], win["frame_th"], 0)
    b = d.linearize(fp, st["precalc"], win["frame_th"], win["calib4"], st["idepth_scaled"], st["idepth_zero_scaled"])
    assert L.compare(b, a, exact_energy=False) == []


def test_reads_after_async_builds_and_rebuilds_wait():
    win = L.window("room", "base")
    fp = [ImagePyramid(win["w"], win["h"], 1) for _ in win["gray"]]
    zero = np.zeros((win["h"], win["w"]), np.float32)
    for p in fp:
        p.build(zero)
    d = Device(win, fp=fp)
    o = L.LinearizeOracle(win)
    st = L.steps(win)[0]
    a = o.linearize(st["idepth_scaled"], st["idepth_zero_scaled"], st["precalc"], win["frame_th"], 0)
    # the builds are asynchronous; the call right behind them must see the new images
    for p, g in zip(fp, win["gray"]):
        p.build(np.ascontiguousarray(g, np.float32))
    b = d.linearize(st["idepth_scaled"], st["idepth_zero_scaled"], st["precalc"], win["frame_th"], 0)
    assert L.compare(b, a, exact_energy=False) == []
    # The call returns only after its reads (it is blocking), so a later rebuild cannot overlap them and its ordering after
    # the call (the event the call records, which the pyramids' streams wait for) is not observable from here.  What is
    # checked: rebuilding every pyramid with other images right after the call, then back, gives the same result again.
    for p in fp:
        p.build(zero)
    for p, g in zip(fp, win["gray"]):
        p.build(np.ascontiguousarray(g, np.float32))
    assert L.compare(d.linearize(st["idepth_scaled"], st["idepth_zero_scaled"], st["precalc"], win["frame_th"], 0), a,
                     exact_energy=False) == []


def test_pinned_output_buffers():
    from tandem_b200._lib import pinned_empty
    win = L.window("seeded", "base")
    d = Device(win)
    st = L.steps(win)[0]
    m = len(win["res_point"])
    out = dict(jacobians=pinned_empty((m, L.JACOBIAN_FLOATS), np.float32), new_state=pinned_empty((m,), np.int8))
    a = d.linearize(st["idepth_scaled"], st["idepth_zero_scaled"], st["precalc"], win["frame_th"], 0)
    b = d.d.linearize(d.fp, st["precalc"], win["frame_th"], win["calib4"], st["idepth_scaled"], st["idepth_zero_scaled"], out=out)
    assert b["jacobians"] is out["jacobians"]
    assert L.compare(b, a, exact_energy=True) == []
    # caller arrays must be what the call writes: wrong shape, dtype, layout or read-only is an error before the call
    sent = np.full((m, L.JACOBIAN_FLOATS), 7.0, np.float32)
    bad = [dict(jacobians=np.empty((m - 1, L.JACOBIAN_FLOATS), np.float32)), dict(jacobians=np.empty((m, L.JACOBIAN_FLOATS))),
           dict(new_state=np.empty(m, np.int32)), dict(jacobians=np.empty((L.JACOBIAN_FLOATS, m), np.float32).T),
           dict(new_energy=np.broadcast_to(np.float32(0), (m,))), dict(energies=np.empty(m, np.float32))]
    for o in bad:
        with pytest.raises((ValueError, TypeError)):
            d.d.linearize(d.fp, st["precalc"], win["frame_th"], win["calib4"], st["idepth_scaled"], st["idepth_zero_scaled"], out=o)
    # an array for an output the call does not return (no Jacobians asked for, no fix) is left as it is
    fixed_only = np.full(m, 5, np.uint8)
    c = d.d.linearize(d.fp, st["precalc"], win["frame_th"], win["calib4"], st["idepth_scaled"], st["idepth_zero_scaled"],
                      jacobians=False, out=dict(jacobians=sent, removed=fixed_only))
    assert "jacobians" not in c and (sent == 7.0).all() and (fixed_only == 5).all()
    assert L.compare(dict(c, jacobians=a["jacobians"]), a, exact_energy=True) == []


def test_load_is_ordered_before_the_next_call_behind_default_stream_work():
    """load() uploads and resets on the set's own stream and returns once that has landed: a window loaded over a set whose
    residuals a previous sequence moved (applied states, OOB), while other work is queued on the default stream, linearizes
    from resetOOB's states."""
    import torch
    win = L.window("room", "sticky_oob")
    d = Device(win)
    L.run_sequence(d, win)
    assert (d.d.get_state()["state"] == L.OOB).any()
    x = torch.randn(4096, 4096, device="cuda")
    for _ in range(20):   # tens of milliseconds of work on the default stream
        x = x @ x
        x = x / x.norm()
    d.load()
    st = L.steps(win)[0]
    b = d.linearize(st["idepth_scaled"], st["idepth_zero_scaled"], st["precalc"], win["frame_th"], 0)
    a = L.LinearizeOracle(win).linearize(st["idepth_scaled"], st["idepth_zero_scaled"], st["precalc"], win["frame_th"], 0)
    assert L.compare(b, a, exact_energy=False) == []
    torch.cuda.synchronize()


def test_shim_runs_the_sequence(tmp_path):
    exe = os.path.join(ROOT, "tests", "cpp", "shim_linearize")
    if not os.path.exists(exe):
        pytest.fail("tests/cpp/shim_linearize was not built")
    win = L.window("room", "sticky_oob")
    path = str(tmp_path / "window.bin")
    seq = L.steps(win)
    with open(path, "wb") as f:
        n, npt, m = win["n_frames"], len(win["host"]), len(win["res_point"])
        f.write(np.array([win["w"], win["h"], n, npt, m, len(seq)], np.int32).tobytes())
        for g in win["gray"]:
            f.write(np.ascontiguousarray(g, np.float32).tobytes())
        f.write(win["calib4"].tobytes())
        f.write(win["frame_th"].tobytes())
        for k in ("host",):
            f.write(win[k].astype(np.int32).tobytes())
        for k in ("u", "v", "color", "weights", "max_rel_baseline"):
            f.write(win[k].astype(np.float32).tobytes())
        f.write(win["num_good"].astype(np.int32).tobytes())
        f.write(win["res_point"].tobytes())
        f.write(win["res_target"].tobytes())
        for st in seq:
            f.write(np.array([st["fix"], st["apply"]], np.int32).tobytes())
            f.write(st["idepth_scaled"].tobytes())
            f.write(st["idepth_zero_scaled"].tobytes())
            f.write(np.ascontiguousarray(st["precalc"], np.float32).tobytes())
    out = str(tmp_path / "out.bin")
    r = subprocess.run([exe, path, out], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout + r.stderr
    assert "shim_linearize: OK" in r.stdout
    b = open(out, "rb").read()
    pos = 0

    def take(dtype, k):
        nonlocal pos
        a = np.frombuffer(b, dtype, k, pos)
        pos += a.nbytes
        return a

    for k, (st, a, th) in enumerate(L.run_sequence(L.LinearizeOracle(win), win)):
        got = dict(energy=float(take(np.float64, 1)[0]), new_frame_energy_th=float(take(np.float32, 1)[0]),
                   new_state=take(np.int8, m), new_energy=take(np.float32, m), new_energy_with_outlier=take(np.float32, m),
                   center_projected_to=take(np.float32, 3 * m).reshape(m, 3),
                   jacobians=take(np.float32, m * L.JACOBIAN_FLOATS).reshape(m, L.JACOBIAN_FLOATS))
        if st["fix"]:
            got.update(state=take(np.int8, m), removed=take(np.uint8, m), max_rel_baseline=take(np.float32, npt),
                       num_good_residuals=take(np.int32, npt))
        assert L.compare(got, a, exact_energy=False) == [], (k, L.compare(got, a, exact_energy=False))
    assert pos == len(b)
