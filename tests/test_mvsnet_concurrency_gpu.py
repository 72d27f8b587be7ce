"""DrMvsnet handles in flight together.  Per-handle state lives in places the process or the device shares: the constant
banks c_call_params / c_conv00 (one slot per live handle, slots reused after a handle is destroyed), the process-wide copy
pool, the once-per-kernel launch set-up of the tensor-core convolutions.  Every handle here must reproduce, bit for bit, a
solo run of its window on a fresh handle that was alone in the process (forwards are deterministic:
test_mvsnet_layers_gpu.py::test_replays_are_bit_identical), whatever the other handles hold (weights, engine, window,
options, host-memory path), and the small windows are checked against the fp64 layer oracle on the concurrent handle
itself."""
import ctypes
import gc
import threading
import time
from dataclasses import dataclass, field
from typing import Optional, Tuple

import numpy as np
import pytest

from oracle import mvsnet_layers as ML
from tandem_b200 import DrMvsnet, DrMvsnetOutput, TandemError, default_weights
from tandem_b200._lib import lib, pinned_empty
from tandem_b200.synthetic import mvs_plane_window
import test_mvsnet_layers_gpu as LG    # tests/ is on sys.path (pytest prepends the rootdir of a test module)

pytestmark = pytest.mark.gpu

W03, W04 = "abl03_view_aggregation", "abl04_fewer_depth_planes"
MAPS = ("depth", "confidence", "depth_dense", "confidence_dense")
MAX_HANDLES = 8          # kMaxEngines (mvsnet_kernels.cuh): constant-bank slots
REPORT = []


@dataclass
class Case:
    name: str
    weights: str
    precision: str
    V: int
    H: int
    W: int
    ref: int
    seed: int
    dn: Optional[Tuple[int, int, int]] = None
    opts: dict = field(default_factory=dict)
    inputs: str = "pageable"      # "pageable", "pinned" (every view page-locked: direct DMA), "mixed" (staged path)
    outputs: str = "pageable"     # "pageable" or "pinned" result maps
    device: int = 0

    def window(self):
        win = mvs_plane_window(V=self.V, H=self.H, W=self.W, seed=self.seed)
        win["ref_index"] = self.ref
        win["depth_min"] = 0.5 + 0.05 * (self.seed % 4)           # per-call parameters differ between handles
        win["depth_max"] = 5.0 - 0.25 * (self.seed % 3)
        win["discard"] = 5.0 + 2.5 * (self.seed % 5)
        return win

    def depth_num(self):
        return tuple(self.dn or LG._weights(self.weights)[1])


# Eight handles alive at once: both checkpoints, all three engines, V 2 .. 16, ref_index first / middle / last, every
# host-memory path (eager_d2h 0 with pageable outputs: GetResult's own D2H), and the options that change the launches.
FLEET = [
    Case("F0 abl03 fp32 128x96v2", W03, "fp32", 2, 96, 128, 0, 1, (16, 8, 8)),
    Case("F1 abl04 mixed16 160x128v5 pinned-in", W04, "mixed16", 5, 128, 160, 2, 2, None, dict(use_is=0), inputs="pinned"),
    Case("F2 abl03 bf16 96x64v3 pinned-out eager0", W03, "bf16", 3, 64, 96, 2, 3, (16, 16, 8), dict(fused_regress=1, eager_d2h=0),
         outputs="pinned"),
    Case("F3 abl03 mixed16 128x96v16 eager0", W03, "mixed16", 16, 96, 128, 15, 4, (16, 24, 8), dict(tc_smem_kb=113, eager_d2h=0)),
    Case("F4 abl04 bf16 224x160v4 pinned-in/out", W04, "bf16", 4, 160, 224, 0, 5, None, {}, inputs="pinned", outputs="pinned"),
    Case("F5 abl04 fp32 64x64v3 pinned-out eager0", W04, "fp32", 3, 64, 64, 1, 6, None, dict(eager_d2h=0), outputs="pinned"),
    Case("F6 abl03 mixed16 160x96v7 pinned-in", W03, "mixed16", 7, 96, 160, 3, 7, (24, 16, 8), dict(use_is=0, fused_regress=1),
         inputs="pinned"),
    Case("F7 abl03 mixed16 64x32v2 pinned-out", W03, "mixed16", 2, 32, 64, 1, 8, (8, 8, 8), {}, outputs="pinned"),
]
# takes the slot of the abl03 mixed16 handle F6 (not the first slot: a kernel that read slot 0 would see F0's state)
REPLACEMENT = Case("R abl04 mixed16 128x96v3", W04, "mixed16", 3, 96, 128, 1, 9)
FP64_MAX = 5 * 128 * 160      # V * H * W up to which the fp64 layer oracle runs on a concurrent handle


def _make(c: Case) -> DrMvsnet:
    m = DrMvsnet(default_weights(c.weights), precision=c.precision, device=c.device)
    if c.dn:
        for s, D in enumerate(c.dn):
            m.set_option(f"depth_num_stage{s + 1}", D)
    for k, v in c.opts.items():
        m.set_option(k, v)
    return m


def _pinned_copy(a):
    p = pinned_empty(a.shape, a.dtype)
    p[...] = a
    return p


def _submit(m: DrMvsnet, c: Case, win, inputs=None):
    inputs = inputs or c.inputs
    bgrs = win["bgrs"]
    if inputs == "pinned":
        bgrs = [_pinned_copy(b) for b in bgrs]
    elif inputs == "mixed":          # some views page-locked, some not: the staged path
        bgrs = [_pinned_copy(b) if v % 2 else b for v, b in enumerate(bgrs)]
    m.CallAsync(c.H, c.W, c.V, win["ref_index"], bgrs, win["K"], win["c2ws"], win["depth_min"], win["depth_max"], win["discard"])


def _fetch(m: DrMvsnet, c: Case, outputs=None):
    if (outputs or c.outputs) == "pinned":
        return m.GetResult(out=DrMvsnetOutput(c.H, c.W, pinned=True))
    return m.GetResult()


def _tensor_names(c: Case):
    fp32 = c.precision == "fp32"
    names = {"f.c0_0", "feat1", "feat2", "feat3", "s3.edge"}
    for L in ML.layer_table(c.depth_num(), not fp32 and c.opts.get("use_tc", 1) == 1, not fp32):
        names.update(n for n in (L.inp, L.out, L.res, L.res_up2) if n)
    return sorted(names)


def _snapshot(m: DrMvsnet, c: Case, out=None):
    """Every output of the forward m last ran: the four GetResult maps (when given), every stage output, thr and every
    debug tensor, as float32 arrays."""
    S = {}
    if out is not None:
        S.update({f"GetResult.{k}": np.array(getattr(out, k)) for k in MAPS})
    S.update({f"s{s}.{k}": m.stage_output(s, k) for s in (1, 2, 3) for k in MAPS})
    S["thr"] = m.debug_tensor("thr")
    S.update({n: m.debug_tensor(n) for n in _tensor_names(c)})
    return S


def _differences(label, got, ref):
    assert got.keys() == ref.keys(), f"{label}: {sorted(set(got) ^ set(ref))}"
    bad = []
    for k, r in ref.items():
        g = got[k]
        if g.shape != r.shape or not np.array_equal(g.view(np.uint32), r.view(np.uint32)):
            n = int((g.view(np.uint32) != r.view(np.uint32)).sum()) if g.shape == r.shape else -1
            bad.append(f"{label}: {k} differs from the solo run on {n} of {r.size} values")
    return bad


def _solo(c: Case, win=None):
    """A fresh handle alone in the process runs the window once."""
    gc.collect()
    win = win or c.window()
    m = _make(c)
    try:
        _submit(m, c, win, "pageable")
        return _snapshot(m, c, _fetch(m, c, "pageable"))
    finally:
        m.close()


@pytest.fixture(scope="module")
def solos():
    """Solo runs of the fleet and its replacement, made before any test of this module keeps a handle alive."""
    gc.collect()
    t0 = time.time()
    out = {c.name: _solo(c) for c in FLEET + [REPLACEMENT]}
    print(f"solo runs of {len(out)} windows: {time.time() - t0:.1f} s")
    return out


@pytest.fixture(scope="module", autouse=True)
def _print_report():
    yield
    worst = {}
    for label, prec, name, path, desc, ratio in REPORT:
        key = (prec, path, desc if path != "regress" else "")
        if ratio >= worst.get(key, (-1,))[0]:
            worst[key] = (ratio, f"{label} {name}")
    if worst:
        print(f"\nconcurrent handles, worst error / bound per kernel family and precision ({len(REPORT)} checks):")
        for (prec, path, desc), (ratio, where) in sorted(worst.items()):
            print(f"  {prec:8s} {path:10s} {desc:55s} {ratio:8.4f}  ({where})")


class Fleet:
    """Handles created in order (on a process without other live handles they take slots 0, 1, ...), closed on exit."""

    def __init__(self, cases):
        gc.collect()
        self.cases = list(cases)
        self.hs = []
        for c in self.cases:
            self.hs.append(_make(c))

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        for h in self.hs:
            h.close()
        self.hs = []
        gc.collect()

    def round(self, order):
        """Every CallAsync before the first GetResult, then the results in `order`; returns the snapshots by index."""
        wins = [c.window() for c in self.cases]
        for h, c, w in zip(self.hs, self.cases, wins):
            _submit(h, c, w)
        snaps = {}
        for i in order:
            snaps[i] = _snapshot(self.hs[i], self.cases[i], _fetch(self.hs[i], self.cases[i]))
        return wins, snaps


def _fp64(m, c: Case, win, label):
    volume = c.V * c.H * c.W <= 2 * 96 * 128
    return LG.check_forward(m, win, c.weights, c.precision, c.depth_num(), c.opts, label, REPORT, volume=volume)


def test_mixed_fleet(solos):
    """Eight handles alive, all submitted before the first result is fetched, fetched in another order: each equals its
    solo run; the small windows also pass the fp64 layer oracle on the concurrent handle."""
    t0 = time.time()
    with Fleet(FLEET) as f:
        wins, snaps = f.round([3, 6, 0, 7, 2, 5, 1, 4])
        bad = [d for i, c in enumerate(FLEET) for d in _differences(c.name, snaps[i], solos[c.name])]
        assert not bad, "\n".join(bad)
        checked = 0
        for i, c in enumerate(FLEET):
            if c.V * c.H * c.W <= FP64_MAX:
                checked += _fp64(f.hs[i], c, wins[i], "fleet " + c.name)
        assert checked > 0
    print(f"test_mixed_fleet: {time.time() - t0:.1f} s")


def test_resident_reruns_of_the_fleet(solos):
    """run_resident_multi round-robin over the fleet's handles (eight different windows on eight streams), three forwards
    each: every stage output and debug tensor still equals the solo run."""
    with Fleet(FLEET) as f:
        f.round(range(len(FLEET)))
        DrMvsnet.run_resident_multi(f.hs, 3 * len(f.hs))
        bad = []
        for i, c in enumerate(FLEET):
            ref = {k: v for k, v in solos[c.name].items() if not k.startswith("GetResult.")}
            bad += _differences("resident " + c.name, _snapshot(f.hs[i], c), ref)
        assert not bad, "\n".join(bad)


def test_slot_lifecycle(solos):
    """A ninth live handle is refused and leaves the eight intact; a destroyed handle's slot is taken by a handle with the
    other checkpoint, whose f.conv0.0 (k_conv00_u8, weights in the slot's constant bank) and whole forward pass the fp64
    oracle and equal its solo run, next to seven handles that still hold other weights."""
    with Fleet(FLEET) as f:
        with pytest.raises(TandemError):
            DrMvsnet(default_weights(W03), precision="mixed16")
        _, snaps = f.round(range(len(FLEET)))
        bad = [d for i, c in enumerate(FLEET) for d in _differences("after the refused ninth handle: " + c.name, snaps[i], solos[c.name])]
        assert not bad, "\n".join(bad)
        k = 6
        assert FLEET[k].weights == W03 and FLEET[k].precision == "mixed16"
        f.hs[k].close()
        gc.collect()
        f.hs[k] = _make(REPLACEMENT)                 # the only free slot
        f.cases[k] = REPLACEMENT
        with pytest.raises(TandemError):
            DrMvsnet(default_weights(W03), precision="mixed16")
        wins, snaps = f.round([k] + [i for i in range(len(FLEET)) if i != k])
        bad = [d for i, c in enumerate(f.cases) for d in _differences("after the slot changed hands: " + c.name, snaps[i], solos[c.name])]
        assert not bad, "\n".join(bad)
        # LG.check_forward checks f.c0_0 against ML.conv00_u8_reference with the abl04 weights first
        assert _fp64(f.hs[k], REPLACEMENT, wins[k], "slot reuse " + REPLACEMENT.name) > 0


def test_page_locked_paths():
    """Page-locked inputs (direct DMA with its own reference-first reorder) at three ref_index values, page-locked result
    maps with eager_d2h 0 and 1, and a window with some views page-locked (the staged path): each bit-identical to the
    pageable call of the same window on the same handle."""
    gc.collect()
    V, H, W = 4, 96, 128
    m = _make(Case("pl", W03, "mixed16", V, H, W, 0, 0))
    try:
        for ref in (0, 2, V - 1):
            c = Case(f"ref_index {ref}", W03, "mixed16", V, H, W, ref, 10 + ref)
            win = c.window()
            _submit(m, c, win, "pageable")
            base = _snapshot(m, c, _fetch(m, c, "pageable"))
            variants = [("pinned inputs", "pinned", "pageable", 1), ("mixed inputs", "mixed", "pageable", 1),
                        ("pinned outputs eager_d2h=1", "pageable", "pinned", 1), ("pinned outputs eager_d2h=0", "pageable", "pinned", 0),
                        ("pageable outputs eager_d2h=0", "pageable", "pageable", 0), ("pinned in + out eager_d2h=0", "pinned", "pinned", 0)]
            bad = []
            for label, inp, outp, eager in variants:
                m.set_option("eager_d2h", eager)
                _submit(m, c, win, inp)
                bad += _differences(f"ref_index {ref} {label}", _snapshot(m, c, _fetch(m, c, outp)), base)
            m.set_option("eager_d2h", 1)
            assert not bad, "\n".join(bad)
    finally:
        m.close()


# Three caller threads, each with its own handle and a different window per round (pageable inputs: concurrent copy-pool
# batches of different sizes).
THREADS = [
    [Case("T0 abl03 mixed16 128x96v2", W03, "mixed16", 2, 96, 128, 0, 21, (16, 16, 8)),
     Case("T0 abl03 mixed16 160x128v4", W03, "mixed16", 4, 128, 160, 2, 22, (16, 16, 8)),
     Case("T0 abl03 mixed16 96x64v3", W03, "mixed16", 3, 64, 96, 2, 23, (16, 16, 8))],
    [Case("T1 abl04 bf16 192x160v5", W04, "bf16", 5, 160, 192, 4, 31),
     Case("T1 abl04 bf16 64x64v2", W04, "bf16", 2, 64, 64, 1, 32),
     Case("T1 abl04 bf16 128x96v6", W04, "bf16", 6, 96, 128, 3, 33)],
    [Case("T2 abl03 fp32 96x64v3", W03, "fp32", 3, 64, 96, 1, 41, (16, 8, 8)),
     Case("T2 abl03 fp32 128x96v2", W03, "fp32", 2, 96, 128, 0, 42, (16, 8, 8)),
     Case("T2 abl03 fp32 64x64v4", W03, "fp32", 4, 64, 64, 3, 43, (16, 8, 8))],
]
ROUNDS = 6


def test_threads_drive_their_own_handles():
    """Each thread runs ROUNDS CallAsync / GetResult rounds on its handle, a different window each round, all threads
    released together into CallAsync; every result equals the solo run of its window.  The ctypes calls must release the
    GIL (else the library never sees two calls at once): a Python ticker thread has to make progress while the callers
    wait inside GetResult."""
    assert isinstance(lib(), ctypes.CDLL) and not isinstance(lib(), ctypes.PyDLL)
    assert not lib().tdm_mvsnet_get_result._flags_ & ctypes._FUNCFLAG_PYTHONAPI
    solo = {c.name: _solo(c) for cases in THREADS for c in cases}
    gc.collect()
    hs = [_make(cases[0]) for cases in THREADS]
    barrier = threading.Barrier(len(THREADS))
    results = [[] for _ in THREADS]
    spans = {"call": [], "get": []}
    errors = []
    stop = threading.Event()
    ticks = []

    def ticker():
        while not stop.is_set():
            ticks.append(time.perf_counter())
            time.sleep(2e-4)

    def drive(t):
        try:
            for r in range(ROUNDS):
                c = THREADS[t][r % len(THREADS[t])]
                win = c.window()
                barrier.wait()
                t0 = time.perf_counter()
                _submit(hs[t], c, win)
                t1 = time.perf_counter()
                out = _fetch(hs[t], c)
                t2 = time.perf_counter()
                spans["call"].append((t, t0, t1))
                spans["get"].append((t, t1, t2))
                results[t].append((c.name, _snapshot(hs[t], c, out)))
        except Exception as e:           # reported by the main thread
            errors.append(f"thread {t}: {e!r}")
            barrier.abort()

    tk = threading.Thread(target=ticker)
    workers = [threading.Thread(target=drive, args=(t,)) for t in range(len(THREADS))]
    try:
        tk.start()
        for w in workers:
            w.start()
        for w in workers:
            w.join()
    finally:
        stop.set()
        tk.join()
        for h in hs:
            h.close()
    assert not errors, "\n".join(errors)
    bad = []
    for t, res in enumerate(results):
        assert len(res) == ROUNDS
        for r, (name, S) in enumerate(res):
            bad += _differences(f"thread {t} round {r} {name}", S, solo[name])
    caught = sum(1 for t, res in enumerate(results) for r, (name, S) in enumerate(res) if _differences("", S, solo[name]))
    print(f"threads: {caught} of {len(THREADS) * ROUNDS} rounds differ from their solo run")
    assert not bad, "\n".join(bad)
    overlap = sum(1 for i, (ta, a0, a1) in enumerate(spans["call"]) for tb, b0, b1 in spans["call"][i + 1:]
                  if ta != tb and a0 < b1 and b0 < a1)
    inside = max(sum(1 for x in ticks if t1 < x < t2) for _, t1, t2 in spans["get"])
    print(f"threads: {overlap} pairs of CallAsync calls of different threads overlapped in time; at most {inside} ticker "
          f"ticks inside one GetResult")
    assert inside >= 3, "no Python thread ran while a caller waited inside GetResult: the ctypes calls hold the GIL"


def test_two_devices():
    """Handles created alternately on devices 0 and 1, device 1's first forward after device 0 has launched (the tensor-core
    kernels' shared-memory opt-in must reach every device): each equals its solo run on its own device."""
    if lib().tdm_device_count() < 2:
        pytest.skip("fewer than two CUDA devices visible")
    cases = [Case(f"D{i % 2} {c.name}", c.weights, c.precision, c.V, c.H, c.W, c.ref, c.seed, c.dn, dict(c.opts), c.inputs,
                  c.outputs, device=i % 2) for i, c in enumerate([FLEET[6], FLEET[4], FLEET[1], FLEET[3]])]
    solo = {c.name: _solo(c) for c in cases}
    gc.collect()
    hs, bad = [], []
    try:
        for c in cases:
            hs.append(_make(c))
            _submit(hs[-1], c, c.window())
            bad += _differences(c.name, _snapshot(hs[-1], c, _fetch(hs[-1], c)), solo[c.name])
        for h, c in zip(hs, cases):      # all four in flight together
            _submit(h, c, c.window())
        for h, c in reversed(list(zip(hs, cases))):
            bad += _differences("in flight together: " + c.name, _snapshot(h, c, _fetch(h, c)), solo[c.name])
    finally:
        for h in hs:
            h.close()
    assert not bad, "\n".join(bad)
