"""n10 test infrastructure: ctypes binding of oracle/pixsel_oracle.c (DSO's PixelSelector restated in C: the random pattern,
makeHists, select and makeMaps) and the cases its pins and the GPU tests run.  CPU only; no reference code.

A case is one image size and a sequence of makeMaps calls on one selector, so currentPotential carries over between calls
as it does across DSO's keyframes.  Each call names its image (RoomScene renders at the poses of oracle/trace.py, or a
synthetic image), its density, recursionsLeft and thFactor, the settings, and optionally a potential set before it (as
CoarseInitializer::setFirst sets 3).  The pyramid of each image is the pinned definition (oracle/front_oracle.c, n2)."""
import ctypes
import functools
import os
import subprocess

import numpy as np

from oracle import trace as T

_HERE = os.path.dirname(os.path.abspath(__file__))
_fp = ctypes.POINTER(ctypes.c_float)
_ip = ctypes.POINTER(ctypes.c_int)
_up = ctypes.POINTER(ctypes.c_ubyte)

SEED = 3141592   # PixelSelector::PixelSelector's std::srand
#: util/settings.cpp:132-135, in the order of pixsel_oracle.c's settings array / tdm_select_settings
DEFAULTS = dict(min_grad_hist_cut=0.5, min_grad_hist_add=7.0, grad_downweight_per_level=0.75, select_direction_distribution=1)
PATTERN_PREFIX = 4096


def settings_array(s):
    return np.array([s[k] for k in DEFAULTS], np.float32)


def _lib():
    path = os.path.join(_HERE, "_build", "libpixsel_oracle.so")
    if not os.path.exists(path) or os.path.getmtime(path) < os.path.getmtime(os.path.join(_HERE, "pixsel_oracle.c")):
        subprocess.run(["make", "-s", "-C", _HERE, "-f", "pixsel_oracle.mk"], check=True)
    return ctypes.CDLL(path)


def _p(a, t=_fp):
    return a.ctypes.data_as(t)


def pattern(n, seed=SEED):
    """rand() & 0xFF for n calls after srand(seed), glibc's generator restated (nothing touches the process's rand state)."""
    out = np.zeros(n, np.uint8)
    _lib().pixsel_oracle_pattern(ctypes.c_uint(seed), n, _p(out, _up))
    return out


def make_hists(w, h, ag0, settings=DEFAULTS):
    out = np.zeros((w // 32) * (h // 32), np.float32)
    _lib().pixsel_oracle_make_hists(w, h, _p(np.ascontiguousarray(ag0, np.float32)), _p(settings_array(settings)), _p(out))
    return out


def levels(gray):
    """The pinned pyramid's level 0 (I, dx, dy) and absSquaredGrad of levels 0..2."""
    from oracle.cpu import FrontOracle
    L = FrontOracle().make_images(np.ascontiguousarray(gray, np.float32), 3)
    return L[0][0], [L[0][1], L[1][1], L[2][1]]


class PixelSelectorOracle:
    """One PixelSelector of a w x h camera: its pattern and currentPotential (3 at construction)."""

    def __init__(self, w, h):
        self.w, self.h = w, h
        self.rp = pattern(w * h)
        self.potential = 3

    def make_maps(self, gray, density, recursions_left=1, th_factor=1.0, **settings):
        """makeMaps on the pyramid of `gray`: dict(ret, map, n (n2, n3, n4), pot_used, pot_before, pot_after, reselected,
        ties, nonuniform, selects)."""
        dI, ag = levels(gray)
        return self.make_maps_on(dI, ag, density, recursions_left, th_factor, **settings)

    def make_maps_on(self, dI, ag, density, recursions_left=1, th_factor=1.0, **settings):
        """make_maps on a pyramid's level 0 (I, dx, dy) and absSquaredGrad of levels 0..2 (levels())."""
        s = dict(DEFAULTS, **settings)
        ths = make_hists(self.w, self.h, ag[0], s)
        m = np.zeros((self.h, self.w), np.float32)
        info = np.zeros(8, np.int32)
        pot = ctypes.c_int(self.potential)
        before = self.potential
        ags = [np.ascontiguousarray(a, np.float32) for a in ag]
        ret = _lib().pixsel_oracle_make_maps(self.w, self.h, _p(np.ascontiguousarray(dI, np.float32)), _p(ags[0]), _p(ags[1]),
                                             _p(ags[2]), _p(ths), _p(self.rp, _up), _p(settings_array(s)), ctypes.byref(pot),
                                             ctypes.c_float(density), int(recursions_left), ctypes.c_float(th_factor), _p(m),
                                             _p(info, _ip))
        self.potential = pot.value
        return dict(ret=ret, map=m, n=info[:3].copy(), pot_used=int(info[3]), pot_before=before, pot_after=pot.value,
                    reselected=int(info[4]), ties=int(info[5]), nonuniform=int(info[6]), selects=int(info[7]))


def selected(m):
    """(flat indices in raster order, types) of a selection map."""
    idx = np.flatnonzero(m.ravel() != 0).astype(np.int32)
    return idx, m.ravel()[idx].astype(np.float32)


def new_traces(m, w, h):
    """makeNewTraces' loop (FullSystem.cpp:1634-1646, patternPadding 2): the map entries of [3, w-4) x [3, h-4) in raster
    order, as (u, v, type)."""
    sub = m[3:h - 4, 3:w - 4]
    ys, xs = np.nonzero(sub != 0)
    return (xs + 3).astype(np.int32), (ys + 3).astype(np.int32), sub[ys, xs].astype(np.float32)


# ---- images ----
def room(k, h, w):
    return T.gray(T.pose(k), h, w).astype(np.float32)


def steps(h, w, seed=0):
    """Integer axis-aligned steps and ramps: many pixels have dx == 0 or dy == 0 (their score is 0 under direction (1, 0)
    or (0, 1), so their cell's selection depends on its direction) and equal scores (tied maxima)."""
    y, x = np.mgrid[0:h, 0:w]
    g = 60.0 * ((x // 9) % 2) + 40.0 * ((y // 13) % 2) + 2.0 * (x % 6) * ((y // 29) % 2) + 3.0 * (y % 5) * ((x // 23) % 2)
    rng = np.random.default_rng(seed)
    blobs = rng.integers(0, 2, (h // 17 + 1, w // 17 + 1)) * 50.0
    g += blobs[y // 17, x // 17]
    return g.astype(np.float32)


def with_nan(g, seed=0):
    g = g.copy()
    rng = np.random.default_rng(seed)
    h, w = g.shape
    g[rng.integers(0, h, 60), rng.integers(0, w, 60)] = np.nan
    return g


def image(spec, h, w):
    kind, arg = spec
    if kind == "room":
        return room(arg, h, w)
    if kind == "room_nan":
        return with_nan(room(arg, h, w), arg)
    if kind == "steps":
        return steps(h, w, arg)
    if kind == "steps_nan":
        return with_nan(steps(h, w, arg), arg)
    if kind == "flat":
        return np.full((h, w), float(arg), np.float32)
    raise ValueError(kind)


def call(img, density=1500.0, rec=1, th=1.0, pot=None, **settings):
    return dict(img=img, density=density, rec=rec, th=th, pot=pot, settings=settings)


# name -> ((h, w), [calls]); one selector per case, the potential carried from call to call
CASES = {
    "room_640x480_sequence": ((480, 640), [call(("room", k)) for k in range(6)]),
    "room_640x480_densities": ((480, 640), [call(("room", 0), 6000.0), call(("room", 0), 100.0), call(("room", 1), 1e6, rec=2),
                                            call(("room", 1), 1500.0, rec=0), call(("room", 2), 300.0, rec=2),
                                            call(("room", 2), 1500.0, select_direction_distribution=0)]),
    "room_752x480": ((480, 752), [call(("room", 0)), call(("room", 3)), call(("room", 4), 0.03 * 752 * 480, th=2.0, pot=3),
                                  call(("room_nan", 5), 1500.0)]),
    "room_331x247": ((247, 331), [call(("room", 1)), call(("room", 2), 700.0), call(("room", 2), 0.03 * 331 * 247, th=2.0, pot=3),
                                  call(("room_nan", 3), 2000.0, rec=2), call(("room", 4), 0.0)]),
    "steps_331x247": ((247, 331), [call(("steps", 0)), call(("steps", 1), 4000.0), call(("steps_nan", 2), 800.0, rec=2),
                                   call(("steps", 3), 1500.0, pot=1), call(("steps", 4), 1500.0, select_direction_distribution=0)]),
    "steps_96x72": ((72, 96), [call(("steps", 5), 200.0), call(("steps", 6), 50.0), call(("steps", 7), 400.0, rec=2, pot=1),
                               call(("steps", 8), 200.0, th=2.0, pot=3)]),
    "flat_96x72": ((72, 96), [call(("flat", 100.0), 200.0), call(("flat", 100.0), 0.0), call(("steps", 9), 0.0, rec=0),
                              call(("flat", 7.0), 200.0, rec=0)]),
}


@functools.lru_cache(maxsize=None)
def case_images(name):
    (h, w), calls = CASES[name]
    return [image(c["img"], h, w) for c in calls]


def run_oracle(name):
    """The oracle's makeMaps results of every call of a case, in order."""
    (h, w), calls = CASES[name]
    o = PixelSelectorOracle(w, h)
    out = []
    for c, g in zip(calls, case_images(name)):
        if c["pot"] is not None:
            o.potential = c["pot"]
        out.append(o.make_maps(g, c["density"], c["rec"], c["th"], **c["settings"]))
    return out
