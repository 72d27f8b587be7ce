"""ctypes bindings of the nodia oracle (coarse_nodia_oracle / idepth_quantile_oracle in oracle/coarse_nodia_oracle.c) and of the
reference's own makeCoarseDepthL0 body with persistent pc_*_nodia and its get_idepth_quantile (oracle/_ref/libcoarse_nodia_ref.so,
oracle/ref_build_coarse_nodia.mk), plus the runs over the cases of oracle/pins_coarse_ref.py.  TEST INFRASTRUCTURE ONLY.

Both sides keep pc_u/v/idepth/color_nodia (w*h floats each, CoarseTracker's members) between the keyframes of a case, so a
keyframe sees the slots the previous one left behind."""
import ctypes
import os
import subprocess

import numpy as np

from oracle import pins_coarse_ref as P
from oracle.coarse_ref import _CoarseRefBase

_HERE = os.path.dirname(os.path.abspath(__file__))

_fp = ctypes.POINTER(ctypes.c_float)


def build():
    subprocess.run(["make", "-s", "-C", _HERE, "-f", "coarse_nodia_oracle.mk"], check=True)


def last_index_fraction(n):
    """A float32 fraction whose index (int)(fraction * (float)n) is n - 1 (0.5 for n == 0, where no index is valid)."""
    if n == 0:
        return np.float32(0.5)
    f = np.float32((n - 0.5) / n)
    assert int(np.float32(f * np.float32(n))) == n - 1, n
    return f


def fractions(n):
    """The quantile fractions the pins check for a cloud of n: the smallest entry, the one deliverDrFrame uses (0.2), the
    largest, and 1 (index n: NaN)."""
    return np.array([0.0, 0.2, last_index_fraction(n), 1.0], np.float32)


class _NodiaBase:
    def __init__(self, w, h):
        self.w, self.h = w, h
        self.nodia = np.zeros(4 * w * h, np.float32)   # pc_u/v/idepth/color_nodia, persistent

    def result(self, n):
        """(u, v, idepth, color) of the first n entries."""
        m = self.w * self.h
        return [self.nodia[k * m:k * m + n].copy() for k in range(4)]

    def quantile(self, n, fraction):
        """(idepth, depth) float32 of get_idepth_quantile over the first n pc_idepth_nodia entries; NaN where it has none."""
        out = np.zeros(2, np.float32)
        ids = np.ascontiguousarray(self.nodia[2 * self.w * self.h:2 * self.w * self.h + max(n, 1)])
        self._quantile(n, ids.ctypes.data_as(_fp), ctypes.c_float(fraction), out.ctypes.data_as(_fp))
        return out


class CoarseNodiaOracle(_NodiaBase):
    """oracle/coarse_nodia_oracle.c: coarse_nodia_oracle + idepth_quantile_oracle."""

    def __init__(self, w, h):
        super().__init__(w, h)
        path = os.path.join(_HERE, "_build", "libcoarse_nodia_oracle.so")
        src = os.path.join(_HERE, "coarse_nodia_oracle.c")
        if not os.path.exists(path) or os.path.getmtime(path) < os.path.getmtime(src):
            build()
        self._l = ctypes.CDLL(path)
        self._l.coarse_nodia_oracle.restype = ctypes.c_int
        self._l.idepth_quantile_oracle.restype = None
        self._quantile = self._l.idepth_quantile_oracle

    def make(self, points, gray0, rgbd=False):
        """points = (u, v, idepth, hessian) or None, as CoarseRefOracle; gray0 = dIp[0][..][0] (h, w).  Returns pc_n_nodia."""
        n = 0 if points is None else len(points[0])
        pts = [np.zeros(1, np.float32)] * 4 if points is None else [np.ascontiguousarray(a, np.float32) for a in points]
        g = np.ascontiguousarray(gray0, np.float32)
        cnt = ctypes.c_int()
        rc = self._l.coarse_nodia_oracle(self.w, self.h, int(bool(rgbd)), n, *[a.ctypes.data_as(_fp) for a in pts],
                                         g.ctypes.data_as(_fp), self.nodia.ctypes.data_as(_fp), ctypes.byref(cnt))
        if rc != 0:
            raise ValueError("a point rounds to a pixel outside the level-0 image")
        return cnt.value


class CoarseNodiaRef(_NodiaBase):
    """The reference's own makeCoarseDepthL0 (all levels, pc_*_nodia persistent) and get_idepth_quantile
    (oracle/ref_wrap_coarse_nodia.cpp); used by oracle/gen_reference_pins_coarse_nodia.py."""

    PATH = os.path.join(_HERE, "_ref", "libcoarse_nodia_ref.so")

    def __init__(self, w, h, levels):
        super().__init__(w, h)
        self._base = _CoarseRefBase(w, h, levels)   # packs the points and the grey pyramid as the n7 pin does
        self._l = ctypes.CDLL(self.PATH)
        self._l.ref_make_coarse_depth_nodia.restype = ctypes.c_int
        self._l.ref_idepth_quantile.restype = None
        self._quantile = self._l.ref_idepth_quantile

    def make(self, points, gray_levels, rgbd=False):
        """As CoarseNodiaOracle.make, with every level's grey image (the reference runs the whole function)."""
        cnt = ctypes.c_int()

        def fn(w, h, levels, rgbd_, n, pu, pv, pid, phs, gray, _idepth, _pc, _pc_n):
            return self._l.ref_make_coarse_depth_nodia(w, h, levels, rgbd_, n, pu, pv, pid, phs, gray,
                                                       self.nodia.ctypes.data_as(_fp), ctypes.byref(cnt))
        self._base._make_coarse_depth(fn, points, gray_levels, rgbd)
        return cnt.value


def run_oracle(name):
    """Runs the case's keyframes through the nodia oracle; per keyframe (pc_n_nodia, the four arrays including slot
    pc_n_nodia, the fractions, their (idepth, depth) quantiles (len(fractions), 2))."""
    (h, w), levels, gray_levels, _, kfs = P.case_inputs(name)
    o = CoarseNodiaOracle(w, h)
    out = []
    for kf in kfs:
        m = o.make(kf["points"], gray_levels[0], kf["rgbd"])
        fr = fractions(m)
        out.append((m, o.result(m + 1), fr, np.stack([o.quantile(m, f) for f in fr])))
    return out
