"""ctypes bindings of the n7 oracle (oracle/coarse_ref_oracle.c) and of the reference's own makeCoarseDepthL0 body
(oracle/_ref/libcoarse_ref_ref.so, oracle/ref_build_coarse_ref.mk).  TEST INFRASTRUCTURE ONLY.

Both keep the reference's persistent pc_* arrays between calls (CoarseTracker's members), so consecutive keyframes see the
slots the previous one left behind, and both chain the dense block of setCoarseTrackingRef (n1: FrontOracle / FrontRef) after
makeCoarseDepthL0, as CoarseTracker::setCoarseTrackingRef does (CoarseTracker.cpp:633-733)."""
import ctypes
import os
import subprocess

import numpy as np

from oracle.cpu import FrontOracle, FrontRef

_HERE = os.path.dirname(os.path.abspath(__file__))
_fp = ctypes.POINTER(ctypes.c_float)
_ip = ctypes.POINTER(ctypes.c_int)


def build():
    subprocess.run(["make", "-s", "-C", _HERE, "-f", "coarse_ref_oracle.mk"], check=True)


class _CoarseRefBase:
    def __init__(self, w, h, levels):
        self.w, self.h, self.levels = w, h, levels
        self.sizes = [(w >> l, h >> l) for l in range(levels)]
        self.off = np.cumsum([0] + [a * b for a, b in self.sizes]).tolist()
        self.pc = np.zeros(4 * self.off[-1], np.float32)   # the reference's pc_u/v/idepth/color[l], persistent

    def level_arrays(self, l):
        n = self.sizes[l][0] * self.sizes[l][1]
        base = 4 * self.off[l]
        return [self.pc[base + k * n:base + (k + 1) * n] for k in range(4)]

    def _make_coarse_depth(self, fn, points, gray_levels, rgbd):
        n = 0 if points is None else len(points[0])
        pts = [np.zeros(1, np.float32)] * 4 if points is None else [np.ascontiguousarray(a, np.float32) for a in points]
        gray = np.concatenate([np.ascontiguousarray(g, np.float32).ravel() for g in gray_levels[:self.levels]])
        idepth = np.zeros(self.off[-1], np.float32)
        pc_n = np.zeros(self.levels, np.int32)
        rc = fn(self.w, self.h, self.levels, int(bool(rgbd)), n, *[a.ctypes.data_as(_fp) for a in pts], gray.ctypes.data_as(_fp),
                idepth.ctypes.data_as(_fp), self.pc.ctypes.data_as(_fp), pc_n.ctypes.data_as(_ip))
        if rc != 0:
            raise ValueError("a point rounds to a pixel outside the level-0 image")
        return [int(x) for x in pc_n], idepth[:self.off[1]].reshape(self.h, self.w)

    def _dense(self, pc_n, idepth0, gray0, call):
        u, v, i, c = self.level_arrays(0)
        n, arrs = call([a[:pc_n[0] + 1].copy() for a in (u, v, i, c)], idepth0, gray0)[:2]
        for dst, src in zip((u, v, i, c), arrs):
            dst[:n + 1] = src
        pc_n[0] = n
        return pc_n

    def result(self, pc_n):
        """[(u, v, idepth, color) of level l, pc_n[l] + 1 entries each (slot pc_n[l] included)]."""
        return [[a[:pc_n[l] + 1].copy() for a in self.level_arrays(l)] for l in range(self.levels)]


class CoarseRefOracle(_CoarseRefBase):
    """oracle/coarse_ref_oracle.c + FrontOracle.dense_reference."""

    def __init__(self, w, h, levels):
        super().__init__(w, h, levels)
        path = os.path.join(_HERE, "_build", "libcoarse_ref_oracle.so")
        src = os.path.join(_HERE, "coarse_ref_oracle.c")
        if not os.path.exists(path) or os.path.getmtime(path) < os.path.getmtime(src):
            build()
        self._l = ctypes.CDLL(path)
        self._l.coarse_ref_oracle.restype = ctypes.c_int

    def set_coarse_tracking_ref(self, points, gray_levels, rgbd=False, depth=None, T_depth_to_ref=None, K4=None, step=1,
                                dense_only=False):
        """points = (u, v, idepth, hessian) or None; gray_levels[l] = dIp[l][..][0] (h_l, w_l).  Returns pc_n per level."""
        pc_n, idepth0 = self._make_coarse_depth(self._l.coarse_ref_oracle, points, gray_levels, rgbd)
        if depth is not None:
            f = FrontOracle()
            pc_n = self._dense(pc_n, idepth0, gray_levels[0], lambda sp, id0, g0: f.dense_reference(
                depth, T_depth_to_ref, K4, step, dense_only, sp, id0, g0))
        return pc_n


class CoarseRefRef(_CoarseRefBase):
    """The reference's own makeCoarseDepthL0 body + its dense block (FrontRef); used by oracle/gen_reference_pins_coarse_ref.py."""

    PATH = os.path.join(_HERE, "_ref", "libcoarse_ref_ref.so")

    @classmethod
    def available(cls):
        return os.path.exists(cls.PATH) and FrontRef.available()

    def __init__(self, w, h, levels):
        super().__init__(w, h, levels)
        self._l = ctypes.CDLL(self.PATH)
        self._l.ref_make_coarse_depth.restype = ctypes.c_int

    def set_coarse_tracking_ref(self, points, gray_levels, rgbd=False, depth=None, c2w_depth=None, c2w_ref=None, K4=None, step=1,
                                dense_only=False):
        """As CoarseRefOracle, but the dense block takes the two camera poses; returns (pc_n, T_depth_to_ref or None)."""
        pc_n, idepth0 = self._make_coarse_depth(self._l.ref_make_coarse_depth, points, gray_levels, rgbd)
        T = [None]
        if depth is not None:
            f = FrontRef()

            def call(sp, id0, g0):
                n, arrs, T[0] = f.dense_reference(depth, c2w_depth, c2w_ref, K4, step, dense_only, sp, id0, g0)
                return n, arrs
            pc_n = self._dense(pc_n, idepth0, gray_levels[0], call)
        return pc_n, T[0]
