"""ctypes bindings of the C oracles (oracle/tsdf_oracle.c, oracle/tracker_oracle.c).  TEST INFRASTRUCTURE ONLY:
imported by tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs."""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_BUILD = os.path.join(_HERE, "_build")


def build():
    subprocess.run(["make", "-s", "-C", _HERE], check=True)


def _load(name):
    path = os.path.join(_BUILD, name)
    src = os.path.join(_HERE, name[3:].replace(".so", ".c"))
    if not os.path.exists(path) or os.path.getmtime(path) < os.path.getmtime(src):
        build()
    return ctypes.CDLL(path)


class _Options(ctypes.Structure):
    _fields_ = [("voxel_size", ctypes.c_float), ("num_buckets", ctypes.c_int), ("bucket_size", ctypes.c_int),
                ("num_blocks", ctypes.c_int), ("block_size", ctypes.c_int), ("max_sdf_weight", ctypes.c_int),
                ("truncation_distance", ctypes.c_float), ("max_sensor_depth", ctypes.c_float),
                ("min_sensor_depth", ctypes.c_float), ("num_render_streams", ctypes.c_int),
                ("fx", ctypes.c_float), ("fy", ctypes.c_float), ("cx", ctypes.c_float), ("cy", ctypes.c_float),
                ("height", ctypes.c_int), ("width", ctypes.c_int)]


VOXEL_DTYPE = np.dtype([("sdf", "<f4"), ("color", "u1", (3,)), ("weight", "u1")])
_fp = ctypes.POINTER(ctypes.c_float)
_dp = ctypes.POINTER(ctypes.c_double)


class TsdfOracle:
    def __init__(self, options):
        """options: any ctypes struct with DrFusionOptions' fields (e.g. tandem_b200._lib.FusionOptions)."""
        self._l = _load("libtsdf_oracle.so")
        self._l.tsdf_oracle_create.restype = ctypes.c_void_p
        self._l.tsdf_oracle_dump.restype = ctypes.c_long
        o = _Options()
        for f, _ in _Options._fields_:
            setattr(o, f, getattr(options, f))
        self.o = o
        self._h = ctypes.c_void_p(self._l.tsdf_oracle_create(ctypes.byref(o)))

    def __del__(self):
        try:
            self._l.tsdf_oracle_destroy(self._h)
        except Exception:
            pass

    def integrate(self, bgr, depth, pose):
        bgr = np.ascontiguousarray(bgr, np.uint8)
        depth = np.ascontiguousarray(depth, np.float32)
        pose = np.ascontiguousarray(pose, np.float32)
        rc = self._l.tsdf_oracle_integrate(self._h, ctypes.c_void_p(bgr.ctypes.data), depth.ctypes.data_as(_fp),
                                           pose.ctypes.data_as(_fp))
        assert rc == 0

    def render(self, pose):
        pose = np.ascontiguousarray(pose, np.float32)
        bgr = np.zeros((self.o.height, self.o.width, 3), np.uint8)
        depth = np.zeros((self.o.height, self.o.width), np.float32)
        self._l.tsdf_oracle_render(self._h, pose.ctypes.data_as(_fp), ctypes.c_void_p(bgr.ctypes.data),
                                   depth.ctypes.data_as(_fp))
        return bgr, depth

    def stats(self):
        out = (ctypes.c_long * 5)()
        self._l.tsdf_oracle_stats(self._h, out)
        return dict(allocated_blocks=out[0], visible_blocks=out[1], dropped_blocks=out[2], candidate_blocks=out[3],
                    render_distinct_voxels=out[4])

    def extract_mesh(self, lower, upper):
        """Brute-force marching cubes over the box (mesh_extractor.cu:244-265) -> (vert (n,3), cols (n,3) rgb)."""
        lo = np.ascontiguousarray(lower, np.float32)
        up = np.ascontiguousarray(upper, np.float32)
        self._l.tsdf_oracle_extract_mesh.restype = ctypes.c_long
        n = self._l.tsdf_oracle_extract_mesh(self._h, lo.ctypes.data_as(_fp), up.ctypes.data_as(_fp), None, None, ctypes.c_long(0))
        vert = np.empty((n, 3), np.float32)
        cols = np.empty((n, 3), np.float32)
        m = self._l.tsdf_oracle_extract_mesh(self._h, lo.ctypes.data_as(_fp), up.ctypes.data_as(_fp), vert.ctypes.data_as(_fp),
                                             cols.ctypes.data_as(_fp), ctypes.c_long(n))
        assert m == n
        return vert, cols

    def dump_blocks(self):
        n = self.stats()["allocated_blocks"]
        coords = np.empty((n, 3), np.int32)
        vox = np.empty((n, 512), VOXEL_DTYPE)
        m = self._l.tsdf_oracle_dump(self._h, ctypes.c_void_p(coords.ctypes.data), ctypes.c_void_p(vox.ctypes.data),
                                     ctypes.c_long(n))
        assert m == n
        return coords, vox


class _TrkCfg(ctypes.Structure):
    _fields_ = [("w", ctypes.c_int), ("h", ctypes.c_int), ("fx", ctypes.c_float), ("fy", ctypes.c_float),
                ("cx", ctypes.c_float), ("cy", ctypes.c_float), ("huber", ctypes.c_float)]


class TrackerOracle:
    """Same call surface as tandem_b200.CudaCoarseTracker, evaluated by oracle/tracker_oracle.c."""

    def __init__(self, w, h, setting_huberTH=9.0, setting_coarseCutoffTH=20.0):
        self._l = _load("libtracker_oracle.so")
        self.cfg = _TrkCfg(w, h, 0, 0, 0, 0, setting_huberTH)

    def setK(self, w, h, fx, fy, cx, cy):
        self.cfg.fx, self.cfg.fy, self.cfg.cx, self.cfg.cy = fx, fy, cx, cy

    def setReference(self, n, pc_u, pc_v, pc_idepth, pc_color, ref_exposure, ref_aff_g2l):
        f = lambda a: np.ascontiguousarray(a, np.float32)
        self.n, self.u, self.v, self.idepth, self.color = n, f(pc_u), f(pc_v), f(pc_idepth), f(pc_color)
        self.ref_exposure, self.ref_aff = float(ref_exposure), np.ascontiguousarray(ref_aff_g2l, np.float64)

    def setNew(self, dInew):
        self.dI = np.ascontiguousarray(dInew, np.float32)

    def _aff(self, new_exposure, aff):
        out = (ctypes.c_float * 2)()
        aff = np.ascontiguousarray(aff, np.float64)
        self._l.tracker_oracle_affll(ctypes.c_float(self.ref_exposure), ctypes.c_float(new_exposure),
                                     self.ref_aff.ctypes.data_as(_dp), aff.ctypes.data_as(_dp), out)
        return out

    def calcRes(self, refToNew, new_exposure, aff_g2l, cutoffTH):
        T = np.ascontiguousarray(refToNew, np.float64)
        aff = self._aff(new_exposure, aff_g2l)
        self.warped = np.zeros((7, self.n), np.float32)
        out7 = np.zeros(7, np.float64)
        self._l.tracker_oracle_calc_res(ctypes.byref(self.cfg), T.ctypes.data_as(_dp), aff, ctypes.c_float(cutoffTH),
                                        self.n, self.u.ctypes.data_as(_fp), self.v.ctypes.data_as(_fp),
                                        self.idepth.ctypes.data_as(_fp), self.color.ctypes.data_as(_fp),
                                        self.dI.ctypes.data_as(_fp), self.warped.ctypes.data_as(_fp),
                                        out7.ctypes.data_as(_dp))
        self.out7 = out7
        res6 = np.zeros(6, np.float64)
        self._l.tracker_oracle_res6(out7.ctypes.data_as(_dp), res6.ctypes.data_as(_dp))
        return res6

    def calcG(self, new_exposure, aff_g2l):
        aff = self._aff(new_exposure, aff_g2l)
        acc = np.zeros(45, np.float64)
        H = np.zeros((8, 8), np.float64)
        b = np.zeros(8, np.float64)
        self._l.tracker_oracle_calc_g(ctypes.byref(self.cfg), aff, ctypes.c_float(self.ref_aff[1]), self.n,
                                      self.color.ctypes.data_as(_fp), self.warped.ctypes.data_as(_fp),
                                      int(self.out7[2]), acc.ctypes.data_as(_dp), H.ctypes.data_as(_dp),
                                      b.ctypes.data_as(_dp))
        return H, b


class FrontOracle:
    """oracle/front_oracle.c: image pyramid + gradients (n2) and the dense tracking reference (n1)."""

    def __init__(self):
        self._l = _load("libfront_oracle.so")
        self._l.front_oracle_dense_reference.restype = ctypes.c_int

    def make_images(self, gray, levels):
        g = np.ascontiguousarray(gray, np.float32)
        h, w = g.shape
        tot = sum((w >> l) * (h >> l) for l in range(levels))
        dI = np.zeros(3 * tot, np.float32)
        ag = np.zeros(tot, np.float32)
        self._l.front_oracle_make_images(g.ctypes.data_as(_fp), w, h, levels, dI.ctypes.data_as(_fp), ag.ctypes.data_as(_fp))
        out, off = [], 0
        for l in range(levels):
            wl, hl = w >> l, h >> l
            out.append((dI[3 * off:3 * (off + wl * hl)].reshape(hl, wl, 3), ag[off:off + wl * hl].reshape(hl, wl)))
            off += wl * hl
        return out

    def krki(self, T, fx, fy, cx, cy):
        T = np.ascontiguousarray(T, np.float64)
        a, b = np.zeros(9, np.float32), np.zeros(3, np.float32)
        self._l.front_oracle_krki(T.ctypes.data_as(_dp), ctypes.c_float(fx), ctypes.c_float(fy), ctypes.c_float(cx),
                                  ctypes.c_float(cy), a.ctypes.data_as(_fp), b.ctypes.data_as(_fp))
        return a, b

    def dense_reference(self, depth, T_depth_to_ref, K4, step, dense_only, sparse, idepth0, ref_gray):
        """sparse = (pc_u, pc_v, pc_idepth, pc_color) with n_before + 1 entries each (last = stale slot) or None."""
        d = np.ascontiguousarray(depth, np.float32)
        h, w = d.shape
        krki, kt = self.krki(T_depth_to_ref, *K4)
        nb = 0 if sparse is None else len(sparse[0]) - 1
        arrs = [np.zeros(nb + 1 + w * h, np.float32) for _ in range(4)]
        if sparse is not None:
            for a, s in zip(arrs, sparse):
                a[:nb + 1] = s
        proj = np.zeros(w * h, np.float32)
        id0 = None if idepth0 is None else np.ascontiguousarray(idepth0, np.float32)
        rg = np.ascontiguousarray(ref_gray, np.float32)
        n = self._l.front_oracle_dense_reference(
            d.ctypes.data_as(_fp), w, h, int(step), krki.ctypes.data_as(_fp), kt.ctypes.data_as(_fp), int(bool(dense_only)), nb,
            None if id0 is None else id0.ctypes.data_as(_fp), rg.ctypes.data_as(_fp), arrs[0].ctypes.data_as(_fp),
            arrs[1].ctypes.data_as(_fp), arrs[2].ctypes.data_as(_fp), arrs[3].ctypes.data_as(_fp), proj.ctypes.data_as(_fp))
        return n, [a[:n + 1] for a in arrs], proj.reshape(h, w)


class FrontRef:
    """oracle/_ref/libfront_ref.so: the REFERENCE's own makeImages / setCoarseTrackingRef bodies (HessianBlocks.cpp:128-191,
    CoarseTracker.cpp:655-725) compiled from where they lie by oracle/ref_build.mk; used by oracle/gen_reference_pins.py."""

    PATH = os.path.join(_HERE, "_ref", "libfront_ref.so")

    @classmethod
    def available(cls):
        return os.path.exists(cls.PATH)

    def __init__(self):
        self._l = ctypes.CDLL(self.PATH)
        self._l.ref_front_make_images.restype = ctypes.c_int
        self._l.ref_front_dense_reference.restype = ctypes.c_int

    def make_images(self, gray, levels):
        g = np.ascontiguousarray(gray, np.float32)
        h, w = g.shape
        tot = sum((w >> l) * (h >> l) for l in range(levels))
        dI = np.zeros(3 * tot, np.float32)
        ag = np.zeros(tot, np.float32)
        rc = self._l.ref_front_make_images(g.ctypes.data_as(_fp), w, h, levels, dI.ctypes.data_as(_fp), ag.ctypes.data_as(_fp))
        assert rc == 0
        out, off = [], 0
        for l in range(levels):
            wl, hl = w >> l, h >> l
            out.append((dI[3 * off:3 * (off + wl * hl)].reshape(hl, wl, 3), ag[off:off + wl * hl].reshape(hl, wl)))
            off += wl * hl
        return out

    def dense_reference(self, depth, c2w_depth, c2w_ref, K4, step, dense_only, sparse, idepth0, ref_gray):
        """Same contract as FrontOracle.dense_reference, but takes the two camera poses (the reference derives
        T_dense_depth_to_last itself, CoarseTracker.cpp:673); also returns that transform (4x4 double)."""
        d = np.ascontiguousarray(depth, np.float32)
        h, w = d.shape
        nb = 0 if sparse is None else len(sparse[0]) - 1
        arrs = [np.zeros(nb + 1 + w * h, np.float32) for _ in range(4)]
        if sparse is not None:
            for a, s in zip(arrs, sparse):
                a[:nb + 1] = s
        id0 = None if idepth0 is None else np.ascontiguousarray(idepth0, np.float32)
        rg = np.ascontiguousarray(ref_gray, np.float32)
        cd = np.ascontiguousarray(c2w_depth, np.float32)
        cr = np.ascontiguousarray(c2w_ref, np.float64)
        T = np.zeros(16, np.float64)
        n = self._l.ref_front_dense_reference(
            d.ctypes.data_as(_fp), w, h, int(step), cd.ctypes.data_as(_fp), cr.ctypes.data_as(_dp), ctypes.c_float(K4[0]),
            ctypes.c_float(K4[1]), ctypes.c_float(K4[2]), ctypes.c_float(K4[3]), int(bool(dense_only)), nb,
            None if id0 is None else id0.ctypes.data_as(_fp), rg.ctypes.data_as(_fp), arrs[0].ctypes.data_as(_fp),
            arrs[1].ctypes.data_as(_fp), arrs[2].ctypes.data_as(_fp), arrs[3].ctypes.data_as(_fp), T.ctypes.data_as(_dp))
        return n, [a[:n + 1] for a in arrs], T.reshape(4, 4)
