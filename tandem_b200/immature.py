"""n8: DSO's immature points of the active keyframes kept in device memory and traced into each new frame
(FullSystem::traceNewCoarse, FullSystem.cpp:650-691; ImmaturePoint::traceOn, ImmaturePoint.cpp:75-414) over the C ABI
(include/tandem_b200.h, block n8); n9: their activation solve (FullSystem::optimizeImmaturePoint,
FullSystemOptPoint.cpp:51-205, for activatePointsMT's candidates); n10: a new keyframe's points selected and constructed on the
device (FullSystem::makeNewTraces, FullSystem.cpp:1623-1647)."""
import ctypes

import numpy as np

from ._lib import ActivateSettings, SelectResult, TraceSettings, check, lib

_fp = ctypes.POINTER(ctypes.c_float)
_ip = ctypes.POINTER(ctypes.c_int)

#: util/settings.cpp:84-148
TRACE_DEFAULTS = dict(max_pix_search=0.027, trace_stepsize=1.0, trace_gn_threshold=0.1, trace_extra_slack_on_th=1.2,
                      trace_slack_interval=1.5, trace_min_improvement_factor=2.0, huber_th=9.0, outlier_th=144.0,
                      outlier_th_sum_component=2500.0, overall_energy_th_weight=1.0, min_trace_test_radius=2,
                      trace_gn_iterations=3)
#: util/settings.cpp:62, 142 and activatePointsMT_Reductor's minObs
ACTIVATE_DEFAULTS = dict(min_idepth_h_act=100.0, gn_iterations=3, min_obs=1)
#: ImmaturePoint::lastTraceStatus
IPS_GOOD, IPS_OOB, IPS_OUTLIER, IPS_SKIPPED, IPS_BADCONDITION, IPS_UNINITIALIZED = range(6)
FIELDS = {"u": (), "v": (), "type": (), "energy_th": (), "color": (8,), "weights": (8,), "grad_h": (4,), "idepth_min": (),
          "idepth_max": (), "quality": (), "status": (), "uv": (2,), "interval": ()}


def _p(a, t=_fp):
    return None if a is None else a.ctypes.data_as(t)


class ImmaturePoints:
    """The immature points of up to 8 host keyframes (slots 0..7, capacity_per_host each) of one w x h camera."""

    def __init__(self, w, h, capacity_per_host, device=0, **settings):
        unknown = set(settings) - set(TRACE_DEFAULTS)
        if unknown:
            raise TypeError(f"unknown trace settings {sorted(unknown)}")
        self.w, self.h = w, h
        self._capacity = capacity_per_host
        self.settings = dict(TRACE_DEFAULTS, **settings)
        st = TraceSettings(**self.settings)
        self._h = ctypes.c_void_p()
        check(lib().tdm_immature_create(w, h, capacity_per_host, ctypes.byref(st), device, ctypes.byref(self._h)))

    def close(self):
        if self._h is not None:
            lib().tdm_immature_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def add(self, slot, host_pyramid, u, v, type=None):
        """The constructor for the pixels (u, v) of host_pyramid's level 0; returns how many points were kept."""
        u = np.ascontiguousarray(u, np.int32)
        v = np.ascontiguousarray(v, np.int32)
        t = np.ones(len(u), np.float32) if type is None else np.ascontiguousarray(type, np.float32)
        if not (len(u) == len(v) == len(t)):
            raise ValueError("u, v and type differ in length")
        n = ctypes.c_int()
        check(lib().tdm_immature_add(self._h, slot, host_pyramid._h, len(u), _p(u, _ip), _p(v, _ip), _p(t), ctypes.byref(n)))
        return n.value

    def trace(self, frame_pyramid, slots, KRKi, Kt, aff, host_pyramids=None):
        """traceOn of every point of `slots` into frame_pyramid's level 0 (asynchronous).  KRKi (n, 3, 3), Kt (n, 3) and
        aff (n, 2) per slot."""
        slots = np.ascontiguousarray(slots, np.int32).ravel()
        n = len(slots)
        K = np.ascontiguousarray(KRKi, np.float32).reshape(n, 9)
        t = np.ascontiguousarray(Kt, np.float32).reshape(n, 3)
        a = np.ascontiguousarray(aff, np.float32).reshape(n, 2)
        hp = None
        if host_pyramids is not None:
            hp = (ctypes.c_void_p * n)(*[None if p is None else p._h.value for p in host_pyramids])
        check(lib().tdm_immature_trace(self._h, frame_pyramid._h, n, _p(slots, _ip), hp, _p(K), _p(t), _p(a)))

    def make_new_traces(self, slot, selector, pyramid, density=1500.0):
        """makeNewTraces: selector.make_maps on pyramid (recursions 1, thFactor 1) and the constructor for every selected pixel
        of [3, w-4) x [3, h-4), appended to the slot in raster order; the map stays on the device.  Blocking.  Returns
        dict(n_added, u, v, type (the kept points), result (PixelSelector.make_maps' dict))."""
        free = self._capacity - self.count(slot)
        u, v = np.empty(max(free, 0), np.int32), np.empty(max(free, 0), np.int32)
        t = np.empty(max(free, 0), np.float32)
        r, n = SelectResult(), ctypes.c_int()
        check(lib().tdm_immature_make_new_traces(self._h, slot, selector._h, pyramid._h, density, ctypes.byref(r), ctypes.byref(n),
                                                 _p(u, _ip), _p(v, _ip), _p(t)))
        k = n.value
        return dict(n_added=k, u=u[:k].copy(), v=v[:k].copy(), type=t[:k].copy(),
                    result={f: getattr(r, f) for f, _ in SelectResult._fields_})

    def count(self, slot):
        c = ctypes.c_int()
        check(lib().tdm_immature_get(self._h, slot, 0, 0, ctypes.byref(c), *([None] * 13)))
        return c.value

    def get(self, slot, first=0, n=None):
        """dict of every field (FIELDS) of points first..first+n-1 of a slot (all of them by default); synchronises."""
        if n is None:
            n = self.count(slot) - first
        out = {k: np.empty((n,) + s, np.int32 if k == "status" else np.float32) for k, s in FIELDS.items()}
        c = ctypes.c_int()
        check(lib().tdm_immature_get(self._h, slot, first, n, ctypes.byref(c), *[
            _p(out[k], _ip if k == "status" else _fp) for k in FIELDS]))
        return out

    def remove(self, slot, indices):
        """Removes points the way activatePointsMT compacts host->immaturePoints (FullSystem.cpp:849-856)."""
        idx = np.ascontiguousarray(indices, np.int32).ravel()
        check(lib().tdm_immature_remove(self._h, slot, len(idx), _p(idx, _ip)))

    def drop_host(self, slot):
        check(lib().tdm_immature_drop_host(self._h, slot))

    def activate(self, frame_slots, frame_pyramids, precalc, calib, cand_frame, cand_index, min_idepth_h_act=100.0,
                 gn_iterations=3, min_obs=1):
        """optimizeImmaturePoint for every candidate (point cand_index[k] of frame cand_frame[k]'s slot) over the frames of
        frameHessians: frame_slots[f] is frame f's slot or -1, frame_pyramids[f] its pyramid, precalc (n, n, 14) holds
        [host][target] PRE_RTll (row-major), PRE_tTll and PRE_aff_mode, calib (fxl, fyl, cxl, cyl).  Blocking.  Returns
        dict(result (n_cand,) int32 1 / 0 / -1, idepth (n_cand,) float32, res_state (n_cand, n_frames) int8 with -1 in the
        host's column, res_energy (n_cand, n_frames) float32 with NaN there)."""
        slots = np.ascontiguousarray(frame_slots, np.int32).ravel()
        n = len(slots)
        if len(frame_pyramids) != n:
            raise ValueError("frame_slots and frame_pyramids differ in length")
        pc = np.ascontiguousarray(precalc, np.float32)
        if pc.size != n * n * 14:
            raise ValueError("precalc must hold n_frames x n_frames x 14 floats")
        cal = np.ascontiguousarray(calib, np.float32).ravel()
        if cal.size != 4:
            raise ValueError("calib must hold fxl, fyl, cxl, cyl")
        cf = np.ascontiguousarray(cand_frame, np.int32).ravel()
        ci = np.ascontiguousarray(cand_index, np.int32).ravel()
        if len(cf) != len(ci):
            raise ValueError("cand_frame and cand_index differ in length")
        k = len(cf)
        out = dict(result=np.empty(k, np.int32), idepth=np.empty(k, np.float32), res_state=np.empty((k, n), np.int8),
                   res_energy=np.empty((k, n), np.float32))
        fp = (ctypes.c_void_p * max(n, 1))(*[None if p is None else p._h.value for p in frame_pyramids])
        st = ActivateSettings(min_idepth_h_act=min_idepth_h_act, gn_iterations=gn_iterations, min_obs=min_obs)
        check(lib().tdm_immature_activate(self._h, n, _p(slots, _ip), fp, _p(pc), _p(cal), ctypes.byref(st), k, _p(cf, _ip),
                                          _p(ci, _ip), _p(out["result"], _ip), _p(out["idepth"]),
                                          _p(out["res_state"], ctypes.POINTER(ctypes.c_byte)), _p(out["res_energy"])))
        return out
