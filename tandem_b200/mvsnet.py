"""Host-side mirror of `class DrMvsnet` (tandem/libdr/dr_mvsnet/src/dr_mvsnet/dr_mvsnet.h:36-66) over the C ABI.

Same method names, argument meaning and blocking behaviour as the reference class:
    m = DrMvsnet("path/to/model.pt" | "weights.tdmw")
    m.CallAsync(height, width, view_num, ref_index, bgrs, intrinsic_matrix, cam_to_worlds, dmin, dmax, discard)
    out = m.GetResult()      # DrMvsnetOutput with .depth .confidence .depth_dense .confidence_dense (H,W) float32
"""
import ctypes
import os

import numpy as np

from ._lib import TandemError, check, lib, pinned_empty

_WEIGHTS_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "weights")
PRECISION = {"fp32": 0, "mixed16": 1, "bf16": 2}


def default_weights(name="abl03_view_aggregation"):
    return os.path.join(_WEIGHTS_DIR, name + ".tdmw")


class DrMvsnetOutput:
    """dr_mvsnet.h:12-34."""

    def __init__(self, height, width, pinned=False):
        """pinned=True: the four maps live in page-locked memory (GetResult(out=...) then DMA's straight into them)."""
        self.height, self.width = height, width
        mk = (lambda: pinned_empty((height, width), np.float32)) if pinned else (lambda: np.empty((height, width), np.float32))
        self.depth, self.confidence, self.depth_dense, self.confidence_dense = mk(), mk(), mk(), mk()


class DrMvsnet:
    def __init__(self, filename, precision="mixed16", device=0):
        self._h = ctypes.c_void_p()
        check(lib().tdm_mvsnet_create(os.fsencode(filename), PRECISION[precision], device, ctypes.byref(self._h)))
        self._hw = None

    def close(self):
        if getattr(self, "_h", None):
            lib().tdm_mvsnet_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_option(self, key, value):
        check(lib().tdm_mvsnet_set_option(self._h, key.encode(), int(value)))

    def _call(self, fn, height, width, view_num, ref_index, bgrs, K, cam_to_worlds, dmin, dmax, discard):
        bgrs = [np.ascontiguousarray(b, dtype=np.uint8) for b in bgrs]
        c2ws = [np.ascontiguousarray(c, dtype=np.float32) for c in cam_to_worlds]
        if len(bgrs) != view_num or len(c2ws) != view_num:
            raise TandemError("view_num does not match the number of images / poses")
        for b in bgrs:
            if b.size != height * width * 3:
                raise TandemError("bgr image has the wrong size")
        K = np.ascontiguousarray(K, dtype=np.float32)
        bp = (ctypes.c_void_p * view_num)(*[b.ctypes.data for b in bgrs])
        cp = (ctypes.c_void_p * view_num)(*[c.ctypes.data for c in c2ws])
        check(fn(self._h, height, width, view_num, ref_index, bp, K.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), cp,
                 float(dmin), float(dmax), float(discard)))
        self._hw = (height, width)

    def CallAsync(self, height, width, view_num, ref_index, bgrs, intrinsic_matrix, cam_to_worlds, depth_min,
                  depth_max, discard_percentage, debug_print=False):
        """Blocking for the last input, non-blocking for this input (dr_mvsnet.h:42)."""
        self._call(lib().tdm_mvsnet_call_async, height, width, view_num, ref_index, bgrs,
                   np.asarray(intrinsic_matrix, np.float32).reshape(9), cam_to_worlds, depth_min, depth_max,
                   discard_percentage)

    def CallAsyncStageK(self, height, width, view_num, ref_index, bgrs, K_stages, cam_to_worlds, depth_min,
                        depth_max, discard_percentage):
        """Like CallAsync but with explicit per-stage intrinsics (stage1..3) as the Python model receives them."""
        self._call(lib().tdm_mvsnet_call_async_k, height, width, view_num, ref_index, bgrs,
                   np.asarray(K_stages, np.float32).reshape(27), cam_to_worlds, depth_min, depth_max,
                   discard_percentage)

    def CallAsyncIds(self, height, width, view_num, ref_index, view_ids, bgrs, intrinsics, cam_to_worlds, depth_min,
                     depth_max, discard_percentage, stage_k=False):
        """CallAsync with the feature cache (tdm_mvsnet_call_async_ids): view_ids[i] names view i; FeatureNet runs only
        for ids the handle does not hold.  bgrs[i] may be None for a held id (and is ignored for one).  intrinsics: the
        3x3 full-resolution K, or with stage_k=True the three per-stage K's of CallAsyncStageK."""
        if len(view_ids) != view_num or len(bgrs) != view_num or len(cam_to_worlds) != view_num:
            raise TandemError("view_num does not match the number of ids / images / poses")
        imgs = [None if b is None else np.ascontiguousarray(b, dtype=np.uint8) for b in bgrs]
        for b in imgs:
            if b is not None and b.size != height * width * 3:
                raise TandemError("bgr image has the wrong size")
        c2ws = [np.ascontiguousarray(c, dtype=np.float32) for c in cam_to_worlds]
        K = np.ascontiguousarray(np.asarray(intrinsics, np.float32).reshape(27 if stage_k else 9))
        ids = (ctypes.c_longlong * view_num)(*[int(i) for i in view_ids])
        bp = (ctypes.c_void_p * view_num)(*[None if b is None else b.ctypes.data for b in imgs])
        cp = (ctypes.c_void_p * view_num)(*[c.ctypes.data for c in c2ws])
        check(lib().tdm_mvsnet_call_async_ids(self._h, height, width, view_num, ref_index, ids, bp,
                                              K.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), int(bool(stage_k)), cp,
                                              float(depth_min), float(depth_max), float(discard_percentage)))
        self._hw = (height, width)

    def feature_cache(self):
        """(ids held in the last window's order, views FeatureNet computed for the last call)."""
        n = ctypes.c_int()
        nc = ctypes.c_int()
        check(lib().tdm_mvsnet_feature_cache(self._h, None, 0, ctypes.byref(n), ctypes.byref(nc)))
        ids = (ctypes.c_longlong * max(n.value, 1))()
        check(lib().tdm_mvsnet_feature_cache(self._h, ids, n.value, ctypes.byref(n), ctypes.byref(nc)))
        return [int(ids[i]) for i in range(n.value)], nc.value

    def GetResult(self, out=None):
        """Returns a fresh DrMvsnetOutput (the reference's ownership contract, dr_mvsnet.h:12-34), or fills `out` - a
        DrMvsnetOutput the caller recycles, e.g. DrMvsnetOutput(h, w, pinned=True) for a zero-copy read-back."""
        if self._hw is None:
            raise TandemError("GetResult before CallAsync")
        o = out if out is not None else DrMvsnetOutput(*self._hw)
        if (o.height, o.width) != tuple(self._hw):
            raise TandemError("GetResult(out=...): output has the wrong size")
        fp = ctypes.POINTER(ctypes.c_float)
        check(lib().tdm_mvsnet_get_result(self._h, o.depth.ctypes.data_as(fp), o.confidence.ctypes.data_as(fp),
                                          o.depth_dense.ctypes.data_as(fp), o.confidence_dense.ctypes.data_as(fp)))
        return o

    def Wait(self):
        check(lib().tdm_mvsnet_wait(self._h))

    def Ready(self):
        return bool(check(lib().tdm_mvsnet_ready(self._h)))

    # ---- introspection used by tests / bench -------------------------------------------------
    def stage_output(self, stage, which):
        h, w = self._hw
        sc = 1 << (3 - stage)
        out = np.empty((h // sc, w // sc), np.float32)
        check(lib().tdm_mvsnet_stage_output(self._h, stage, which.encode(),
                                            out.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), out.size))
        return out

    def debug_tensor(self, name):
        dims = (ctypes.c_int * 4)()
        n = check(lib().tdm_mvsnet_debug_tensor(self._h, name.encode(), None, 0, dims))
        out = np.empty(tuple(dims), np.float32)
        check(lib().tdm_mvsnet_debug_tensor(self._h, name.encode(), out.ctypes.data_as(ctypes.POINTER(ctypes.c_float)),
                                            n, dims))
        return out

    def run_resident(self, iters):
        ms = ctypes.c_float()
        nl = ctypes.c_int()
        check(lib().tdm_mvsnet_run_resident(self._h, iters, ctypes.byref(ms), ctypes.byref(nl)))
        return ms.value, nl.value

    def run_resident_new(self, n_new, iters):
        """run_resident with FeatureNet recomputing only the last n_new views of the last window."""
        ms = ctypes.c_float()
        nl = ctypes.c_int()
        check(lib().tdm_mvsnet_run_resident_new(self._h, n_new, iters, ctypes.byref(ms), ctypes.byref(nl)))
        return ms.value, nl.value

    @staticmethod
    def run_resident_multi(handles, iters_total):
        """iters_total resident forwards round-robin over several handles of one device, one CUDA-event clock."""
        arr = (ctypes.c_void_p * len(handles))(*[h._h.value for h in handles])
        ms = ctypes.c_float()
        nl = ctypes.c_int()
        check(lib().tdm_mvsnet_run_resident_multi(arr, len(handles), iters_total, ctypes.byref(ms), ctypes.byref(nl)))
        return ms.value, nl.value

    def profile(self):
        buf = ctypes.create_string_buffer(1 << 16)
        check(lib().tdm_mvsnet_profile(self._h, buf, len(buf)))
        rows = []
        for line in buf.value.decode().splitlines():
            name, ms, b, fl = line.split()
            rows.append((name, float(ms), int(b), int(fl)))
        return rows
