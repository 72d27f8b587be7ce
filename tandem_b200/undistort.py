"""n11: DSO's per-frame input on the device (PhotometricUndistorter::processFrame, Undistort::undistort's remap, the dataset
reader's BGR remap and makeImages' gamma weights, tandem/src/util/Undistort.cpp) over the C ABI (include/tandem_b200.h,
block n11).  The raw 8-bit frame goes in; the frame's ImagePyramid comes out."""
import ctypes

import numpy as np

from ._lib import UndistortSettings, check, lib

_fp = ctypes.POINTER(ctypes.c_float)


class Undistorter:
    """One camera's undistortion: remap tables (w*h each, -1 outside; None for both: passthrough), the photometric
    calibration's response (its first line, G before normalisation) and vignette (w_org*h_org, 8- or 16-bit), and the
    camera's gamma state B (identity until set_gamma)."""

    def __init__(self, w_org, h_org, w, h, remap_x=None, remap_y=None, response=None, vignette=None, photometric_calibration=2,
                 use_exposure=True, gamma_weights=True, device=0):
        self.w_org, self.h_org, self.w, self.h = w_org, h_org, w, h
        # the library copies every array during create; these only need to live until then
        rx = None if remap_x is None else np.ascontiguousarray(remap_x, np.float32).ravel()
        ry = None if remap_y is None else np.ascontiguousarray(remap_y, np.float32).ravel()
        g = None if response is None else np.ascontiguousarray(response, np.float32).ravel()
        v = None if vignette is None else np.ascontiguousarray(vignette, np.uint16).ravel()
        for a, n, what in ((rx, w * h, "remap_x"), (ry, w * h, "remap_y"), (v, w_org * h_org, "vignette")):
            if a is not None and a.size != n:
                raise ValueError(f"{what} needs {n} entries, got {a.size}")
        s = UndistortSettings(w_org=w_org, h_org=h_org, w=w, h=h,
                              remap_x=None if rx is None else rx.ctypes.data_as(_fp),
                              remap_y=None if ry is None else ry.ctypes.data_as(_fp),
                              response=None if g is None else g.ctypes.data_as(_fp), n_response=0 if g is None else g.size,
                              vignette=None if v is None else v.ctypes.data_as(ctypes.POINTER(ctypes.c_ushort)),
                              photometric_calibration=int(photometric_calibration), use_exposure=int(bool(use_exposure)),
                              gamma_weights=int(bool(gamma_weights)))
        self._h = ctypes.c_void_p()
        check(lib().tdm_undistort_create(ctypes.byref(s), device, ctypes.byref(self._h)))

    def close(self):
        if self._h is not None:
            lib().tdm_undistort_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def get_gamma(self):
        """PhotometricUndistorter::getG(): the normalised G[0..255] (float32), or None when the calibration is not valid."""
        G = np.zeros(256, np.float32)
        valid = ctypes.c_int()
        check(lib().tdm_undistort_get_gamma(self._h, G.ctypes.data_as(_fp), ctypes.byref(valid)))
        return G if valid.value else None

    def set_gamma(self, binv):
        """FullSystem::setGammaFunction(binv) on this camera's B; None is a no-op."""
        b = None if binv is None else np.ascontiguousarray(binv, np.float32)
        if b is not None and b.size != 256:
            raise ValueError("binv needs 256 entries")
        check(lib().tdm_undistort_set_gamma(self._h, None if b is None else b.ctypes.data_as(_fp)))

    def frame(self, gray, exposure, pyramid, factor=1.0, bgr=None, bgr_out=None):
        """processFrame + remap + makeImages of the raw (h_org, w_org) uint8 frame into `pyramid` (asynchronous, ordered
        like ImagePyramid.build).  With bgr ((h_org, w_org, 3) uint8) the colour frame is remapped too, into bgr_out (a
        (h, w, 3) uint8 array, page-locked or not) or a new array.  Returns (exposure_time, the remapped BGR or None)."""
        g = np.ascontiguousarray(gray, np.uint8)
        if g.size != self.w_org * self.h_org:
            raise ValueError(f"gray needs {self.w_org * self.h_org} pixels, got {g.size}")
        b = out = None
        if bgr is not None:
            b = np.ascontiguousarray(bgr, np.uint8)
            if b.size != 3 * self.w_org * self.h_org:
                raise ValueError("bgr needs h_org x w_org x 3 bytes")
            out = np.empty((self.h, self.w, 3), np.uint8) if bgr_out is None else bgr_out
            if out.dtype != np.uint8 or out.size != 3 * self.w * self.h or not out.flags["C_CONTIGUOUS"]:
                raise ValueError("bgr_out must be a contiguous uint8 array of h x w x 3")
        t = ctypes.c_float()
        check(lib().tdm_undistort_frame(self._h, g.ctypes.data, float(exposure), float(factor), pyramid._h, ctypes.byref(t),
                                        None if b is None else b.ctypes.data, None if out is None else out.ctypes.data))
        return t.value, out
