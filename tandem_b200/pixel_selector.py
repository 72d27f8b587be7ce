"""n10: DSO's pixel selection on the device (PixelSelector::makeMaps, tandem/src/FullSystem/PixelSelector2.cpp:142-291, with
makeHists and select) over the C ABI (include/tandem_b200.h, block n10).  ImmaturePoints.make_new_traces runs it together
with the ImmaturePoint constructor, as FullSystem::makeNewTraces does."""
import ctypes

import numpy as np

from ._lib import SelectResult, SelectSettings, check, lib

#: util/settings.cpp:132-135
SELECT_DEFAULTS = dict(min_grad_hist_cut=0.5, min_grad_hist_add=7.0, grad_downweight_per_level=0.75,
                       select_direction_distribution=1)


class PixelSelector:
    """One PixelSelector of a w x h camera (w // 32 and h // 32 at least 1).  Its potential (currentPotential, 3 at
    construction) carries over from call to call."""

    def __init__(self, w, h, device=0, **settings):
        unknown = set(settings) - set(SELECT_DEFAULTS)
        if unknown:
            raise TypeError(f"unknown selection settings {sorted(unknown)}")
        self.w, self.h = w, h
        self.settings = dict(SELECT_DEFAULTS, **settings)
        st = SelectSettings(**self.settings)
        self._h = ctypes.c_void_p()
        check(lib().tdm_selector_create(w, h, ctypes.byref(st), device, ctypes.byref(self._h)))

    def close(self):
        if self._h is not None:
            lib().tdm_selector_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def potential(self):
        p = ctypes.c_int()
        check(lib().tdm_selector_get_potential(self._h, ctypes.byref(p)))
        return p.value

    @potential.setter
    def potential(self, p):
        check(lib().tdm_selector_set_potential(self._h, int(p)))

    def make_maps(self, pyramid, density=1500.0, recursions_left=1, th_factor=1.0, want_map=True):
        """makeMaps on pyramid's levels 0..2 (blocking).  Returns (map (h, w) float32 of 0 / 1 / 2 / 4, or None without
        want_map; dict of tdm_select_result: num_selected (the return value), n2, n3, n4, potential_used,
        potential_after, reselected, nonuniform_cells)."""
        m = np.empty((self.h, self.w), np.float32) if want_map else None
        r = SelectResult()
        check(lib().tdm_selector_make_maps(self._h, pyramid._h, density, recursions_left, th_factor,
                                           None if m is None else m.ctypes.data_as(ctypes.POINTER(ctypes.c_float)), ctypes.byref(r)))
        return m, {f: getattr(r, f) for f, _ in SelectResult._fields_}
