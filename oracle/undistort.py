"""n11 test infrastructure: ctypes binding of oracle/undistort_oracle.c (PhotometricUndistorter's constructor, processFrame,
Undistort::undistort's remap, the BGR remap, setGammaFunction and the gamma-weighted makeImages restated in C) and the cases
its pins and the GPU tests run.  CPU only; no reference code.

A case is one camera (raw and rectified sizes, remap tables from a RadTan-style distortion or passthrough, response and
vignette, settings), a sequence of Binv given to setGammaFunction before the frames, and a sequence of raw frames with their
exposure and factor.  The frames are RoomScene renders quantised to 8 bits."""
import ctypes
import functools
import os
import subprocess

import numpy as np

from oracle.pins_coarse_ref import GRAY_W, K4
from oracle import trace as T
from tandem_b200.synthetic import RoomScene

_HERE = os.path.dirname(os.path.abspath(__file__))
_fp = ctypes.POINTER(ctypes.c_float)
_up = ctypes.POINTER(ctypes.c_ubyte)
_sp = ctypes.POINTER(ctypes.c_ushort)


def _lib():
    path = os.path.join(_HERE, "_build", "libundistort_oracle.so")
    srcs = [os.path.join(_HERE, f) for f in ("undistort_oracle.c", "front_oracle.c")]
    if not os.path.exists(path) or os.path.getmtime(path) < max(os.path.getmtime(s) for s in srcs):
        subprocess.run(["make", "-s", "-C", _HERE, "-f", "undistort_oracle.mk"], check=True)
    l = ctypes.CDLL(path)
    l.undistort_oracle_frame.restype = ctypes.c_float
    return l


def _p(a, t=_fp):
    return None if a is None else a.ctypes.data_as(t)


# ---- inputs ----
def remap_tables(w_org, h_org, w, h, k1=-0.28, k2=0.07, p1=4e-4, p2=-3e-4):
    """Undistort's tables (w*h each): each rectified pixel through a RadTan distortion into the raw frame; entries whose
    footprint leaves the raw frame are -1 (the reference's intent, 0 < x < w_org - 1 and 0 < y < h_org - 1)."""
    fx_o, fy_o, cx_o, cy_o = 0.62 * w_org, 0.83 * h_org, 0.5 * w_org - 0.3, 0.5 * h_org + 0.2
    fx, fy, cx, cy = 0.55 * w, 0.74 * h, 0.5 * w + 0.1, 0.5 * h - 0.4
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    xn, yn = (x - cx) / fx, (y - cy) / fy
    r2 = xn * xn + yn * yn
    rad = 1 + k1 * r2 + k2 * r2 * r2
    xd = xn * rad + 2 * p1 * xn * yn + p2 * (r2 + 2 * xn * xn)
    yd = yn * rad + p1 * (r2 + 2 * yn * yn) + 2 * p2 * xn * yn
    ix, iy = (fx_o * xd + cx_o).astype(np.float32), (fy_o * yd + cy_o).astype(np.float32)
    ok = (ix > 0) & (iy > 0) & (ix < w_org - 1) & (iy < h_org - 1)
    return np.where(ok, ix, -1).astype(np.float32).ravel(), np.where(ok, iy, -1).astype(np.float32).ravel()


def response(kind):
    """The first line of a photometric calibration file (G before normalisation)."""
    n = 1024 if kind == "long" else 256
    i = np.arange(n, dtype=np.float64)
    g = (3.1 + 1000.0 * (i / (n - 1)) ** 1.7 + 0.37 * i).astype(np.float32)
    if kind == "not_increasing":
        g[100] = g[99]
    return g


def vignette(kind, w, h):
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    r2 = ((x - 0.5 * w) / w) ** 2 + ((y - 0.5 * h) / h) ** 2
    v = np.clip(1.0 - 1.1 * r2, 0.2, 1.0)
    if kind == "v8":
        return np.round(250.0 * v).astype(np.uint16).ravel()
    out = np.round(60000.0 * v).astype(np.uint16)
    if kind == "v16_zero":
        out[h // 3:h // 3 + 2, w // 4:w // 4 + 3] = 0
        out[2 * h // 3, 2 * w // 3] = 0
        out[1, 1] = 0
    return out.ravel()


def binv(kind, G):
    """A Binv for setGammaFunction: the camera's own G, or G with plateaus (equal neighbours, one exactly on an integer)
    scaled so that B entries above 191 are not found."""
    if kind == "G":
        return G.astype(np.float32).copy()
    b = (G.astype(np.float32) * np.float32(0.75)).astype(np.float32)
    b[40:60] = b[40]
    b[1:4] = np.float32(1.0)
    b[120:123] = np.float32(round(float(b[120])))
    return b


@functools.lru_cache(maxsize=None)
def render(w, h, k):
    bgr, _ = RoomScene().render(T.pose(k), h, w, *K4(h, w))
    bgr = np.ascontiguousarray(bgr, np.uint8)
    gray = np.clip(np.round(bgr.astype(np.float32) @ GRAY_W), 0, 255).astype(np.uint8)
    return gray, bgr


def frame_inputs(case, k):
    """(gray (h_org, w_org) uint8, bgr (h_org, w_org, 3) uint8) of frame k of a case."""
    c = CASES[case]
    gray, bgr = render(c["w_org"], c["h_org"], c["frames"][k][2])
    gray = gray.copy()
    if c.get("dark_spots"):
        gray[c["h_org"] // 3, c["w_org"] // 4:c["w_org"] // 4 + 3] = 0   # raw 0 on vignette 0: G[0] * inf = NaN
    return gray, bgr


def case(w_org, h_org, w, h, remap=True, resp="gamma", vig="v16", mode=2, use_exposure=1, gamma_weights=1, gammas=("G",),
         frames=((10.0, 1.0, 0), (20.0, 1.0, 1)), levels=3, select=False, dark_spots=False):
    return dict(w_org=w_org, h_org=h_org, w=w, h=h, remap=remap, resp=resp, vig=vig, mode=mode, use_exposure=use_exposure,
                gamma_weights=gamma_weights, gammas=gammas, frames=frames, levels=levels, select=select, dark_spots=dark_spots)


# name -> case; frames are (exposure, factor, render index).  Cases up to 103 x 79 are pinned as full arrays, larger ones as
# digests.  The selection of frame 0 is pinned on the cases with select.
CASES = {
    "tum_640x480_mode2": case(640, 480, 640, 480, levels=5, select=True),
    "euroc_752to640_mode1": case(752, 480, 640, 480, resp="long", vig="v8", mode=1, gammas=("G", "plateau"), levels=5,
                                 select=True),
    "down_97x75to91x67_mode0": case(97, 75, 91, 67, mode=0, gammas=("G", "plateau"),
                                    frames=((5.0, 1.0, 2), (0.0, 2.5, 3))),
    "up_91x67to103x79_noexp": case(91, 67, 103, 79, use_exposure=0, gammas=("plateau", "G"),
                                   frames=((-1.0, 0.7, 4), (3.0, 1.0, 5))),
    "invalid_response": case(80, 60, 72, 56, resp="not_increasing", gammas=(), frames=((10.0, 1.3, 0),)),
    "missing_vignette": case(80, 60, 72, 56, vig=None, gammas=("plateau",), frames=((10.0, 1.0, 1),)),
    "vignette_zero_passthrough": case(64, 48, 64, 48, remap=False, vig="v16_zero", dark_spots=True, frames=((10.0, 1.0, 2),)),
    "vignette_zero_remap": case(80, 60, 72, 56, vig="v16_zero", dark_spots=True, frames=((12.0, 1.0, 3),)),
    "passthrough_mode1_unweighted": case(96, 72, 96, 72, remap=False, vig="v8", mode=1, gamma_weights=0,
                                         frames=((10.0, 1.0, 4), (-2.0, 1.5, 5))),
}


def full(name):
    c = CASES[name]
    return c["w"] * c["h"] <= 103 * 79


def camera(name):
    """The create arguments of a case: dict(remap_x, remap_y, response, vignette) (None where absent)."""
    c = CASES[name]
    rx = ry = None
    if c["remap"]:
        rx, ry = remap_tables(c["w_org"], c["h_org"], c["w"], c["h"])
    return dict(remap_x=rx, remap_y=ry, response=response(c["resp"]) if c["resp"] else None,
                vignette=vignette(c["vig"], c["w_org"], c["h_org"]) if c["vig"] else None)


# ---- oracle ----
def create(name):
    """(valid, G (256 float32), vinv) of a case's camera."""
    c, cam = CASES[name], camera(name)
    G = np.zeros(256, np.float32)
    vinv = np.zeros(c["w_org"] * c["h_org"], np.float32)
    r, v = cam["response"], cam["vignette"]
    valid = _lib().undistort_oracle_create(_p(r), 0 if r is None else r.size, _p(v, _sp), c["w_org"] * c["h_org"], c["mode"],
                                           _p(G), _p(vinv))
    return bool(valid), G, vinv


def set_gamma(binv_arr, B):
    B = np.array(B, np.float32)
    _lib().undistort_oracle_set_gamma(_p(np.ascontiguousarray(binv_arr, np.float32)), _p(B))
    return B


def gamma_sequence(name, G):
    """The Binv arrays a case gives setGammaFunction, in order, and the B after them."""
    B = np.arange(256, dtype=np.float32)
    seq = []
    for kind in CASES[name]["gammas"]:
        b = binv(kind, G)
        seq.append(b)
        B = set_gamma(b, B)
    return seq, B


def make_images(gray, levels, B):
    g = np.ascontiguousarray(gray, np.float32)
    h, w = g.shape
    tot = sum((w >> l) * (h >> l) for l in range(levels))
    dI = np.zeros(3 * tot, np.float32)
    ag = np.zeros(tot, np.float32)
    _lib().undistort_oracle_make_images(_p(g), w, h, levels, _p(None if B is None else np.ascontiguousarray(B, np.float32)),
                                        _p(dI), _p(ag))
    out, off = [], 0
    for l in range(levels):
        wl, hl = w >> l, h >> l
        out.append((dI[3 * off:3 * (off + wl * hl)].reshape(hl, wl, 3), ag[off:off + wl * hl].reshape(hl, wl)))
        off += wl * hl
    return out


def run_oracle(name):
    """dict(valid, G, B, binv (list), frames: [dict(exposure_time, image (h, w), bgr (h, w, 3), levels [(dI, ag)])])."""
    c, cam = CASES[name], camera(name)
    valid, G, vinv = create(name)
    seq, B = gamma_sequence(name, G)
    frames = []
    scratch = np.zeros(c["w_org"] * c["h_org"], np.float32)
    for k, (exposure, factor, _) in enumerate(c["frames"]):
        gray, bgr = frame_inputs(name, k)
        img = np.zeros((c["h"], c["w"]), np.float32)
        t = _lib().undistort_oracle_frame(_p(gray, _up), c["w_org"], c["h_org"], c["w"], c["h"], _p(cam["remap_x"]),
                                          _p(cam["remap_y"]), int(valid), c["mode"], c["use_exposure"], _p(G), _p(vinv),
                                          ctypes.c_float(exposure), ctypes.c_float(factor), _p(scratch), _p(img))
        bo = np.zeros((c["h"], c["w"], 3), np.uint8)
        _lib().undistort_oracle_bgr(_p(bgr, _up), c["w_org"], c["h_org"], c["w"], c["h"], _p(cam["remap_x"]), _p(cam["remap_y"]),
                                    _p(bo, _up))
        frames.append(dict(exposure_time=np.float32(t), image=img, bgr=bo,
                           levels=make_images(img, c["levels"], B if c["gamma_weights"] else None)))
    return dict(valid=valid, G=G, B=B, binv=seq, frames=frames)


def digest(a):
    return T.digest(a)


def matches_pin(g, key, a):
    """a equals pin `key` of an npz: the full array (NaN equal to NaN), or its digest under key + "_digest"."""
    a = np.asarray(a)
    if key in g.files:
        return a.shape == g[key].shape and np.array_equal(a, g[key], equal_nan=a.dtype.kind == "f")
    return digest(a) == str(g[key + "_digest"])


def frame_mismatches(g, name, k, exposure_time, image, bgr, levels):
    """The names of the pinned outputs of frame k of a case that the given ones do not equal ([] when all match); levels is
    [(dI (h_l, w_l, 3), absSquaredGrad (h_l, w_l))] for every level."""
    pre = f"{name}_f{k}_"
    bad = []
    if np.float32(exposure_time) != g[pre + "exposure_time"]:
        bad.append("exposure_time")
    if not matches_pin(g, pre + "image", image):
        bad.append("image")
    if bgr is not None and not matches_pin(g, pre + "bgr", bgr):
        bad.append("bgr")
    for l, (d, a) in enumerate(levels):
        if not matches_pin(g, pre + f"dI{l}", d):
            bad.append(f"dI{l}")
        if not matches_pin(g, pre + f"ag{l}", a):
            bad.append(f"ag{l}")
    return bad


def pinned_selection_map(g, name, w, h):
    """The reference's selection map of frame 0 of a case with `select`."""
    m = np.zeros(w * h, np.float32)
    m[g[f"{name}_f0_select_index"]] = g[f"{name}_f0_select_type"]
    return m.reshape(h, w)
