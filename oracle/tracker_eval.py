"""fp64 restatement of the coarse tracker's evaluation (k_tracker<MODE>, tandem_b200/csrc/tracker.cu) with an a-priori error
bound on every output.  TEST INFRASTRUCTURE ONLY.

What is exact and what is bounded:
  * The host parameters (Ki, RKi, affLL, maxEnergy) and the per-point projection (pt, p1, u, v, Ku, Kv, nid and the flow
    statistics' a, c, d) are restated in float32 numpy operations, one rounding per operation as the kernel's __f*_rn
    intrinsics: u, v, Ku, Kv, nid and with them the in-frame / nid > 0 decision are bit-identical to the device's.
  * Everything nvcc may contract (the bilinear fetch, the flow terms, the energy, the 45 products of calcG) is evaluated in
    fp64 from those fp32 values; the device's result must lie within a bound made of
      - the per-point term error: a few units of 2^-24 times the absolute sub-terms of each contracted expression,
      - the per-thread fp32 accumulation over ceil(n / 67584) points (264 CTAs x 256 threads stride over the points),
      - a (negligible) term for the fp64 reductions.
  * The 45 G sums are taken over per-point values handed in (the device's own warped buffers): calcG reads exactly those.
    The fused kernel recomputes them, so its bound adds the bilinear error of the per-point check (`g_sums(..., pert=...)`).
A point whose fp64 |res| lies within the residual bound of the cutoff may be decided either way; such points are `excused`
and counted, and every bound that depends on the decision covers both outcomes.
"""
import math

import numpy as np

F32 = np.float32
U = 2.0 ** -24            # fp32 unit roundoff
UD = 2.0 ** -53           # fp64 unit roundoff
GRID = 264 * 256          # k_tracker threads: point i is accumulated by thread i % GRID
SCALE = np.array([1.0, 1.0, 1.0, 0.5, 0.5, 0.5, 10.0, 1000.0])
PAIRS = [(j1, j2) for j1 in range(9) for j2 in range(j1, 9)]        # the kernel's order of the 45 products
RED = 600 * UD            # fp64 reductions: warp shuffles, 8 warps, 264 CTAs (and numpy's pairwise sums here)


def _f(x):
    return F32(x)


class Params:
    """The host-side float parameters of one evaluation, as TrackerImpl::set_k / prepare / set_aff compute them."""

    def __init__(self, w, h, fx, fy, cx, cy, huber, refToNew, cutoff, ref_exposure, new_exposure, ref_aff, new_aff):
        self.w, self.h = int(w), int(h)
        self.fx, self.fy, self.cx, self.cy = _f(fx), _f(fy), _f(cx), _f(cy)
        fxd, fyd, cxd, cyd = float(self.fx), float(self.fy), float(self.cx), float(self.cy)
        self.Ki = np.array([1.0 / fxd, 0, -cxd / fxd, 0, 1.0 / fyd, -cyd / fyd, 0, 0, 1], np.float64).astype(F32)
        T = np.asarray(refToNew, np.float64).reshape(4, 4)
        R = T[:3, :3].astype(F32)
        self.t = T[:3, 3].astype(F32)
        RKi = np.zeros(9, F32)
        for r in range(3):
            for q in range(3):
                s = F32(0)
                for k in range(3):
                    s = F32(s + F32(R[r, k] * self.Ki[3 * k + q]))
                RKi[3 * r + q] = s
        self.RKi = RKi
        eF, eT = float(_f(ref_exposure)), float(_f(new_exposure))
        if eF == 0 or eT == 0:
            eF = eT = 1.0
        ra, na = np.asarray(ref_aff, np.float64), np.asarray(new_aff, np.float64)
        a = math.exp(na[0] - ra[0]) * eT / eF
        self.affa, self.affb = _f(a), _f(na[1] - a * ra[1])
        self.ref_b = _f(ra[1])
        self.huber, self.cutoff = _f(huber), _f(cutoff)
        self.maxE = F32(F32(F32(F32(2) * self.huber) * self.cutoff) - F32(self.huber * self.huber))


def project(P, pc_u, pc_v, pc_idepth):
    """Per-point fp32 projection, bit for bit as the kernel does it."""
    x, y, id_ = (np.asarray(a, F32) for a in (pc_u, pc_v, pc_idepth))
    with np.errstate(all="ignore"):
        pt = [F32(0)] * 3
        for r in range(3):
            pt[r] = (P.RKi[3 * r] * x + P.RKi[3 * r + 1] * y) + P.RKi[3 * r + 2] * F32(1)
        p1 = [pt[r] + P.t[r] * id_ for r in range(3)]
        u, v = p1[0] / p1[2], p1[1] / p1[2]
        Ku, Kv = P.fx * u + P.cx, P.fy * v + P.cy
        nid = id_ / p1[2]
    inframe = (Ku > 2) & (Kv > 2) & (Ku < P.w - 3) & (Kv < P.h - 3) & (nid > 0)
    return dict(x=x, y=y, id=id_, pt=pt, p1=p1, u=u, v=v, Ku=Ku, Kv=Kv, nid=nid, inframe=inframe)


def _huber_w(r, h):
    a = np.abs(r)
    with np.errstate(all="ignore"):
        return np.where(a < h, 1.0, h / a)


def _energy(r, h):
    a = np.abs(r)
    return np.where(a < h, a * a, 2 * h * a - h * h)


class Eval:
    """calcRes of one pose in fp64 with bounds.  Per point (n): the projection (see project), hit (n, 3) fp64 bilinear fetch
    at the fp32 Ku, Kv (NaN outside the frame), bil (n, 3) its bound against the device's fetch, res / res_b, the decisions
    finite / sat / accepted and excused.  Outputs: res6 and res6_b (bounds), counts nE / nW / nS, out7."""

    def __init__(self, P, pc_u, pc_v, pc_idepth, pc_color, dI):
        n = len(pc_u)
        self.P, self.n = P, n
        self.m = max(1, -(-n // GRID))
        pr = project(P, pc_u, pc_v, pc_idepth)
        self.pr = pr
        color = np.asarray(pc_color, F32)
        self.color = color
        dI = np.asarray(dI, F32).reshape(P.h, P.w, 3)
        inf = pr["inframe"]
        hit = np.full((n, 3), np.nan)
        bil = np.zeros((n, 3))
        idx = np.nonzero(inf)[0]
        if idx.size:
            Ku, Kv = pr["Ku"][idx].astype(np.float64), pr["Kv"][idx].astype(np.float64)
            ix, iy = pr["Ku"][idx].astype(np.int64), pr["Kv"][idx].astype(np.int64)
            dx, dy = Ku - ix, Kv - iy
            c = [dI[iy, ix].astype(np.float64), dI[iy, ix + 1].astype(np.float64), dI[iy + 1, ix].astype(np.float64),
                 dI[iy + 1, ix + 1].astype(np.float64)]
            wts = [(1 - dx) * (1 - dy), dx * (1 - dy), (1 - dx) * dy, dx * dy]
            with np.errstate(all="ignore"):
                hit[idx] = sum(w[:, None] * ck for w, ck in zip(wts, c))
                sabs = sum(np.abs(ck) for ck in c)
            # exact at integer positions (weights 1, 0, 0, 0); otherwise weight roundings (<= 4u each) + the 4-term sum
            exact = (dx == 0) & (dy == 0)
            bil[idx] = np.where(exact[:, None], 0.0, 16 * U * sabs + 8 * UD * sabs)
        self.hit, self.bil = hit, bil
        with np.errstate(all="ignore"):
            c32 = P.affa * color + P.affb                       # fp32, as __fadd_rn(__fmul_rn(affa, refc), affb)
            res = hit[:, 0] - c32.astype(np.float64)
        self.res = res
        # res = __fsub_rn(hit, c): with an exact fetch the device's res is res rounded to fp32 (0 error if representable)
        with np.errstate(all="ignore"):
            rnd = np.abs(np.nan_to_num(res.astype(F32).astype(np.float64) - res))
        self.res_b = np.where(bil[:, 0] == 0, rnd, bil[:, 0] + U * (np.abs(np.nan_to_num(res)) + bil[:, 0]))
        h, cut = float(P.huber), float(P.cutoff)
        self.finite = inf & np.isfinite(hit[:, 0])
        ar = np.abs(np.where(self.finite, res, 0.0))
        self.sat = self.finite & (ar > cut)
        self.accepted = self.finite & ~self.sat
        self.excused = self.finite & (self.res_b > 0) & (np.abs(ar - cut) <= self.res_b)
        self.n_excused = int(self.excused.sum())
        self.hw = np.where(self.accepted, _huber_w(res, h), 0.0)
        self.nE, self.nW, self.nS = int(self.finite.sum()), int(self.accepted.sum()), int(self.sat.sum())
        self._stats()

    def _stats(self):
        P, h = self.P, float(self.P.huber)
        maxE = float(P.maxE)
        acc, exc = self.accepted, self.excused
        r = np.where(self.finite, self.res, 0.0)
        dr = np.where(self.finite, self.res_b, 0.0)
        ar = np.abs(r)
        e = np.where(acc, _energy(r, h), np.where(self.sat, maxE, 0.0))
        # e = hw r^2 (2 - hw): Lipschitz 2 min(|r|, huber) in r; <= 6 roundings (hw included) of terms <= 3 hw r^2
        hwm = _huber_w(np.maximum(ar - dr, 0.0), h)
        L = 2 * np.minimum(ar + dr, h)
        eb = np.where(acc, L * dr + 18 * U * hwm * (ar + dr) ** 2, 0.0)
        # an excused point may land on the other side of the cutoff: maxEnergy instead of its energy, or the reverse
        eb = eb + np.where(exc, np.abs(_energy(r, h)) + abs(maxE) + L * dr + 18 * U * (ar + dr) ** 2, 0.0)
        E = float(np.sum(e))
        Eb = float(np.sum(eb) + 1.01 * self.m * U * np.sum(np.abs(e) + eb) + RED * np.sum(np.abs(e)))
        self.point_energy, self.point_energy_b = e, eb
        # flow statistics on every 32nd point (kernel: i % 32 == 0)
        pr = self.pr
        fi = np.arange(0, self.n, 32)
        x, y, id_ = pr["x"][fi], pr["y"][fi], pr["id"][fi]
        s4 = np.zeros(fi.size)
        b4 = np.zeros(fi.size)
        s5 = np.zeros(fi.size)
        b5 = np.zeros(fi.size)
        with np.errstate(all="ignore"):
            ptK = [(P.Ki[3 * r] * x + P.Ki[3 * r + 1] * y) + P.Ki[3 * r + 2] * F32(1) for r in range(3)]
            tid = [P.t[r] * id_ for r in range(3)]
            a = [ptK[r] + tid[r] for r in range(3)]
            c = [ptK[r] - tid[r] for r in range(3)]
            d = [pr["pt"][r][fi] - tid[r] for r in range(3)]
            fx, fy, cx, cy = (float(q) for q in (P.fx, P.fy, P.cx, P.cy))

            def kproj(num, den, f, cc):                    # f * (num / den) + cc, contracted or not
                q = (num / den).astype(np.float64)
                return f * q + cc, 2 * U * (np.abs(f * q) + abs(cc))

            def sq(K, dK, ref):
                dd = K - ref.astype(np.float64)
                e = dK + U * (np.abs(dd) + dK)
                return dd * dd, 2 * np.abs(dd) * e + e * e

            terms4 = [sq(*kproj(a[0], a[2], fx, cx), x), sq(*kproj(a[1], a[2], fy, cy), y),
                      sq(*kproj(c[0], c[2], fx, cx), x), sq(*kproj(c[1], c[2], fy, cy), y)]
            terms5 = [sq(pr["Ku"][fi].astype(np.float64), 0.0, x), sq(pr["Kv"][fi].astype(np.float64), 0.0, y),
                      sq(*kproj(d[0], d[2], fx, cx), x), sq(*kproj(d[1], d[2], fy, cy), y)]
            for terms, s, b in ((terms4, s4, b4), (terms5, s5, b5)):
                for t, tb in terms:
                    s += t
                    b += tb
                b += 4 * U * (s + b)
                s[s > 1e38] = np.inf                       # beyond fp32: the device's square overflows
            S4, S5 = float(np.sum(s4)), float(np.sum(s5))
            B4 = float(np.sum(b4) + 1.01 * self.m * U * np.sum(s4 + b4) + RED * S4)
            B5 = float(np.sum(b5) + 1.01 * self.m * U * np.sum(s5 + b5) + RED * S5)
            n6 = np.float64(2.0 * fi.size)
            nE, nS, ne = float(self.nE), float(self.nS), self.n_excused
            self.out7 = np.array([E, nE, float(self.nW), nS, S4, S5, n6])
            self.res6 = np.array([E, nE, np.float64(S4) / n6, 0.0, np.float64(S5) / n6, np.float64(nS) / nE])
            self.res6_b = np.array([Eb, 0.0, B4 / n6, 0.0, B5 / n6, ne / nE if nE else 0.0])

    def point_values(self, sel):
        """(7, k) fp64 per-point values of the points `sel` as this evaluation has them: u, v, dx, dy, idepth, res, hw."""
        pr = self.pr
        return np.stack([pr["u"][sel], pr["v"][sel], self.hit[sel, 1], self.hit[sel, 2], pr["nid"][sel], self.res[sel],
                         _huber_w(self.res[sel], float(self.P.huber))]).astype(np.float64)


def _jacobian(P, W, color, dd=None):
    """J (9, k), its rounding bound eJ (9, k) and - with dd = (ddxI, ddyI, dres) - its perturbation bound dJ (9, k)."""
    u, v, dxI, dyI, id_, res = (W[i] for i in range(6))
    fx, fy, affa, rb = float(P.fx), float(P.fy), float(P.affa), float(P.ref_b)
    dx, dy = dxI * fx, dyI * fy
    refc = np.asarray(color, np.float64)
    k = u.size
    J = np.stack([id_ * dx, id_ * dy, -id_ * (u * dx + v * dy), -(u * v * dx + dy + dy * v * v), u * v * dy + dx + dx * u * u,
                  u * dy - v * dx, affa * (rb - refc), -np.ones(k), res])
    A = np.stack([np.abs(id_ * dx), np.abs(id_ * dy), np.abs(id_) * (np.abs(u * dx) + np.abs(v * dy)),
                  np.abs(u * v * dx) + np.abs(dy) + np.abs(dy) * v * v, np.abs(u * v * dy) + np.abs(dx) + np.abs(dx) * u * u,
                  np.abs(u * dy) + np.abs(v * dx), abs(affa) * (abs(rb) + np.abs(refc)), np.zeros(k), np.zeros(k)])
    dJ = np.zeros_like(J)
    if dd is not None:
        ex, ey, er = dd[0] * fx, dd[1] * fy, dd[2]
        au, av, ai = np.abs(u), np.abs(v), np.abs(id_)
        dJ = np.stack([ai * ex, ai * ey, ai * (au * ex + av * ey), au * av * ex + (1 + v * v) * ey,
                       au * av * ey + (1 + u * u) * ex, au * ey + av * ex, np.zeros(k), np.zeros(k), er])
        A = A + dJ * 4                                     # the roundings act on the perturbed values
    return J, (8 * U + 8 * UD) * A, dJ


def g_terms(P, W, color, dd=None):
    """Per point the 45 products J[j1] hw J[j2] (45, k) and the bound on the device's value of each (45, k): its own
    rounding and, with dd, the perturbation of its inputs."""
    hw = W[6]
    J, eJ, dJ = _jacobian(P, W, color, dd)
    dhw = np.zeros_like(hw)
    if dd is not None:
        h, ar, dr = float(P.huber), np.abs(W[5]), dd[2]
        dhw = np.minimum(dr * h / np.maximum(ar - dr, h) ** 2, 1.0)
    Pp = np.empty((45, hw.size))
    Pb = np.empty((45, hw.size))
    for k, (a, b) in enumerate(PAIRS):
        Ja, Jb = np.abs(J[a]) + dJ[a], np.abs(J[b]) + dJ[b]
        Pp[k] = J[a] * hw * J[b]
        Pb[k] = (hw * (dJ[a] * Jb + np.abs(J[a]) * dJ[b]) + dhw * Ja * Jb
                 + (hw + dhw) * (eJ[a] * (Jb + eJ[b]) + Ja * eJ[b]) + U * (hw + dhw) * (Ja + eJ[a]) * (Jb + eJ[b]))
    return Pp, Pb


def g_sums(P, W, color, n, pert=None, extra=None):
    """The 45 sums over the points with W[6] != 0 of the (7, n) per-point values W (the device's warped buffers) and their
    bounds.  pert = (ddxI, ddyI, dres) per point (n each) perturbs the inputs (the fused kernel's own fetch); extra = (acc,
    bound) of points that may or may not be in the device's sum (added to the bound only)."""
    W = np.asarray(W, np.float64)
    sel = W[6] != 0
    m = max(1, -(-n // GRID))
    dd = None if pert is None else [np.asarray(q, np.float64)[sel] for q in pert]
    Pp, Pb = g_terms(P, W[:, sel], np.asarray(color, np.float64)[sel], dd)
    acc = Pp.sum(axis=1)
    bound = Pb.sum(axis=1) + 1.01 * m * U * (np.abs(Pp) + Pb).sum(axis=1) + RED * np.abs(Pp).sum(axis=1)
    if extra is not None:
        bound = bound + extra
    return acc, bound


def excused_g_bound(ev, pert):
    """Bound on the 45 sums of the excused points of `ev` (taken from the fp64 evaluation, perturbed by pert)."""
    sel = np.nonzero(ev.excused)[0]
    if sel.size == 0:
        return np.zeros(45)
    W = ev.point_values(sel)
    dd = [np.asarray(q, np.float64)[sel] for q in pert]
    Pp, Pb = g_terms(ev.P, W, ev.color[sel], dd)
    return 1.01 * (np.abs(Pp) + Pb).sum(axis=1) * (1 + ev.m * U)


def pack_hb(acc, bound, num_warped):
    """finish_g (cuda_coarse_tracker.cpp:335-355): the 45 sums -> H (8, 8), b (8) and their bounds."""
    with np.errstate(all="ignore"):
        factor = np.float64(1.0) / np.float64(num_warped)
    H, Hb, b, bb = np.zeros((8, 8)), np.zeros((8, 8)), np.zeros(8), np.zeros(8)
    with np.errstate(all="ignore"):
        for r in range(8):
            for q in range(8):
                lo, hi = min(r, q), max(r, q)
                k = lo * 9 + hi - lo * (lo + 1) // 2
                H[r, q] = acc[k] * factor * SCALE[r] * SCALE[q]
                Hb[r, q] = bound[k] * abs(factor) * SCALE[r] * SCALE[q] + 4 * UD * abs(H[r, q])
            k = r * 9 + 8 - r * (r + 1) // 2
            b[r] = acc[k] * factor * SCALE[r]
            bb[r] = bound[k] * abs(factor) * SCALE[r] + 4 * UD * abs(b[r])
    return H, Hb, b, bb


def ratio(got, ref, bound):
    """Worst |got - ref| / bound.  A non-finite reference must be reproduced exactly (NaN as NaN, inf with its sign); where
    the bound is 0 the values must be equal.  Returns inf on any violation of those rules."""
    got, ref, bound = (np.asarray(a, np.float64).ravel() for a in (got, ref, bound))
    fin = np.isfinite(ref)
    nf_ok = (np.isnan(ref) & np.isnan(got)) | (ref == got)
    if not nf_ok[~fin].all():
        return math.inf
    if not fin.any():
        return 0.0
    g, r, b = got[fin], ref[fin], bound[fin]
    err = np.abs(g - r)
    if not np.isfinite(err).all():
        return math.inf
    with np.errstate(all="ignore"):
        q = np.where(b > 0, err / np.where(b > 0, b, 1.0), np.where(err == 0, 0.0, math.inf))
    return float(q.max())


# ---------------------------------------------------------------------------------------------------------------------
# The exact scene: fx = fy = 1, integer cx, cy.  Under the identity pose Ku = x and Kv = y exactly, so integer and dyadic
# pixel positions probe the border test, the idepth signs, non-finite image values under a nonzero and a zero bilinear
# weight, and |res| at huber and at the cutoff +- 1 ulp, all without rounding.  Under `translated` (t = (0, 0, -1)) the
# points with idepth 1 land on p1.z = 0 and those with idepth > 1 behind the camera.
# ---------------------------------------------------------------------------------------------------------------------
def exact_pose(translated):
    T = np.eye(4)
    if translated:
        T[2, 3] = -1.0
    return T


def exact_scene(w, h, huber, cutoff, seed=0):
    """Returns dict(w, h, fx, fy, cx, cy, n, pc_u, pc_v, pc_idepth, pc_color, dInew (h, w, 3)).  Requires w >= 33, h >= 25."""
    rng = np.random.default_rng(seed)
    hub, cut = F32(huber), F32(cutoff)
    cx, cy = float(w // 2), float(h // 2)
    lo = F32(0.3) * cut                                     # ordinary residuals stay below 0.3 cutoff
    dI = np.empty((h, w, 3), F32)
    dI[..., 0] = (rng.integers(0, 64, (h, w)) / 64.0 * float(lo)).astype(F32)
    dI[..., 1:] = rng.integers(-8, 9, (h, w, 2)).astype(F32)
    special = []                                           # (x, y, idepth, color): every probe point
    bulk = []

    def put(px, py, val):                                 # a constant 2x2 patch with top-left (px, py)
        dI[py:py + 2, px:px + 2, 0] = val

    # |res| = huber, cutoff and their neighbours (color 0, affa * 0 + affb = 0 -> res = I exactly) on rows 3..7
    vals = []
    for base in (hub, cut):
        for v in (np.nextafter(base, F32(0)), base, np.nextafter(base, F32(np.inf))):
            vals += [F32(v), F32(-v)]
    for k, val in enumerate(vals):
        px, py = 4 + 3 * (k // 2), 3 + 3 * (k % 2)
        put(px, py, val)
        special += [(px, py, 1.0, 0.0), (px + 1, py + 1, 1.0, 0.0)]
    # non-finite image values on row h-7 (all three channels): hit under weight 1, under weight 0 (the pixel right of /
    # below / diagonal to the point's corner) and under a fractional weight
    for k, val in enumerate((np.nan, np.inf, -np.inf)):
        px, py = 4 + 4 * k, h - 7
        dI[py, px, :] = val
        special += [(px, py, 1.0, 0.0), (px - 1, py, 1.0, 0.0), (px, py - 1, 1.0, 0.0), (px - 1, py - 1, 1.0, 0.0),
                    (px - 0.5, py, 1.0, 0.0)]
    # border probes: Ku, Kv at 2, 2 +- 2^-8, w-3 / h-3 +- 2^-8 (the other coordinate mid-frame)
    e = 2.0 ** -8
    for ku in (2.0, 2.0 + e, 2.0 - e, w - 3.0, w - 3.0 - e, w - 3.0 + e):
        special.append((ku, cy, 1.0, 0.0))
    for kv in (2.0, 2.0 + e, 2.0 - e, h - 3.0, h - 3.0 - e, h - 3.0 + e):
        special.append((cx, kv, 1.0, 0.0))
    # idepth signs and magnitudes: -1, -0, 0, a denormal, 1, and 1.5, 2 (behind the camera once translated)
    for idp in (-1.0, -0.0, 0.0, 1e-40, 1.0, 1.5, 2.0):
        special.append((cx + 1, cy, idp, 0.0))
    # bulk: integer positions on rows 8 .. h-10, idepth 0.5 / 0.75 (p1.z = 0.5 / 0.25 once translated: still exact)
    for yy in range(8, h - 9):
        for xx in range(3, w - 3):
            if rng.random() < 0.5 and (xx, yy) != (cx + 1, cy):
                bulk.append((float(xx), float(yy), (0.5, 0.75)[int(rng.integers(0, 2))], float(rng.integers(0, 64)) / 64.0 * float(lo)))
    # saturating points: color -3 cutoff
    for k in range(40):
        bulk.append((3.0 + (k // 2) % (w - 8), 8.0 + k % 2, 0.5, -3.0 * float(cut)))
    # order: flow points (i % 32 == 0) are always bulk points, the special ones fill the other slots
    pts, si, bi = [], 0, 0
    while si < len(special) or bi < len(bulk):
        if len(pts) % 32 != 0 and si < len(special):
            pts.append(special[si]); si += 1
        elif bi < len(bulk):
            pts.append(bulk[bi]); bi += 1
        else:
            pts.append(special[si]); si += 1
    a = np.array(pts, np.float64)
    return dict(w=w, h=h, fx=1.0, fy=1.0, cx=cx, cy=cy, n=len(pts), pc_u=a[:, 0].astype(F32), pc_v=a[:, 1].astype(F32),
                pc_idepth=a[:, 2].astype(F32), pc_color=a[:, 3].astype(F32), dInew=dI)
