"""CPU checks of the fp64 per-layer reference (oracle/mvsnet_layers.py) that tests/test_mvsnet_layers_gpu.py applies to
the engine: a faithful simulation of a 16-bit layer never exceeds the bound, the subtle kernel faults the GPU test exists
to catch always do (also at the plan geometry of the four-warpgroup kernels), and the GPU test's windows run every launch
class (tile edges, warpgroup occupancy, register partials, ring depth: oracle/mvsnet_layers.py launch_classes) the product
can reach."""
import numpy as np
import pytest
import torch

from oracle import mvsnet_layers as ML
from tandem_b200 import default_weights
from tandem_b200.weights_io import load_tdmw

W_ABL03, _, _ = load_tdmw(default_weights("abl03_view_aggregation"))
DT = {"mixed16": torch.float16, "bf16": torch.bfloat16}


shapes = ML.shapes


def r16(t, precision):
    return t.to(DT[precision]).to(torch.float64)


def rand16(shape, precision, rng, kind="random"):
    if kind == "zero":
        x = np.zeros(shape)
    elif kind == "saturated":            # large, all positive: no cancellation, largest products
        x = np.full(shape, 60.0) * rng.uniform(0.5, 1.0, shape)
    else:
        x = np.maximum(rng.standard_normal(shape), 0) * 2.0
    return r16(torch.from_numpy(x), precision).numpy().astype(np.float32)


def simulate(L, T, precision, path, hi_only=False, weights=W_ABL03, weight_scale=1.0, halo=None):
    """A 16-bit layer as the engine computes it: fp32 folded weights rounded to 16 bit (hi + lo where the engine does),
    fp32 accumulation, bias / ReLU / residual in fp32, output rounded to 16 bit (fp32 for the logits)."""
    W, b = ML.fold(weights, L.conv_w, L.bn, L.bias, L.transposed)
    W32 = (W * weight_scale).to(torch.float32).to(torch.float64)
    cin, cout = (W.shape[0], W.shape[1]) if L.transposed else (W.shape[1], W.shape[0])
    ar = ML.arith_for(path, precision, cin, cout, 1 if L.dim == 2 else 3, L.plain, L.transposed)
    if path in ("", "direct"):
        Wq = W32
    else:
        hi = r16(W32, precision)
        hilo = ar.u_w < ML.U_FP32 + ML.U16[precision]
        Wq = hi + r16(W32 - hi, precision) if hilo and not hi_only else hi
    x = ML._as_batch(T[L.inp], L.dim)[:, :cin].to(torch.float32)
    if halo is not None:                 # a non-zero halo ring around every plane instead of the zero padding
        x = F_pad_ring(x, halo)
        y = ML._op(L.__class__(**{**L.__dict__, "pad": 0}), x, Wq.to(torch.float32), None if b is None else b.to(torch.float32))
    else:
        y = ML._op(L, x, Wq.to(torch.float32), None if b is None else b.to(torch.float32))
    if L.extra_bias:
        y = y + torch.from_numpy(np.asarray(weights[L.extra_bias], np.float32)).view(1, -1, 1, 1)
    if L.relu:
        y = torch.relu(y)
    if L.res:
        y = y + ML._as_batch(T[L.res], L.dim).float()
    if L.res_up2:
        y = y + ML._up2(ML._as_batch(T[L.res_up2], L.dim).float())
    y = ML._from_batch(y.to(torch.float64), L.dim)
    if not L.plain:
        y = r16(torch.from_numpy(y), precision).numpy()
    return y.astype(np.float32), ar


def F_pad_ring(x, value):
    pad = (1, 1, 1, 1) if x.dim() == 4 else (1, 1, 1, 1, 1, 1)
    return torch.nn.functional.pad(x, pad, value=value)


def ratio(L, T, y, ar, weights=W_ABL03, weight_scale=1.0):
    y_ref, bound = ML.reference(L, weights, T, ar, weight_scale)
    return ML.check(L.out, y, y_ref, bound, ar)


# (layer, path the engine runs it on): every weight-image class and output type
CASES = [("f.c3", "tc"), ("f.c1_0", "tc-s2"), ("f.c2_1", "tc"), ("feat1", ""), ("f.i2", ""), ("f.i2b", ""), ("feat2", "tc"),
         ("s1.c0", "tc-is"), ("s1.c1", "tc-s2"), ("s1.c2", "tc"), ("s1.c4", "tc"), ("s1.c6", "tc"), ("s1.x7", "tc"),
         ("s1.x9", "tc"), ("s1.x11", "tc"), ("s1.logits", "tc-is"), ("s1.logits", "direct"), ("s2.c0", ""), ("s3.x11", "")]
DN = (16, 24, 8)


def _inputs(L, precision, rng, kind):
    S = shapes(2, 96, 128, DN)
    T = {n: rand16(S[n], precision, rng, kind) for n in (L.inp, L.res, L.res_up2) if n}
    return T


def _layers():
    return {L.out: L for L in ML.layer_table(DN, True, True)}


@pytest.mark.parametrize("precision", ["mixed16", "bf16"])
@pytest.mark.parametrize("kind", ["random", "zero", "saturated"])
def test_faithful_16bit_layer_stays_within_bound(precision, kind):
    rng = np.random.default_rng(1)
    layers = _layers()
    worst = []
    for name, path in CASES:
        L = layers[name]
        T = _inputs(L, precision, rng, kind)
        y, ar = simulate(L, T, precision, path)
        if kind == "saturated" and precision == "mixed16" and not np.isfinite(y).all():
            continue                     # beyond the fp16 range: the range test on the GPU reports where values end up
        r = ratio(L, T, y, ar)
        worst.append((name, path, r.worst[1]))
        assert r.worst[1] <= 1.0, (name, path, r.worst)
    print(f"\n{precision} {kind}: " + ", ".join(f"{n}[{p or 'direct'}] {v:.3f}" for n, p, v in worst))


def test_mvsnet_layer_reference_matches_torch_graph():
    """The layer table + fp64 folding restate the reference graph: chained on exact inputs they give the oracle's fp32
    CostRegNet (mvsnet_oracle.cost_reg) to fp32 accuracy."""
    from oracle import mvsnet_oracle as O
    rng = np.random.default_rng(2)
    vol = torch.from_numpy(rng.standard_normal((32, 8, 16, 16)).astype(np.float32))
    keep = {}
    with torch.no_grad():
        lg = O.cost_reg(W_ABL03, "stage1", vol, 8, keep)
    T = {"s1.volume": vol.numpy()}
    ar = ML.Arith(0, 0, 0, 0, 0)
    for L in ML.layer_table((8, 8, 8), True, True):
        if not L.out.startswith("s1."):
            continue
        T[L.out], _ = ML.reference(L, W_ABL03, T, ar)
    for k in ("c0", "c3", "c6", "x7", "x11"):
        ref = keep[k].numpy()
        assert np.abs(T["s1." + k] - ref).max() <= 1e-4 * np.abs(ref).max(), k
    assert np.abs(T["s1.logits"][0] - lg.numpy()).max() <= 1e-4 * np.abs(lg.numpy()).max()


# ------------------------------------------------------------------------------------------------------------ mutations
def _caught(L, T, y, ar):
    return ratio(L, T, y, ar).worst[1] > 1.0


def _plan(L, path, S, smem=225):
    args = ML.plan_args(L, path, S)
    return args, ML.query_plan(args, smem)


def test_mutations_are_caught():
    rng = np.random.default_rng(3)
    layers = _layers()
    S = shapes(2, 96, 128, DN)
    caught = {}
    # 1. the last column of a partial last tile along W zeroed / taken from its left neighbour, on a stride-1 layer and a
    #    transposed one (whose tiles live on the input grid) of the GPU windows
    for (V, H, W, dn), name in (((2, 96, 128, (16, 24, 40)), "s3.c0"), ((7, 480, 640, (48, 32, 8)), "s3.x11")):
        Sw = shapes(V, H, W, dn)
        L = {l.out: l for l in ML.layer_table(dn, True, True)}[name]
        args, pl = _plan(L, "tc", Sw)
        grid_w = args[5]
        assert grid_w % pl["TW"] != 0, (name, grid_w, pl["TW"])          # the last tile along W is partial
        T = {n: rand16(Sw[n], "mixed16", rng) for n in (L.inp, L.res) if n}
        y, ar = simulate(L, T, "mixed16", "tc")
        w_last = y.shape[-1] - 1
        rows = pl["R"] * (2 if args[-1] == 1 else 1)                      # the first tile row, in output rows
        yz = y.copy(); yz[..., :rows, w_last] = 0
        ys = y.copy(); ys[..., :rows, w_last] = y[..., :rows, w_last - 1]
        t0 = (grid_w - 1) // pl["TW"] * pl["TW"]
        caught[f"{name}: last column of the partial tile at w={t0} (TW {pl['TW']} of {grid_w}) zeroed"] = _caught(L, T, yz, ar)
        caught[f"{name}: last column of the partial tile at w={t0} (TW {pl['TW']} of {grid_w}) shifted by one"] = _caught(L, T, ys, ar)
    # 2. a non-zero halo
    L = layers["f.c3"]
    T = _inputs(L, "mixed16", rng, "random")
    y, ar = simulate(L, T, "mixed16", "tc", halo=0.5)
    caught["f.c3: halo ring 0.5 instead of 0"] = _caught(L, T, y, ar)
    # 3. hi-only weights on hi/lo layers (the kernel would have dropped the lo columns)
    for name, path in (("f.c3", "tc"), ("s1.c2", "tc"), ("feat2", "tc")):
        L = layers[name]
        T = _inputs(L, "mixed16", rng, "random")
        y, ar = simulate(L, T, "mixed16", path, hi_only=True)
        caught[f"{name}: hi-only weights"] = _caught(L, T, y, ar)
    # 4. the last plane of a partial depth tile taken from the wrong plane
    L = layers["s1.c0"]
    T = _inputs(L, "mixed16", rng, "random")
    y, ar = simulate(L, T, "mixed16", "tc-is")
    yd = y.copy(); yd[:, -1] = y[:, -2]
    caught["s1.c0: last depth plane from the plane before"] = _caught(L, T, yd, ar)
    # 5. the cost volume: one source view sampled one pixel off
    from tandem_b200.synthetic import mvs_plane_window
    from oracle.mvsnet_oracle import stage_intrinsics_cpp
    win = mvs_plane_window(V=3, H=96, W=128)
    order = [win["ref_index"]] + [v for v in range(3) if v != win["ref_index"]]
    c2w = [win["c2ws"][v] for v in order]
    K = stage_intrinsics_cpp(win["K"])[0].numpy()
    feats = rand16((32, 3, 24, 32), "mixed16", rng)
    hy = ML.hypotheses(1, 8, 0.5, 5.0, 8, None, 24, 32)
    car = ML.cv_arith("mixed16", 3, 32, 8)
    iv = ML.stage_interval(0.5, 5.0, 8, 1)
    v_ref, vb, excl = ML.cost_volume_reference(W_ABL03, 1, feats, hy, K, c2w, car, iv)
    shifted = feats.copy()
    shifted[:, 2] = np.roll(feats[:, 2], 1, axis=-1)
    v_bad, _, _ = ML.cost_volume_reference(W_ABL03, 1, shifted, hy, K, c2w, car, iv)
    caught["cost volume: one source view sampled one pixel off"] = bool((np.where(excl[None], 0, np.abs(v_bad - v_ref) / vb) > 1).any())
    assert all(caught.values()), {k: v for k, v in caught.items() if not v}
    print("\n" + "\n".join(f"caught: {k}" for k in caught))


def test_regress_and_filter_mutations_are_caught():
    rng = np.random.default_rng(4)
    D, H, W = 24, 24, 32
    logits = (rng.standard_normal((D, H, W)) * 3).astype(np.float32)
    hy = ML.hypotheses(1, D, 0.5, 5.0, D, None, H, W)
    d_ref, c_ref, isum, _ = ML.regress_reference(logits, hy)
    dtol, itol, ctol = ML.regress_tolerances(D, hy, isum)
    # fp32 emulation of regress_px
    l = logits.astype(np.float32)
    e = np.exp(l - l.max(0))
    p = (e / e.sum(0, dtype=np.float32)).astype(np.float32)
    dd = (p * hy.astype(np.float32)).sum(0, dtype=np.float32)
    isum32 = (p * np.arange(D, dtype=np.float32)[:, None, None]).sum(0, dtype=np.float32)
    idx = np.clip(isum32.astype(np.int64), 0, D - 1)
    cs = np.concatenate([np.zeros((1, H, W), np.float32), np.cumsum(p, 0, dtype=np.float32)])

    def conf(shift):
        lo, hi = np.clip(idx - 1 + shift, 0, D), np.clip(idx + 3 + shift, 0, D)
        return np.take_along_axis(cs, hi[None], 0)[0] - np.take_along_axis(cs, lo[None], 0)[0]

    flip = np.abs(isum - np.round(isum)) <= itol
    assert (np.abs(dd - d_ref) <= dtol).all()
    assert (np.where(flip, 0, np.abs(conf(0) - c_ref)) <= ctol).all()
    assert (np.where(flip, 0, np.abs(conf(1) - c_ref)) > ctol).any(), "confidence window shifted by one plane not caught"
    # an edge threshold one rank off changes the threshold bits and the filtered map (the GPU test compares both exactly)
    depth = (1 + rng.random((H, W))).astype(np.float32)
    depth[:, W // 2:] += 2
    for discard in (2.5, 10.0, 37.3):
        d_ref, _, edge, thr = ML.filter_reference(depth, depth, discard)
        es = np.sort(edge.reshape(-1))
        k = ML.edge_cutoff(edge.size, discard)
        for off in (es[k - 1], es[k + 1]):
            assert off != thr
            assert not np.array_equal(np.where(edge > off, np.float32(0), depth), d_ref)
    assert ML.edge_cutoff(H * W, 0.0) == H * W - 1 and ML.edge_cutoff(H * W, 100.0) == 0


# ------------------------------------------------------------------------------------------------------------ launch classes
# What the product can launch: H and W multiples of 32 up to 480 x 640, 2 to 16 views, every legal depth number per stage
# (4 at stages 2 and 3 as in the abl04 checkpoint, 8 to 64 in steps of 8), use_is 1 / 0, the fused soft-argmin tails, and
# tc_smem_kb 225 / 113.  The 2-D layers depend on (V, H, W) only, a stage's 3-D layers on its depth number and (H, W) only.
OPTS_3D = ({}, {"use_is": 0}, {"fused_regress": 1}, {"fused_regress": 1, "use_is": 0})


def _reachable_launches():
    """{(plan_args, smem_kb)} of every tensor-core launch the product can make (deduplicated: the plan depends on nothing else)."""
    table = ML.layer_table((8, 8, 8), True, True)
    names2d = [L.out for L in table if L.dim == 2] + ["feat3"]
    sizes = [(H, W) for H in range(32, 481, 32) for W in range(32, 641, 32)]
    args = set()
    for V in range(2, 17):
        for H, W in sizes:
            args.update(a for _, a in ML.window_launches(V, H, W, (8, 8, 8), None, names2d))
    for s in (1, 2, 3):
        names = [L.out for L in table if L.out.startswith(f"s{s}.")]
        for D in ([4] if s > 1 else []) + list(range(8, 65, 8)):
            dn = tuple(D if i == s - 1 else 8 for i in range(3))
            for H, W in sizes:
                for opts in OPTS_3D:
                    args.update(a for _, a in ML.window_launches(2, H, W, dn, opts, names))
    return {(a, smem) for a in args for smem in (225, 113)}


def _window_classes(windows):
    """(key, class) -> first window of the table that runs it."""
    hit = {}
    for V, H, W, dn, opts, *_ in windows:
        smem = opts.get("tc_smem_kb", 225)
        for name, args in ML.window_launches(V, H, W, dn, opts):
            key, cls = ML.launch_classes(args, ML.query_plan(args, smem))
            for c in cls:
                hit.setdefault((key, c), f"{W}x{H}v{V} {dn} {opts or ''} {name}")
    return hit


def _unrun(windows, reachable):
    hit = _window_classes(windows)
    return sorted(kc for kc in reachable if kc not in hit), hit


def test_gpu_windows_reach_every_launch_class():
    """Every (kernel family, consumer warpgroups, tail bucket, class) a product launch can reach is run by a window of
    ML.WINDOWS, which tests/test_mvsnet_layers_gpu.py runs in both 16-bit precisions."""
    reachable = {}
    for args, smem in _reachable_launches():
        key, cls = ML.launch_classes(args, ML.query_plan(args, smem))
        for c in cls:
            reachable.setdefault((key, c), (args, smem))
    unrun, hit = _unrun(ML.WINDOWS, reachable)
    print(f"\n{len(reachable)} reachable launch classes, {len(ML.WINDOWS)} windows:")
    for (fam, nwg, bucket), c in sorted(reachable):
        where = hit.get(((fam, nwg, bucket), c), "NOT RUN")
        print(f"  {fam:28s} NWG {nwg} tail {bucket:2d}  {c:20s} {where}")
    assert not unrun, "reachable but run by no window: " + "; ".join(
        f"{k} {c} (e.g. plan_args {reachable[(k, c)][0]} at {reachable[(k, c)][1]} KB)" for k, c in unrun)
    # the table is minimal in the sense that each window runs a class no other window runs
    for i in range(len(ML.WINDOWS)):
        rest = ML.WINDOWS[:i] + ML.WINDOWS[i + 1:]
        assert _unrun(rest, reachable)[0], f"window {ML.WINDOWS[i]} runs no class of its own"


# -------------------------------------------------------------------------------------------- mutations at the plan geometry
def _find_launch(fam, cls, paths=("tc", "tc-is"), need=None):
    """The smallest layer of the GPU windows whose launch (family fam, on a path simulate() models) reaches class cls and
    satisfies need(args, plan): (layer, path, shapes, plan_args, plan)."""
    best = None
    for V, H, W, dn, opts, _ in ML.WINDOWS:
        S = ML.shapes(V, H, W, dn)
        smem = opts.get("tc_smem_kb", 225)
        use_is, tail = opts.get("use_is", 1) == 1, opts.get("fused_regress", 0) == 1
        for L in ML.layer_table(dn, True, True):
            path = ML.default_path(L, use_is)
            if path not in paths or L.transposed:
                continue
            args = ML.plan_args(L, path, S, tail and L.plain)
            pl = ML.query_plan(args, smem)
            key, c = ML.launch_classes(args, pl)
            size = int(np.prod(S[L.out]))
            if key[0] == fam and cls in c and (need is None or need(args, pl)) and (best is None or size < best[0]):
                best = (size, L, path, S, args, pl)
    assert best is not None, (fam, cls)
    return best[1:]


def _subchunk_pixels(args, pl, sc, tile=(0, 0)):
    """{tile position l: (h, w)} of the output pixels sub-chunk sc of tile (th, tw) stores (frag_pixel: l = row * P + col,
    pad columns and positions beyond the grid dropped)."""
    H, W = args[4], args[5]
    h0, w0 = tile[0] * pl["R"], tile[1] * pl["TW"]
    out = {}
    for l in range(sc * 64, sc * 64 + 64):
        hh, ww = divmod(l, pl["P"])
        if hh < pl["R"] and ww < pl["TW"] and h0 + hh < H and w0 + ww < W:
            out[l] = (h0 + hh, w0 + ww)
    return out


def _sim(L, path, S, rng, weights=W_ABL03, T=None):
    T = T or {n: rand16(S[n], "mixed16", rng) for n in (L.inp, L.res) if n}
    y, ar = simulate(L, T, "mixed16", path, weights=weights)
    return T, y, ar


def test_warpgroup_and_ring_mutations_are_caught():
    """Faults of the four-warpgroup kernels, simulated at the plan the planner makes for a layer of the GPU windows: a
    position a kernel does not store holds the debug_poison NaN."""
    rng = np.random.default_rng(5)
    caught = {}
    # ragged last round: the last round's sub-chunks of tile (0, 0), plane 0 not stored / copied from sub-chunk sc - NWG
    for fam in ("k_conv_tc mode 0", "k_conv_tc_is"):
        L, path, S, args, pl = _find_launch(fam, "ragged last round")
        T, y, ar = _sim(L, path, S, rng)
        nsub, nwg = 2 * pl["nch"], pl["nwg"]
        last = range(nsub - nsub % nwg, nsub)
        yn, yc = y.copy(), y.copy()
        for sc in last:
            src = _subchunk_pixels(args, pl, sc - nwg)
            for l, (h, w) in _subchunk_pixels(args, pl, sc).items():
                yn[:, 0, h, w] = np.nan
                if l - 64 * nwg in src:
                    yc[:, 0, h, w] = y[(slice(None), 0) + src[l - 64 * nwg]]
        what = f"{L.out} [{fam}, nch {pl['nch']}, NWG {nwg}]: last round's sub-chunks {list(last)}"
        caught[what + " not stored"] = _caught(L, T, yn, ar)
        caught[what + f" copied from sub-chunk sc - {nwg}"] = _caught(L, T, yc, ar)
    # idle warpgroups (nch == 1): sub-chunk 1 not stored, on every plane of tile (0, 0)
    for fam in ("k_conv_tc mode 0", "k_conv_tc_is"):
        L, path, S, args, pl = _find_launch(fam, "idle warpgroups", need=lambda a, p: _subchunk_pixels(a, p, 1))
        T, y, ar = _sim(L, path, S, rng)
        yn = y.copy()
        for h, w in _subchunk_pixels(args, pl, 1).values():
            yn[:, :pl["DR"], h, w] = np.nan
        caught[f"{L.out} [{fam}, nch {pl['nch']}, NWG {pl['nwg']}]: sub-chunk 1 not stored"] = _caught(L, T, yn, ar)
    # nch == kIsMaxCh: sub-chunks NWG * (KSUB - 1) + wg (the last entries of the partial arrays) miss the kd = 1 fold
    L, path, S, args, pl = _find_launch("k_conv_tc_is", "nch == kIsMaxCh")
    T, y, ar = _sim(L, path, S, rng)
    w_nokd1 = dict(W_ABL03)
    w_nokd1[L.conv_w] = np.asarray(W_ABL03[L.conv_w]).copy()
    w_nokd1[L.conv_w][:, :, 1] = 0
    _, yk, _ = _sim(L, path, S, rng, weights=w_nokd1, T=T)
    nwg = pl["nwg"]
    ksub = 2 * ML.IS_MAX_CH // nwg
    yb = y.copy()
    for th in range(pl["tiles_h"]):
        for tw in range(pl["tiles_w"]):
            for wg in range(nwg):
                for h, w in _subchunk_pixels(args, pl, nwg * (ksub - 1) + wg, (th, tw)).values():
                    yb[:, :, h, w] = yk[:, :, h, w]
    caught[f"{L.out} [k_conv_tc_is, nch {pl['nch']} == kIsMaxCh, NWG {nwg}]: sub-chunks {nwg * (ksub - 1)}.. miss the kd=1 fold"] = \
        _caught(L, T, yb, ar)
    # ring wrap: output plane od = S - 1 of tile 0 reads its newest input plane from the slot S planes stale
    for fam in ("k_conv_tc mode 0", "k_conv_tc_is"):
        L, path, S, args, pl = _find_launch(fam, "ring nin > 2S")
        if L.dim != 3:
            continue
        T, y, ar = _sim(L, path, S, rng)
        od = pl["S"] - 1                      # newest padded input plane od + 2 >= S: its slot held plane od + 2 - S before
        x = T[L.inp]
        T2 = dict(T)
        T2[L.inp] = x.copy()
        stale = od + 1 - pl["S"]
        T2[L.inp][:, od + 1] = x[:, stale] if stale >= 0 else 0
        _, y2, _ = _sim(L, path, S, rng, T=T2)
        yb = y.copy()
        yb[:, od] = y2[:, od]
        caught[f"{L.out} [{fam}, S {pl['S']}, DR {pl['DR']}]: output plane {od} from an input plane {pl['S']} slots stale"] = \
            _caught(L, T, yb, ar)
    assert len(caught) == 9 and all(caught.values()), {k: v for k, v in caught.items() if not v} or caught
    print("\n" + "\n".join(f"caught: {k}" for k in caught))


@pytest.mark.parametrize("precision", ["mixed16", "bf16"])
def test_faithful_16bit_layer_stays_within_bound_at_window_plans(precision):
    """The faithful simulation of the layers the mutation test picks from the GPU windows stays within the bound."""
    rng = np.random.default_rng(6)
    for fam, cls in (("k_conv_tc mode 0", "ragged last round"), ("k_conv_tc_is", "ragged last round"),
                     ("k_conv_tc mode 0", "idle warpgroups"), ("k_conv_tc_is", "idle warpgroups"),
                     ("k_conv_tc_is", "nch == kIsMaxCh"), ("k_conv_tc mode 0", "ring nin > 2S"), ("k_conv_tc_is", "ring nin > 2S")):
        L, path, S, args, pl = _find_launch(fam, cls)
        T = {n: rand16(S[n], precision, rng) for n in (L.inp, L.res) if n}
        y, ar = simulate(L, T, precision, path)
        r = ratio(L, T, y, ar)
        print(f"{precision} {fam} {cls}: {L.out} {S[L.out]} ratio {r.worst[1]:.3f}")
        assert r.worst[1] <= 1.0, (fam, cls, L.out, r.worst)
