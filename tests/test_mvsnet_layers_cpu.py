"""CPU checks of the fp64 per-layer reference (oracle/mvsnet_layers.py) that tests/test_mvsnet_layers_gpu.py applies to
the engine: a faithful simulation of a 16-bit layer never exceeds the bound, the subtle kernel faults the GPU test exists
to catch always do, and the GPU test's windows drive every tile planner into single tiles and partial last tiles."""
import numpy as np
import pytest
import torch

from oracle import mvsnet_layers as ML
from tandem_b200 import default_weights
from tandem_b200.weights_io import load_tdmw

W_ABL03, _, _ = load_tdmw(default_weights("abl03_view_aggregation"))
DT = {"mixed16": torch.float16, "bf16": torch.bfloat16}


def shapes(V, H, W, dn):
    """debug-tensor shapes (C, D, H, W) of the forward (mvsnet.cu ensure_plan)."""
    S = {"f.img": (8, V, H, W), "f.c0_0": (8, V, H, W), "f.c3": (8, V, H, W), "f.c1_0": (16, V, H // 2, W // 2),
         "f.c1_1": (16, V, H // 2, W // 2), "f.c2": (16, V, H // 2, W // 2), "f.c2_0": (32, V, H // 4, W // 4),
         "f.c2_1": (32, V, H // 4, W // 4), "f.c1": (32, V, H // 4, W // 4), "feat1": (32, V, H // 4, W // 4),
         "f.i2": (32, V, H // 2, W // 2), "f.i2b": (32, V, H // 2, W // 2), "feat2": (16, V, H // 2, W // 2),
         "f.i3": (32, V, H, W), "feat3": (8, V, H, W)}
    for s in (1, 2, 3):
        sc = 1 << (3 - s)
        h, w, D = H // sc, W // sc, dn[s - 1]
        D3 = D // 4 if D == 4 else D // 8
        S.update({f"s{s}.volume": (32 >> (s - 1), D, h, w), f"s{s}.c0": (8, D, h, w), f"s{s}.c1": (16, D // 2, h // 2, w // 2),
                  f"s{s}.c2": (16, D // 2, h // 2, w // 2), f"s{s}.c3": (32, D // 4, h // 4, w // 4),
                  f"s{s}.c4": (32, D // 4, h // 4, w // 4), f"s{s}.c5": (64, D3, h // 8, w // 8), f"s{s}.c6": (64, D3, h // 8, w // 8),
                  f"s{s}.x7": (32, D // 4, h // 4, w // 4), f"s{s}.x9": (16, D // 2, h // 2, w // 2), f"s{s}.x11": (8, D, h, w),
                  f"s{s}.logits": (1, D, h, w)})
    return S


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


# ------------------------------------------------------------------------------------------------------------ tile coverage
# the windows of tests/test_mvsnet_layers_gpu.py: (V, H, W, depth numbers)
# (V, H, W, depth numbers, prob tails run there: "is" fused_regress=1, "os" fused_regress=1 with use_is=0)
GPU_WINDOWS = [(7, 480, 640, (48, 32, 8), ()), (7, 320, 512, (48, 4, 4), ()), (2, 96, 128, (16, 24, 40), ()),
               (16, 224, 288, (56, 64, 8), ()), (4, 352, 480, (24, 40, 56), ("is", "os")), (2, 96, 128, (16, 24, 8), ("is",)),
               (2, 32, 64, (8, 8, 8), ())]


def _default_path(L, dn):
    """The launch the mixed16 engine picks for L with default options (mvsnet.cu conv / conv_tc_dispatch)."""
    if L.out in ("feat1", "f.i2", "f.i2b", "f.i3"):
        return ""
    if L.dim == 2:
        return "tc-s2" if L.stride[0] == 2 else "tc"
    if L.out.endswith((".c0", ".logits")):
        return "tc-is"
    if L.transposed:
        return "tc" if L.stride[0] == 2 else ""
    if L.stride == (2, 2, 2):
        return "tc-s2"
    return "" if L.stride != (1, 1, 1) else "tc"


def _family(args):
    mode = args[-1]
    return {0: "mode 0 (stride 1)", 1: "mode 1 (deconv)", 3: "mode 3 (up-2)", 100: "mode 100 (prob tail)",
            200: "mode 200 (input-stationary)", 300: "mode 300 (input-stationary prob tail)", 400: "stride-2"}[mode]


# what these windows do not reach: no single-tile layer of the input-stationary and up-2 planners or of the prob tails (their
# smallest layers are still split), no partial W tile of the input-stationary tail, and the 2-D up-2 layer splits its view
# axis only at 113 KB.  The tails span all of D by construction.
NO_SINGLE = ("mode 200 (input-stationary)", "mode 3 (up-2)", "mode 100 (prob tail)", "mode 300 (input-stationary prob tail)")
NO_PARTIAL_D = ("mode 3 (up-2)", "mode 100 (prob tail)", "mode 300 (input-stationary prob tail)")
NO_PARTIAL_W = ("mode 300 (input-stationary prob tail)",)


@pytest.mark.parametrize("smem_kb", [225, 113])
def test_gpu_windows_reach_single_and_partial_tiles(smem_kb):
    seen = {}
    for V, H, W, dn, tails in GPU_WINDOWS:
        S = shapes(V, H, W, dn)
        todo = []
        for L in ML.layer_table(dn, True, True):
            path = _default_path(L, dn)
            args = ML.plan_args(L, path, S)
            if args is not None:
                todo.append((L.out, args))
                if path == "tc-is" and (V, H, W) == (2, 96, 128):          # the use_is=0 option runs this window
                    todo.append((L.out + " (use_is=0)", ML.plan_args(L, "tc", S)))
                if L.plain:
                    for t in tails:
                        todo.append((L.out + f" ({t} tail)", ML.plan_args(L, "tc-is" if t == "is" else "tc", S, True)))
        todo.append(("feat3 (out3a)", (32, 64, 1, V, H // 2, W // 2, 0, 3)))
        todo.append(("feat3 (out3b)", (8, 32, 1, V, H, W, 0, 0)))
        for name, args in todo:
            pl = ML.query_plan(args, smem_kb)
            D, Hh, Ww = args[3:6]
            fam = _family(args)
            hit = seen.setdefault(fam, {"single": [], "W": [], "H": [], "D": []})
            where = f"{W}x{H}v{V} {name} ({D}x{Hh}x{Ww}: TW {pl['TW']} R {pl['R']} DR {pl['DR']})"
            if pl["tiles_w"] == pl["tiles_h"] == pl["tiles_d"] == 1:
                hit["single"].append(where)
            if Ww % pl["TW"]:
                hit["W"].append(where)
            if Hh % pl["R"]:
                hit["H"].append(where)
            if D % pl["DR"]:
                hit["D"].append(where)
    print(f"\ntile coverage at {smem_kb} KB:")
    for fam, hit in sorted(seen.items()):
        for k in ("single", "W", "H", "D"):
            print(f"  {fam:30s} {k:6s} {len(hit[k]):3d}  e.g. {hit[k][0] if hit[k] else '-'}")
    for fam, hit in seen.items():
        assert (hit["W"] or fam in NO_PARTIAL_W) and hit["H"], (fam, {k: len(v) for k, v in hit.items()})
        if fam not in NO_SINGLE:
            assert hit["single"], (fam, "no single-tile layer")
        if fam not in NO_PARTIAL_D:
            assert hit["D"], (fam, "no partial depth tile")
