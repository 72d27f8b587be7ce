"""ORACLE (test infrastructure, never shipped, never on the product path).

Layer-by-layer fp64 reference of the CVA-MVSNet forward for the 16-bit and the fp32 engines.  Every layer is recomputed in float64 on
the engine's OWN stored input (DrMvsnet.debug_tensor: the exact 16-bit or fp32 values the kernel consumed, converted to fp32
without loss), so no upstream rounding leaks in, and the engine's output must lie inside an a-priori per-element bound:

    |y - y_ref| <= (1 + u_out) * E + u_out * |y_ref| + a_out (+ u_out * |partial| where a partial result is stored)
    E = (u_w + n * u_acc) * (sum |w||x| + |b|) + a_w * sum |x|,      n = taps * cin + 4 (epilogue adds)

The weights are folded from the .tdmw checkpoint in float64 here (BatchNorm after module.py:104-110 / 213-219, graph after
module.py:496-531 and 577-600 as oracle/mvsnet_oracle.py restates them); the engine's own folding is not used.
The per-class constants are derived from the arithmetic of the kernels (conv_tc*.cuh, mvsnet_kernels.cuh):

  * fp32 folded weight   w32 = fl32(w): relative error 2^-24.
  * hi/lo 16-bit image   hi = rn16(w32), lo = rn16(w32 - hi) (w32 - hi is exact in fp32):
                         |hi + lo - w32| <= u16 * |w32 - hi| <= u16^2 |w32|  ->  u_w = 2^-24 + u16^2
  * single 16-bit image  u_w = 2^-24 + u16
  * fp32-weight kernels  (k_conv_direct, k_prob_direct, k_conv00_u8) u_w = 2^-24
  * fp16 subnormals      a weight (or lo half) below 2^-14 is rounded on a grid of 2^-24: a_w = 2^-25; bf16 keeps the
                         fp32 exponent range: a_w = 0
  * accumulation         fp32 FFMA rounds to nearest: u_acc = 2^-24.  The wgmma fp32 accumulation is not specified to
                         round to nearest (it may truncate): u_acc = 2^-23 for the tensor-core kernels.
  * output               fp16 u_out = 2^-11 with a_out = 2^-25 (subnormal grid), bf16 u_out = 2^-8, fp32 logits 0 (the
                         last fp32 add is one of the n epilogue adds).

u16 is 2^-11 for fp16 and 2^-8 for bf16 (unit roundoff of an 11- / 8-bit significand).

The fp32 engine runs every layer on the direct FFMA kernels (k_conv_direct, its transposed gather, the prob layer), with
fp32 weights, fp32 activations and no fused FPN tail:
  * weights / accumulation  u_w = 2^-24, u_acc = 2^-24, a_w = 0 (fp32 keeps the exponent range of the folded weights)
  * output               fp32 stores: u_out = 0, the last rounding (bias add, ReLU is exact) is one of the n epilogue adds, as
                         for the logits.  A residual is added after that and rounds once more, relative to the stored value:
                         u_out = 2^-24 for the layers that carry one (the deconvolutions and the FPN top-down sums).
  * input                f.img = fl32(u8 / 255) (IEEE division, k_preprocess_bgr<float>): f.conv0.0 runs on the generic
                         direct kernel against the stored image, so the division's rounding is not part of its error.
"""
import math
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch
import torch.nn.functional as F

BN_EPS = 1e-5
U16 = {"mixed16": 2.0 ** -11, "bf16": 2.0 ** -8}
A16 = {"mixed16": 2.0 ** -25, "bf16": 0.0}
U_FP32 = 2.0 ** -24
U_ACC = {"fma": 2.0 ** -24, "tc": 2.0 ** -23}

FP = "feature_net."


def _c(p: int) -> str:
    return f"cost_regularization_net.stage{p}."


# ------------------------------------------------------------------------------------------------------------- weights
def fold(w, conv_w: str, bn: Optional[str] = None, bias: Optional[str] = None, transposed: bool = False):
    """BN folded into the conv in float64: (W64 in torch layout, b64 or None).  BN: y = (x - mean) / sqrt(var + eps) * gamma +
    beta per OUTPUT channel (dim 0 of a conv weight, dim 1 of a transposed-conv weight)."""
    W = torch.from_numpy(np.asarray(w[conv_w], np.float64))
    b = torch.from_numpy(np.asarray(w[bias], np.float64)) if bias else None
    if bn:
        g = torch.from_numpy(np.asarray(w[bn + ".weight"], np.float64))
        be = torch.from_numpy(np.asarray(w[bn + ".bias"], np.float64))
        mu = torch.from_numpy(np.asarray(w[bn + ".running_mean"], np.float64))
        var = torch.from_numpy(np.asarray(w[bn + ".running_var"], np.float64))
        s = g / torch.sqrt(var + BN_EPS)
        shape = [1, -1] + [1] * (W.dim() - 2) if transposed else [-1] + [1] * (W.dim() - 1)
        W = W * s.view(shape)
        b = ((b if b is not None else torch.zeros_like(mu)) - mu) * s + be
    return W, b


# ------------------------------------------------------------------------------------------------------------ layer table
@dataclass
class Layer:
    out: str                      # debug name of the output
    inp: str                      # debug name of the input
    wkey: str                     # the engine's weight key (profile names are wkey + "[path]")
    conv_w: str
    bn: Optional[str] = None
    bias: Optional[str] = None
    dim: int = 3                  # 2: FeatureNet (views are the batch), 3: CostRegNet
    stride: Tuple[int, ...] = (1, 1, 1)
    pad: int = 1
    out_pad: Tuple[int, ...] = (0, 0, 0)
    transposed: bool = False
    relu: bool = True
    res: Optional[str] = None     # same-shape residual added after the activation
    res_up2: Optional[str] = None # nearest x2 up-sampled residual (FPN top-down)
    extra_bias: Optional[str] = None   # f.i2b: the second output carries + skip3's bias
    plain: bool = False           # fp32 output (logits)


def layer_table(depth_num, fused_fpn: bool, direct_conv00: bool) -> List[Layer]:
    """The forward's layers (cva_mvsnet.py:98-184 with module.py:496-531, 577-600), by debug-tensor name."""
    L = []
    if not direct_conv00:
        L.append(Layer("f.c0_0", "f.img", "f.conv0.0", FP + "conv0.0.conv.weight", FP + "conv0.0.bn", dim=2))
    L += [Layer("f.c3", "f.c0_0", "f.conv0.1", FP + "conv0.1.conv.weight", FP + "conv0.1.bn", dim=2),
          Layer("f.c1_0", "f.c3", "f.conv1.0", FP + "conv1.0.conv.weight", FP + "conv1.0.bn", dim=2, stride=(2, 2), pad=2),
          Layer("f.c1_1", "f.c1_0", "f.conv1.1", FP + "conv1.1.conv.weight", FP + "conv1.1.bn", dim=2),
          Layer("f.c2", "f.c1_1", "f.conv1.2", FP + "conv1.2.conv.weight", FP + "conv1.2.bn", dim=2),
          Layer("f.c2_0", "f.c2", "f.conv2.0", FP + "conv2.0.conv.weight", FP + "conv2.0.bn", dim=2, stride=(2, 2), pad=2),
          Layer("f.c2_1", "f.c2_0", "f.conv2.1", FP + "conv2.1.conv.weight", FP + "conv2.1.bn", dim=2),
          Layer("f.c1", "f.c2_1", "f.conv2.2", FP + "conv2.2.conv.weight", FP + "conv2.2.bn", dim=2),
          Layer("feat1", "f.c1", "f.out1", FP + "out.stage1.weight", dim=2, pad=0, relu=False),
          Layer("f.i2", "f.c2", "f.skip2", FP + "skip.stage2.weight", bias=FP + "skip.stage2.bias", dim=2, pad=0,
                relu=False, res_up2="f.c1"),
          Layer("feat2", "f.i2", "f.out2", FP + "out.stage2.weight", dim=2, relu=False)]
    if fused_fpn:
        L.append(Layer("f.i2b", "f.c2", "f.skip2", FP + "skip.stage2.weight", bias=FP + "skip.stage2.bias", dim=2, pad=0,
                       relu=False, res_up2="f.c1", extra_bias=FP + "skip.stage3.bias"))
    else:
        L += [Layer("f.i3", "f.c3", "f.skip3", FP + "skip.stage3.weight", bias=FP + "skip.stage3.bias", dim=2, pad=0,
                    relu=False, res_up2="f.i2"),
              Layer("feat3", "f.i3", "f.out3", FP + "out.stage3.weight", dim=2, relu=False)]
    for s in (1, 2, 3):
        k, p = f"s{s}.", _c(s)
        four = depth_num[s - 1] == 4
        s5 = (1, 2, 2) if four else (2, 2, 2)
        op7 = (0, 1, 1) if four else (1, 1, 1)

        def cv(o, i, n, st=(1, 1, 1)):
            return Layer(k + o, k + i, k + n, p + n + ".conv.weight", p + n + ".bn", stride=st)

        def dc(o, i, n, res, st=(2, 2, 2), op=(1, 1, 1)):
            return Layer(k + o, k + i, k + n, p + n + ".conv.weight", p + n + ".bn", stride=st, out_pad=op,
                         transposed=True, res=k + res)

        L += [cv("c0", "volume", "conv0"), cv("c1", "c0", "conv1", (2, 2, 2)), cv("c2", "c1", "conv2"),
              cv("c3", "c2", "conv3", (2, 2, 2)), cv("c4", "c3", "conv4"), cv("c5", "c4", "conv5", s5), cv("c6", "c5", "conv6"),
              dc("x7", "c6", "conv7", "c4", s5, op7), dc("x9", "x7", "conv9", "c2"), dc("x11", "x9", "conv11", "c0"),
              Layer(k + "logits", k + "x11", k + "prob", p + "prob.weight", relu=False, plain=True)]
    return L


# ------------------------------------------------------------------------------------------------------------ arithmetic
@dataclass
class Arith:
    """Error constants of one layer's kernel (see the module docstring)."""
    u_w: float
    u_acc: float
    a_w: float
    u_out: float
    a_out: float
    desc: str = ""


def is_hilo_tc(cin: int, cout: int, kd: int) -> bool:
    """Which stride-1 [tc] layers carry a hi/lo B image (mvsnet.cu add_conv): N = 2 * npad <= 64 columns and cin <= 32,
    except the 3-D 32 -> 32 conv4 whose doubled image would not leave room for the input ring."""
    npad = 16 if cout < 16 else (32 if cin == 64 else cout)
    return npad <= 32 and cin <= 32 and not (kd == 3 and cin == 32 and cout == 32)


def direct_family(L: Layer, out_shape) -> str:
    """The k_conv_direct instantiation that computes L on the fp32 engine (mvsnet.cu conv_inst): with at least 16 output
    channels and fewer than 128 * 592 output positions a thread owns 8 channels and blockIdx.y picks the group."""
    if L.plain:
        return "k_conv_direct prob, fp32 logits"
    split = out_shape[0] >= 16 and int(np.prod(out_shape[1:])) < 128 * 592
    kind = f"transposed {L.stride}" if L.transposed else ("2-D" if L.dim == 2 else "3-D")
    return f"k_conv_direct {kind}, " + ("8-channel split" if split else "all channels") + (", + residual" if L.res or L.res_up2 else "")


def arith_for(path: str, precision: str, cin: int, cout: int, kd: int, plain: bool, transposed: bool = False,
              residual: bool = False, family: str = "") -> Arith:
    """path: the profile suffix of the launch ('' direct, 'tc', 'tc-is', 'tc-s2', 'tc-up2', 'direct', 'u8-direct').
    The transposed-conv and stride-2 images are single 16-bit.  fp32: every layer is direct (residual: a residual is added
    after the accumulation; family: the report's name of the instantiation, direct_family)."""
    if precision == "fp32":
        assert path == "", f"the fp32 engine has no {path} launch"
        return Arith(U_FP32, U_ACC["fma"], 0.0, U_FP32 if residual else 0.0, 0.0, family or "fp32 weights, FFMA, fp32 store")
    u16, a16 = U16[precision], A16[precision]
    u_out, a_out = (0.0, 0.0) if plain else (u16, a16)
    if path in ("", "direct", "u8-direct"):
        return Arith(U_FP32, U_ACC["fma"], 0.0, u_out, a_out, "fp32 weights, FFMA")
    if path in ("tc-is", "tc-up2") or (path == "tc" and not transposed and is_hilo_tc(cin, cout, kd)):
        return Arith(U_FP32 + u16 * u16, U_ACC["tc"], a16, u_out, a_out, "hi/lo 16-bit weights, wgmma")
    return Arith(U_FP32 + u16, U_ACC["tc"], a16, u_out, a_out, "single 16-bit weights, wgmma")


def _as_batch(t: np.ndarray, dim: int) -> torch.Tensor:
    """debug_tensor layout (C, D, H, W) -> (N, C, ...) for torch: 2-D layers (views, C, H, W), 3-D (1, C, D, H, W)."""
    x = torch.from_numpy(np.ascontiguousarray(t)).to(torch.float64)
    return x.permute(1, 0, 2, 3) if dim == 2 else x.unsqueeze(0)


def _from_batch(x: torch.Tensor, dim: int) -> np.ndarray:
    return (x.permute(1, 0, 2, 3) if dim == 2 else x[0]).numpy()


def _op(L: Layer, x, W, b=None):
    if L.dim == 2:
        return F.conv2d(x, W, b, stride=L.stride[:2], padding=L.pad)
    if L.transposed:
        return F.conv_transpose3d(x, W, b, stride=L.stride, padding=L.pad, output_padding=L.out_pad)
    return F.conv3d(x, W, b, stride=L.stride, padding=L.pad)


def _up2(t: torch.Tensor) -> torch.Tensor:
    return t.repeat_interleave(2, dim=-2).repeat_interleave(2, dim=-1)


@dataclass
class Result:
    name: str
    ratio: np.ndarray             # |y - y_ref| / bound, (C, D, H, W)
    err: np.ndarray
    bound: np.ndarray
    arith: Arith

    @property
    def worst(self):
        i = int(np.argmax(self.ratio))
        return np.unravel_index(i, self.ratio.shape), float(self.ratio.reshape(-1)[i])


def reference(L: Layer, w, T: Dict[str, np.ndarray], ar: Arith, weight_scale: float = 1.0):
    """(y_ref, bound) of one layer on the engine's own tensors T (name -> debug_tensor array)."""
    W, b = fold(w, L.conv_w, L.bn, L.bias, L.transposed)
    W = W * weight_scale
    x = _as_batch(T[L.inp], L.dim)
    cin = W.shape[0] if L.transposed else W.shape[1]
    if cin < x.shape[1]:                      # f.img carries 3 real + 5 zero channels
        x = x[:, :cin]
    n = cin * int(np.prod(W.shape[2:])) + 4
    y = _op(L, x, W, b)
    if L.extra_bias:
        y = y + torch.from_numpy(np.asarray(w[L.extra_bias], np.float64)).view(1, -1, 1, 1)
    if L.relu:
        y = torch.relu(y)
    absb = b.abs() if b is not None else None
    if L.extra_bias:
        absb = absb + torch.from_numpy(np.abs(np.asarray(w[L.extra_bias], np.float64)))
    E = _op(L, x.abs(), (ar.u_w + n * ar.u_acc) * W.abs() + ar.a_w,
            (ar.u_w + n * ar.u_acc) * absb if absb is not None else None)
    if L.res:
        y = y + _as_batch(T[L.res], L.dim)
    if L.res_up2:
        y = y + _up2(_as_batch(T[L.res_up2], L.dim))
    y_ref = _from_batch(y, L.dim)
    E = _from_batch(E, L.dim)
    bound = (1 + ar.u_out) * E + ar.u_out * np.abs(y_ref) + ar.a_out
    return y_ref, bound


def check(name: str, y: np.ndarray, y_ref: np.ndarray, bound: np.ndarray, ar: Arith) -> Result:
    err = np.abs(y.astype(np.float64) - y_ref)
    err[~np.isfinite(y)] = np.inf
    with np.errstate(divide="ignore", invalid="ignore"):
        ratio = np.where(err == 0, 0.0, err / bound)
    return Result(name, ratio, err, bound, ar)


# --------------------------------------------------------------------------------------------- layers with their own ref
def conv00_u8_reference(w, bgr_ref_first: np.ndarray, precision: str):
    """f.conv0.0 of k_conv00_u8: x = u8 / 255 formed in fp32 (relative error 2^-24, counted as a weight error), RGB order,
    fp32 BN-folded weights, FFMA.  bgr_ref_first (V, H, W, 3) u8 in the engine's view order."""
    W, b = fold(w, FP + "conv0.0.conv.weight", FP + "conv0.0.bn")
    x = torch.from_numpy(np.ascontiguousarray(bgr_ref_first[..., ::-1])).permute(0, 3, 1, 2).to(torch.float64) / 255.0
    ar = Arith(2 * U_FP32, U_ACC["fma"], 0.0, U16[precision], A16[precision], "u8 input, fp32 weights, FFMA")
    n = 27 + 4
    y = torch.relu(F.conv2d(x, W, b, padding=1))
    E = F.conv2d(x.abs(), (ar.u_w + n * ar.u_acc) * W.abs(), (ar.u_w + n * ar.u_acc) * b.abs(), padding=1)
    y_ref, E = y.permute(1, 0, 2, 3).numpy(), E.permute(1, 0, 2, 3).numpy()
    return y_ref, (1 + ar.u_out) * E + ar.u_out * np.abs(y_ref) + ar.a_out, ar


def fused_feat3_reference(w, T: Dict[str, np.ndarray], precision: str):
    """feat3 of the fused FPN tail (mvsnet.cu build_fused_fpn): out3a = [conv3x3(W3) o up2](f.i2b) is stored as a 16-bit
    partial in feat3, then out3b = conv3x3(W3 . Ws3)(f.c3) adds it as its residual and rounds again.  Reference: the unfused
    math, feat3 = conv3x3(W3, up2(f.i2b) + conv1x1(Ws3, f.c3)), with f.i2b = i2 + b3 as the engine stored it (checked as a
    layer of its own).  The host pre-sums up to four fp32 weights per coarse tap and forms W3 . Ws3 in double: both are
    covered by the relative fp32 weight error against sum |W3| |up2(i2b)| + |W3| |Ws3| |c3|."""
    W3, _ = fold(w, FP + "out.stage3.weight")
    Ws, _ = fold(w, FP + "skip.stage3.weight")
    i2b = _up2(_as_batch(T["f.i2b"], 2))
    c3 = _as_batch(T["f.c3"], 2)
    y = F.conv2d(i2b + F.conv2d(c3, Ws), W3, padding=1)
    part_abs = F.conv2d(i2b.abs(), W3.abs(), padding=1)              # |out3a| <= this
    u16, a16 = U16[precision], A16[precision]
    u_w = 4 * U_FP32 + u16 * u16                                      # pre-summed fp32 weights, hi/lo images (both layers)
    n = 9 * 32 + 9 * 8 + 8
    A = part_abs + F.conv2d(F.conv2d(c3.abs(), Ws.abs()), W3.abs(), padding=1)
    S = F.conv2d(i2b.abs(), torch.ones_like(W3), padding=1) + F.conv2d(c3.abs(), torch.ones(8, 8, 3, 3, dtype=torch.float64), padding=1)
    E = (u_w + n * U_ACC["tc"]) * A + a16 * S + u16 * part_abs + a16  # + the rounding of the stored out3a partial
    y_ref = y.permute(1, 0, 2, 3).numpy()
    E = E.permute(1, 0, 2, 3).numpy()
    ar = Arith(u_w, U_ACC["tc"], a16, u16, a16, "fused FPN tail: up2 hi/lo + residual partial")
    return y_ref, (1 + u16) * E + u16 * np.abs(y_ref) + a16, ar


# ------------------------------------------------------------------------------------------- hypotheses and soft-argmin
def stage_interval(dmin: float, dmax: float, D1: int, s: int) -> float:
    """The engine's per-stage interval as it computes it in fp32 (hyp_spec): (dmax - dmin) / (D1 - 1) * ratio."""
    base = np.float32(np.float32(dmax) - np.float32(dmin)) / np.float32(D1 - 1)
    return float(np.float32(np.float32((1.0, 0.5, 0.25)[s - 1]) * np.float32(base)))


def hypotheses(s: int, D: int, dmin: float, dmax: float, D1: int, prev_depth: Optional[np.ndarray], H: int, W: int):
    """fp64 hypotheses (D, H, W): uniform for stage 1 (module.py:1480-1500); adaptive from the previous stage's depth,
    bilinear x2 with align_corners=False, minus D/2 intervals, clamped at 0.001 (module.py:1503-1565)."""
    iv = stage_interval(dmin, dmax, D1, s)
    if s == 1:
        return np.float64(np.float32(dmin)) + iv * np.arange(D, dtype=np.float64)[:, None, None] * np.ones((1, H, W))
    up = F.interpolate(torch.from_numpy(prev_depth.astype(np.float64))[None, None], (H, W), mode="bilinear",
                       align_corners=False)[0, 0].numpy()
    dm = np.maximum(up - (D / 2.0) * iv, 0.001)
    return dm[None] + (D * iv) * (np.arange(D, dtype=np.float64) / D)[:, None, None]


def regress_reference(logits: np.ndarray, hyps: np.ndarray):
    """softmax over D, soft-argmin depth, 4-neighbour confidence at trunc(sum p_j j) (module.py:1116-1133) in fp64.
    Returns depth, confidence, isum and conf_at(isum_shifted): the confidence window of another trunc(isum)."""
    l = logits.astype(np.float64)
    p = np.exp(l - l.max(0, keepdims=True))
    p /= p.sum(0, keepdims=True)
    D = l.shape[0]
    depth = (p * hyps).sum(0)
    isum = (p * np.arange(D, dtype=np.float64)[:, None, None]).sum(0)
    cs = np.concatenate([np.zeros((1,) + p.shape[1:]), np.cumsum(p, 0)], 0)       # cs[k] = sum_{j<k} p_j

    def conf_at(v):
        idx = np.clip(np.trunc(v).astype(np.int64), 0, D - 1)
        lo, hi = np.clip(idx - 1, 0, D), np.clip(idx + 3, 0, D)
        return np.take_along_axis(cs, hi[None], 0)[0] - np.take_along_axis(cs, lo[None], 0)[0]

    return depth, conf_at(isum), isum, conf_at


def regress_tolerances(D: int, hyps: np.ndarray, isum: np.ndarray):
    """Error bounds of regress_px (fp32, expf / division to a few ulp, D-term FMA sums): every p_j carries a relative error
    below (D + 8) 2^-24 (the sum s has D roundings, expf and the division a few ulp); the depth and isum sums add D roundings of
    their partials; the hypotheses themselves are formed in fp32 from fp32 inputs (a few ulp of the largest one)."""
    u = U_FP32
    dtol = (2 * D + 24) * u * hyps.max(0)
    itol = (2 * D + 16) * u * np.maximum(isum, 1.0)
    ctol = (D + 16) * u
    return dtol, itol, ctol


# ------------------------------------------------------------------------------------------------------------ edge filter
def edge_metric_f32(depth: np.ndarray) -> np.ndarray:
    """15th smallest |v - c| over the zero-padded 5x5 window (module.py:1335-1343), in fp32 exactly as the kernel."""
    d = depth.astype(np.float32)
    H, W = d.shape
    pad = np.zeros((H + 4, W + 4), np.float32)
    pad[2:-2, 2:-2] = d
    win = np.stack([pad[dy:dy + H, dx:dx + W] for dy in range(5) for dx in range(5)])
    e = np.abs(win - d[None])
    return np.sort(e, axis=0)[14]


def edge_cutoff(n: int, discard: float) -> int:
    """trunc(n * (100 - p) / 100) in fp32, clamped (module.py:1347-1348)."""
    cf = np.float32(np.float32(n) * np.float32(np.float32(100.0) - np.float32(discard))) / np.float32(100.0)
    return int(min(max(int(cf), 0), n - 1))


def filter_reference(depth_dense: np.ndarray, conf_dense: np.ndarray, discard: float):
    e = edge_metric_f32(depth_dense)
    thr = np.sort(e.reshape(-1))[edge_cutoff(e.size, discard)]
    m = e > thr
    return np.where(m, np.float32(0), depth_dense), np.where(m, np.float32(0), conf_dense), e, np.float32(thr)


# ------------------------------------------------------------------------------------------------------------ tile plans
def plan_args(L: Layer, path: str, T_shapes: Dict[str, tuple], precision_tail: bool = False):
    """tdm_debug_conv_plan arguments (cin, npad, kd, D, H, W, pd, mode) of the tensor-core launch that computed layer L, or
    None for the FMA kernels.  T_shapes: debug name -> (C, D, H, W)."""
    ci, Di, Hi, Wi = T_shapes[L.inp]
    co, Do, Ho, Wo = T_shapes[L.out]
    kd = 1 if L.dim == 2 else 3
    if path == "tc-s2":
        npad = co // (2 if co == 64 else 1)
        return (ci, npad, kd, Do, Ho, Wo, 5 if L.dim == 2 else 3, 400)
    if path == "tc-is":
        return (ci, 8 if co == 1 else 16, 3, Di, Hi, Wi, 1, 300 if precision_tail else 200)
    if path == "tc-up2":
        return (32, 64, 1, Di, Hi, Wi, 0, 3)
    if path != "tc":
        return None
    if L.transposed:
        nsplit = 4 if ci == 64 else 1
        return (ci, 8 * co // nsplit, 2, Di, Hi, Wi, 1, 1)
    npad = 16 if co < 16 else (32 if ci == 64 else co)
    hilo = is_hilo_tc(ci, co, kd)
    return (ci, 2 * npad if hilo else npad, kd, Di, Hi, Wi, 1 if kd == 3 else 0, 100 if precision_tail else 0)


def query_plan(args, smem_kb: int = 225):
    import ctypes
    from tandem_b200._lib import CONV_PLAN_KEYS, lib
    out = (ctypes.c_longlong * len(CONV_PLAN_KEYS))()
    rc = lib().tdm_debug_conv_plan_n(*args, smem_kb, out, len(out))
    if rc != 0:
        raise RuntimeError(f"tdm_debug_conv_plan_n{args}: {lib().tdm_last_error()}")
    return dict(zip(CONV_PLAN_KEYS, (int(v) for v in out)))


def tile_of(args, plan, c, d, h, w):
    """The tile (td, th, tw) that computes output element (c, d, h, w).  Transposed / up2 layers tile the input grid."""
    mode = args[-1]
    if mode in (1, 3):
        d, h, w = (d // 2 if mode == 1 else d), h // 2, w // 2
    return (d // plan["DR"], h // plan["R"], w // plan["TW"])


# -------------------------------------------------------------------------------------------------------- launch classes
# The situations a tensor-core launch can put its kernel in, from its plan_args and plan.  The GPU layer test runs a table
# of windows (WINDOWS) chosen so that every class the product can reach is run; tests/test_mvsnet_layers_cpu.py enumerates
# the reachable launches and checks that.
IS_MAX_CH = 8       # kIsMaxCh (conv_tc_is.cuh): most 128-position chunks per plane of the input-stationary kernel

FAMILY = {0: "k_conv_tc mode 0", 1: "k_conv_tc mode 1 (deconv)", 3: "k_conv_tc mode 3 (up-2)", 100: "k_conv_tc prob tail",
          200: "k_conv_tc_is", 300: "k_conv_tc_is prob tail", 400: "k_conv_tc_s2"}


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


def default_path(L: Layer, use_is: bool = True) -> str:
    """The launch a 16-bit engine picks for L with the fused FPN and the direct conv0.0 (mvsnet.cu conv / conv_tc_dispatch)."""
    if L.out in ("feat1", "f.i2", "f.i2b", "f.i3"):
        return ""
    if L.dim == 2:
        return "tc-s2" if L.stride[0] == 2 else "tc"
    if L.out.endswith((".c0", ".logits")):
        return "tc-is" if use_is else "tc"
    if L.transposed:
        return "tc" if L.stride[0] == 2 else ""
    if L.stride == (2, 2, 2):
        return "tc-s2"
    return "" if L.stride != (1, 1, 1) else "tc"


def window_launches(V: int, H: int, W: int, dn, opts=None, layers=None):
    """(name, plan_args) of every tensor-core launch of one forward with options opts (use_is, fused_regress; the other
    options either leave the launches alone or are not modelled here).  layers: only these debug names (None: all)."""
    opts = opts or {}
    use_is, tail = opts.get("use_is", 1) == 1, opts.get("fused_regress", 0) == 1
    S = shapes(V, H, W, dn)
    out = []
    for L in layer_table(dn, True, True):
        if layers is not None and L.out not in layers:
            continue
        args = plan_args(L, default_path(L, use_is), S, tail and L.plain)
        if args is not None:
            out.append((L.out, args))
    if layers is None or "feat3" in layers:
        out.append(("feat3 (out3a)", (32, 64, 1, V, H // 2, W // 2, 0, 3)))
        out.append(("feat3 (out3b)", (8, 32, 1, V, H, W, 0, 0)))
    return out


def tail_bucket(args) -> int:
    """RegressTail<MAXD> of a prob launch with the soft-argmin tail (mvsnet.cu TDM_TAIL), 0 without one."""
    if args[-1] not in (100, 300):
        return 0
    D = args[3]
    return 8 if D <= 8 else 32 if D <= 32 else 48 if D <= 48 else 64


def nsplit_of(args) -> int:
    """blockIdx.y slices of the output columns: the 64-channel layers (conv6, the conv7 deconv) and the stride-2 conv5
    (32 -> 64) do not fit one B image."""
    cin, npad, kd, mode = args[0], args[1], args[2], args[-1]
    if mode == 400:
        return 2 if (cin == 32 and kd == 3) else 1
    if mode == 1:
        return 4 if cin == 64 else 1
    return 2 if cin == 64 else 1


def ring_nin(args, ndo: int) -> int:
    """Input planes a tile of ndo output planes streams through the ring."""
    kd, mode = args[2], args[-1]
    if mode == 400:
        return 2 * ndo + 1 if kd == 3 else ndo
    if mode >= 200:
        return ndo + 2
    return ndo + kd - 1


def launch_classes(args, plan):
    """(key, classes) of one launch: key = (kernel family, consumer warpgroups, tail bucket), classes the set of situations
    it puts its kernel in (tile edges, warpgroup occupancy, register partials, ring depth, row pitch, N slicing)."""
    mode = args[-1]
    D, H, W = args[3:6]
    nwg, nsub, S = plan["nwg"], 2 * plan["nch"], plan["S"]
    c = set()
    if plan["tiles_w"] == plan["tiles_h"] == plan["tiles_d"] == 1:
        c.add("single tile")
    if W % plan["TW"]:
        c.add("partial W tile")
    if H % plan["R"]:
        c.add("partial H tile")
    if D % plan["DR"]:
        c.add("partial D tile")
    # 2 * nch sub-chunks dealt round-robin to nwg warpgroups
    c.add("idle warpgroups" if nsub < nwg else ("ragged last round" if nsub % nwg else "even rounds"))
    if mode in (200, 300) and plan["nch"] == IS_MAX_CH:
        c.add("nch == kIsMaxCh")
    for ndo in {plan["DR"], D - (plan["tiles_d"] - 1) * plan["DR"]}:
        nin = ring_nin(args, ndo)
        c.add("ring nin <= S" if nin <= S else ("ring S < nin <= 2S" if nin <= 2 * S else "ring nin > 2S"))
    if plan["P"] <= 8:
        c.add("pitch P <= 8")
    if nsplit_of(args) > 1:
        c.add("nsplit > 1")
    return (FAMILY[mode], nwg, tail_bucket(args)), c


# Windows of tests/test_mvsnet_layers_gpu.py::test_layers_launch_classes, each run in both 16-bit precisions on a fresh engine
# with debug_poison: (V, H, W, depth numbers, options, the (family, NWG, tail bucket, class) it alone runs).  Together they
# run every launch class the product can reach (tests/test_mvsnet_layers_cpu.py::test_gpu_windows_reach_every_launch_class
# computes that set and checks it).  Picked greedily by classes run per unit of window size; a window with a depth number
# of 4 runs the abl04 checkpoint.
WINDOWS = [
    (2, 32, 32, (40, 16, 4), {'fused_regress': 1},
     (('k_conv_tc_is prob tail', 2, 48, 'single tile'),)),
    (2, 32, 224, (40, 16, 8), {'fused_regress': 1, 'use_is': 0},
     (('k_conv_tc prob tail', 4, 32, 'even rounds'),)),
    (2, 32, 32, (8, 56, 40), {'fused_regress': 1},
     (('k_conv_tc_is prob tail', 4, 8, 'idle warpgroups'), ('k_conv_tc_is prob tail', 4, 8, 'single tile'))),
    (2, 32, 32, (8, 56, 4), {'fused_regress': 1, 'use_is': 0},
     (('k_conv_tc prob tail', 2, 64, 'partial H tile'), ('k_conv_tc prob tail', 4, 8, 'idle warpgroups'), ('k_conv_tc prob tail', 4, 8, 'single tile'))),
    (2, 32, 352, (40, 4, 16), {'fused_regress': 1},
     (('k_conv_tc_is prob tail', 2, 48, 'partial W tile'),)),
    (2, 32, 32, (16, 4, 4), {'fused_regress': 1},
     (('k_conv_tc_is prob tail', 4, 32, 'idle warpgroups'), ('k_conv_tc_is prob tail', 4, 32, 'single tile'))),
    (2, 32, 32, (16, 40, 4), {'fused_regress': 1, 'use_is': 0},
     (('k_conv_tc prob tail', 2, 48, 'partial H tile'), ('k_conv_tc prob tail', 4, 32, 'idle warpgroups'), ('k_conv_tc prob tail', 4, 32, 'single tile'))),
    (13, 96, 448, (8, 4, 4), {'tc_smem_kb': 113},
     (('k_conv_tc mode 3 (up-2)', 4, 0, 'partial D tile'), ('k_conv_tc mode 3 (up-2)', 4, 0, 'ring nin > 2S'))),
    (2, 32, 352, (56, 40, 4), {'fused_regress': 1, 'use_is': 0},
     (('k_conv_tc prob tail', 2, 48, 'partial W tile'), ('k_conv_tc prob tail', 2, 64, 'partial W tile'))),
    (2, 32, 32, (40, 4, 4), {'fused_regress': 1, 'use_is': 0},
     (('k_conv_tc prob tail', 2, 48, 'single tile'),)),
    (2, 32, 32, (56, 4, 4), {'fused_regress': 1},
     (('k_conv_tc_is prob tail', 2, 64, 'single tile'),)),
    (2, 32, 32, (56, 4, 4), {'fused_regress': 1, 'use_is': 0},
     (('k_conv_tc prob tail', 2, 64, 'single tile'),)),
    (2, 32, 352, (56, 4, 4), {'fused_regress': 1},
     (('k_conv_tc_is prob tail', 2, 64, 'partial W tile'),)),
    (5, 160, 608, (8, 4, 4), {'fused_regress': 1},
     (('k_conv_tc_is prob tail', 4, 8, 'nch == kIsMaxCh'),)),
    (2, 256, 640, (8, 4, 4), {'fused_regress': 1, 'use_is': 0, 'tc_smem_kb': 113},
     (('k_conv_tc prob tail', 4, 8, 'ragged last round'),)),
    (3, 288, 448, (8, 4, 8), {},
     (('k_conv_tc mode 3 (up-2)', 4, 0, 'ragged last round'), ('k_conv_tc_s2', 4, 0, 'ragged last round'))),
    (2, 160, 608, (8, 4, 16), {'fused_regress': 1},
     (('k_conv_tc_is prob tail', 4, 32, 'nch == kIsMaxCh'),)),
    (2, 288, 448, (8, 24, 4), {'tc_smem_kb': 113},
     (('k_conv_tc_is', 4, 0, 'ragged last round'),)),
    (2, 416, 256, (8, 4, 24), {'tc_smem_kb': 113},
     (('k_conv_tc mode 1 (deconv)', 4, 0, 'ring nin > 2S'),)),
    (2, 256, 640, (8, 4, 16), {'fused_regress': 1, 'use_is': 0, 'tc_smem_kb': 113},
     (('k_conv_tc prob tail', 4, 32, 'ragged last round'),)),
    (2, 224, 512, (8, 4, 40), {'fused_regress': 1},
     (('k_conv_tc_is prob tail', 2, 48, 'nch == kIsMaxCh'),)),
    (2, 224, 512, (8, 4, 56), {'fused_regress': 1},
     (('k_conv_tc_is prob tail', 2, 64, 'nch == kIsMaxCh'),)),
]


# ------------------------------------------------------------------------------------------------------------ cost volume
def gate_params(w, s: int):
    """volume_gates[stage] (cva_mvsnet.py:76-83) folded in fp64: g(sq) = relu(w2 * relu(gw1 . sq + b1) + b2) + 1."""
    p = f"volume_gates.stage{s}."

    def bn(pre, bias):
        sc = float(w[pre + ".weight"][0]) / math.sqrt(float(w[pre + ".running_var"][0]) + BN_EPS)
        return sc, (bias - float(w[pre + ".running_mean"][0])) * sc + float(w[pre + ".bias"][0])

    s1, b1 = bn(p + "1", float(w[p + "0.bias"][0]))
    s2, b2 = bn(p + "4", float(w[p + "3.bias"][0]))
    return np.asarray(w[p + "0.weight"], np.float64).reshape(-1) * s1, b1, float(np.asarray(w[p + "3.weight"]).reshape(-1)[0]) * s2, b2


def homography64(K, c2w_ref, c2w_src):
    """ref pixel -> src pixel (module.py:795-808) in fp64 from the fp32 inputs the engine receives."""
    def proj(c2w):
        P = np.linalg.inv(np.asarray(c2w, np.float64))
        P[:3, :4] = np.asarray(K, np.float64) @ P[:3, :4]
        return P
    return proj(c2w_src) @ np.linalg.inv(proj(c2w_ref))


@dataclass
class CvArith:
    """Error constants of a cost-volume kernel (mvsnet_kernels.cuh k_cost_volume / k_cost_volume_va16):
      u_bil    relative rounding of the bilinear sample: fp16 weights (2^-11) and four fp16 partial roundings (HFMA2 chain), or
               fp32 weights and FFMA (a few 2^-24) for the bf16 engine
      ref_chain  the chain starts from -ref / 64 (va16: the difference is formed in fp16); else warped - ref in fp32
      a_diff   absolute error of fp16 subnormals in the chain (true units)
      u_sq, a_sq  rounding of the square (fp16 x 2^-12 in va16: subnormal grid 2^-25 * 4096), fp32 otherwise
      u_dot, dot_steps  gate weights in fp16 (2^-11) and C/2 HFMA2 partial roundings (va16), or fp32 FFMA over C channels
      u_acc    rounding of the accumulation over views per view: fp16 (va16) or fp32
      a_acc    subnormal grid of the fp16 accumulator in true units (2^-25 * 4096)
      u_out, a_out  the stored volume: fp16 x 2^-5 (subnormal grid 2^-25 * 32), bf16, or fp32 (0: the division by the view
               count is the last rounding and is counted below)
      grid_sample  the fp32 engine's sample coordinate: ix = ((qx / qz / half_w - 1 + 1) * 0.5) * (W - 1), the normalise /
               un-normalise round trip of grid_sample, four more roundings after the division"""
    u_bil: float
    ref_chain: bool
    a_diff: float
    u_sq: float
    a_sq: float
    u_dot: float
    dot_steps: int
    u_acc: float
    a_acc: float
    u_out: float
    a_out: float
    desc: str
    grid_sample: bool = False


def cv_arith(precision: str, cv_variant: int, C: int, D: int) -> CvArith:
    """cv_variant: the engine's set_option("cv_variant") value, 3 (default) or 4; it selects how many depths a thread of
    k_cost_volume_va16 owns, which leaves the arithmetic of every entry unchanged."""
    if cv_variant not in (3, 4):
        raise ValueError(f"cv_variant {cv_variant}: the engine has variants 3 and 4 only")
    u, h = U_FP32, 2.0 ** -11
    if precision == "fp32":        # generic kernel, fp32 features / math / volume: bilinear weights (1 - ax)(1 - ay) carry 3
        # roundings, the 4-tap FMA chain 4 more
        return CvArith(7 * u, False, 0.0, u, 0.0, u, C, u, 0.0, 0.0, 0.0, "generic, fp32 math, fp32 volume", grid_sample=True)
    if precision == "bf16":        # generic kernel, fp32 arithmetic on bf16 features, bf16 volume
        return CvArith(6 * u, False, 0.0, u, 0.0, u, C, u, 0.0, 2.0 ** -8, 0.0, "generic, fp32 math, bf16 volume")
    # mixed16: k_cost_volume_va16, fp16 from the bilinear chain to the accumulation over views
    return CvArith(5 * h, True, 5 * 2.0 ** -25 * 64, h, 2.0 ** -25 * 4096, h, C // 2 + 2, h, 2.0 ** -25 * 4096, h,
                   2.0 ** -25 * 32.0, "va16, fp16 accumulate")


def cost_volume_reference(w, s: int, feats: np.ndarray, hyps: np.ndarray, K, c2ws, ar: CvArith, interval: float):
    """fp64 restatement of the view-aggregation cost volume (module.py:1068-1110, cva_mvsnet.py:76-83) on the engine's own
    feat{s} (C, V, H, W; reference view first) and hypotheses (D, H, W), with the per-entry bound of ar.  Returns
    (vol_ref, bound, excluded): excluded marks entries whose q.z in some view lies within its fp32 error of the 0.001 cut, where
    the kernel may take either side of a discontinuity.  Elsewhere the zero-padded bilinear sample is continuous and piecewise
    linear in the sample coordinate (also across cell edges and at the border of the valid range), so a coordinate error e
    moves it by at most 2 e max|f| over the 4x4 neighbourhood of the cell."""
    C, V, H, W = feats.shape
    D = hyps.shape[0]
    u = U_FP32
    gw1, gb1, gw2, gb2 = gate_params(w, s)
    agw = np.abs(gw1)[:, None, None]
    gw1_scale = 2.0 ** -math.frexp(float(np.abs(gw1).max()))[1]
    f = feats.astype(np.float64)
    ref = f[:, 0]
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float64)
    vol = np.zeros((C, D, H, W))
    bound = np.zeros((C, D, H, W))
    excl = np.zeros((D, H, W), bool)
    Ms = [homography64(K, c2ws[0], c2ws[v]) for v in range(1, V)]
    mx = []        # per source view: max |f| over padded rows y0 .. y0+3, columns x0 .. x0+3 (cell (y0-1, x0-1) and its neighbours)
    for v in range(1, V):
        a = np.zeros((C, H + 5, W + 5))
        a[:, 2:H + 2, 2:W + 2] = np.abs(f[:, v])
        m4 = np.max([a[:, i:i + H + 2, :] for i in range(4)], axis=0)
        mx.append(np.max([m4[:, :, j:j + W + 2] for j in range(4)], axis=0))
    for d in range(D):
        depth = hyps[d]
        e_depth = 16 * u * (depth + D * interval)
        acc = np.zeros((C, H, W))
        E = np.zeros((C, H, W))
        for v, M in enumerate(Ms, 1):
            r = [M[i, 0] * xx + M[i, 1] * yy + M[i, 2] for i in range(3)]
            ra = [np.abs(M[i, 0] * xx) + np.abs(M[i, 1] * yy) + abs(M[i, 2]) for i in range(3)]
            q = [r[i] * depth + M[i, 3] for i in range(3)]
            # fp32 errors of q: rounded M (2^-24), the 3-term row (3 roundings), the hypothesis, the FMA
            eq = [4 * u * ra[i] * depth + np.abs(r[i]) * e_depth + u * (np.abs(q[i]) + abs(M[i, 3])) for i in range(3)]
            with np.errstate(divide="ignore", invalid="ignore"):
                ix, iy = q[0] / q[2], q[1] / q[2]
                # rcp (approx, 2^-23) and the product (2^-24) on top of the propagated errors of qx, qy, qz
                eix = (eq[0] + np.abs(ix) * eq[2]) / np.abs(q[2]) + 3 * u * np.abs(ix)
                eiy = (eq[1] + np.abs(iy) * eq[2]) / np.abs(q[2]) + 3 * u * np.abs(iy)
            if ar.grid_sample:
                # / half_w, - 1, + 1 and * (W - 1): u |ix| each, except that - 1 rounds at |ix| + half_w in pixel units
                eix = eix + u * (4 * np.abs(ix) + 0.5 * (W - 1))
                eiy = eiy + u * (4 * np.abs(iy) + 0.5 * (H - 1))
            valid = (q[2] >= 0.001) & (ix >= -1) & (iy >= -1) & (ix < W) & (iy < H)
            near = (q[2] >= 0.001) & (ix >= -1 - eix) & (iy >= -1 - eiy) & (ix < W + eix) & (iy < H + eiy)
            excl[d] |= np.abs(q[2] - 0.001) <= eq[2]
            fx, fy = ix - np.floor(ix), iy - np.floor(iy)
            x0 = np.where(valid, np.floor(ix), 0).astype(np.int64)
            y0 = np.where(valid, np.floor(iy), 0).astype(np.int64)
            ax, ay = np.where(valid, fx, 0), np.where(valid, fy, 0)
            pad = np.zeros((C, H + 2, W + 2))
            pad[:, 1:-1, 1:-1] = f[:, v]
            g = [pad[:, y0 + 1 + dy, x0 + 1 + dx] for dy in (0, 1) for dx in (0, 1)]     # f00 f01 f10 f11
            wts = [(1 - ax) * (1 - ay), ax * (1 - ay), (1 - ax) * ay, ax * ay]
            warped = np.where(valid, sum(wt * gi for wt, gi in zip(wts, g)), 0.0)
            swf = np.where(valid, sum(wt * np.abs(gi) for wt, gi in zip(wts, g)), 0.0)
            sf = np.where(valid, sum(np.abs(gi) for gi in g), 0.0)
            xc = np.clip(np.where(near, np.floor(ix), 0), -1, W - 1).astype(np.int64) + 1
            yc = np.clip(np.where(near, np.floor(iy), 0), -1, H - 1).astype(np.int64) + 1
            slope = np.where(near, 2 * (eix + eiy) * mx[v - 1][:, yc, xc], 0.0)
            diff = warped - ref
            ed = slope + ar.u_bil * (swf + (np.abs(ref) if ar.ref_chain else 0.0)) + ar.a_diff * (1 + sf) + u * np.abs(diff)
            sq = diff * diff
            esq = (2 * np.abs(diff) + ed) * ed + ar.u_sq * (np.abs(diff) + ed) ** 2 + ar.a_sq
            dot = (gw1[:, None, None] * sq).sum(0)
            sdot = (agw * sq).sum(0)
            # fp16 weights (u_dot) and dot_steps partial roundings (each on the fp16 subnormal grid a_sq / gw1_scale in
            # true units for va16), the fp32 gate weights and the un-scaling (4 u)
            edot = (agw * esq).sum(0) + ar.u_dot * (1 + ar.dot_steps) * (agw * (sq + esq)).sum(0) \
                + ar.dot_steps * ar.a_sq / gw1_scale + 4 * u * sdot
            h1 = np.maximum(dot + gb1, 0)
            gv = np.maximum(gw2 * h1 + gb2, 0) + 1
            eg = abs(gw2) * (edot + 2 * u * (np.abs(dot) + abs(gb1))) + 4 * u * (abs(gw2) * h1 + abs(gb2) + gv)
            acc += gv * sq
            # the gate factor is rounded to fp16 in the fp16 accumulation (u_acc = 2^-11), exact in fp32 (u_acc = 2^-24)
            E += gv * esq + sq * eg + ar.u_acc * gv * (sq + esq)
        n = len(Ms)
        E += n * ar.u_acc * acc + n * ar.a_acc                # one rounding of the running sum per view
        vol[:, d] = acc / n
        e = E / n + 3 * u * vol[:, d]                         # 1 / nsrc and the output scale in fp32
        bound[:, d] = (1 + ar.u_out) * e + ar.u_out * vol[:, d] + ar.a_out
    return vol, bound, excl
