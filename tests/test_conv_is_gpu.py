"""The input-stationary 3x3x3 kernel (conv_tc_is.cuh, option use_is) against the output-stationary k_conv_tc on the
same inputs: each stage's conv0 and prob.  The three kd contributions are summed in fp32 outside the tensor core, so
the two differ by rounding only."""
import numpy as np
import pytest

from tandem_b200 import DrMvsnet, default_weights

pytestmark = pytest.mark.gpu


def _run_opts(g, weights, **opts):
    V = g["bgr"].shape[0]
    H, W = g["bgr"].shape[1:3]
    bgrs = [np.ascontiguousarray(g["bgr"][v]) for v in range(V)]
    c2ws = [np.ascontiguousarray(g["c2w"][v]) for v in range(V)]
    Ks = np.stack([g["K1"], g["K2"], g["K3"]]).astype(np.float32)
    m = DrMvsnet(default_weights(weights), precision="mixed16")
    for k, v in opts.items():
        m.set_option(k, v)
    m.CallAsyncStageK(H, W, V, int(g["ref_index"]), bgrs, Ks, c2ws, float(g["depth_min"]), float(g["depth_max"]),
                      float(g["discard"]))
    return m, m.GetResult()


def _absrel(ref, est):
    m = ref > 0
    return float(np.mean(np.abs(ref[m] - est[m]) / ref[m]))


@pytest.mark.parametrize("weights", ["abl03_view_aggregation", "abl04_fewer_depth_planes"])
def test_input_stationary_matches_output_stationary(golden_small, weights):
    mo, oo = _run_opts(golden_small, weights, use_is=0)
    mi, oi = _run_opts(golden_small, weights, use_is=1)
    names = [r[0] for r in mi.profile()]
    assert sorted(n for n in names if n.endswith("[tc-is]")) == \
        sorted(f"s{s}.{n}[tc-is]" for s in (1, 2, 3) for n in ("conv0", "prob")), names
    assert not any(n.endswith("[tc-is]") for n in (r[0] for r in mo.profile()))
    assert np.array_equal(mo.debug_tensor("s1.volume"), mi.debug_tensor("s1.volume")), "inputs of stage-1 conv0 differ"
    for name in ("s1.c0", "s1.logits"):
        a, b = mi.debug_tensor(name), mo.debug_tensor(name)
        scale = float(np.abs(b).max())
        e = np.abs(a - b)
        print(f"{name}: max|d| {e.max():.3e} mean|d| {e.mean():.3e} (scale {scale:.3e})")
        assert np.isfinite(a).all() and e.max() <= 1e-3 * scale, name
    ar = _absrel(oo.depth_dense, oi.depth_dense)
    dc = float(np.mean(np.abs(oo.confidence_dense - oi.confidence_dense)))
    print(f"depth_dense Abs Rel {ar:.3e}, confidence mean-abs {dc:.3e}")
    assert ar < 1e-4 and dc < 1e-3
