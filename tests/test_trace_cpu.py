"""n8 without a GPU: the C oracle of DSO's ImmaturePoint constructor and traceOn (oracle/trace_oracle.c) equals the reference's
own statements (ImmaturePoint.cpp:32-61, 75-414, compiled unmodified by oracle/ref_build_trace.mk) bit for bit on every case of
oracle/trace.py: the count and every point field each add leaves, and every state field (idepth_min, idepth_max, quality,
status, lastTraceUV, lastTracePixelInterval; NaN equal to NaN) after every trace of every host.  The reference's results are
stored as digests in tests/golden/reference_pins_trace.npz (oracle/gen_reference_pins_trace.py)."""
import collections
import functools
import os

import numpy as np
import pytest

from oracle import trace as T

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_pins_trace.npz")


@functools.lru_cache(maxsize=None)
def run(name):
    return T.run_oracle(T.case_inputs(name))


@pytest.mark.parametrize("name", list(T.CASES))
def test_trace_oracle_pinned_to_reference(name):
    g = np.load(GOLDEN)
    adds, traces = run(name)
    for slot, (m, fields) in adds.items():
        assert m == int(g[f"{name}_add{slot}_n"]), slot
        for k in T.POINT:
            assert T.digest(fields[k]) == str(g[f"{name}_add{slot}_{k}"]), (slot, k)
    for j, tr in enumerate(traces):
        for slot, (state, path, steps, oob_read) in tr.items():
            assert not oob_read.any(), (j, slot)          # the pinned cases read inside the image only
            for k in T.STATE:
                assert T.digest(state[k]) == str(g[f"{name}_t{j}_{slot}_{k}"]), (j, slot, k)


def test_pins_reach_every_return_path_and_the_step_cap():
    paths, cap, rejected = collections.Counter(), 0, 0
    for name in T.CASES:
        c = T.case_inputs(name)
        adds, traces = run(name)
        rejected += sum(len(h["u"]) - adds[h["slot"]][0] for h in c["hosts"])
        for tr in traces:
            for state, path, steps, _ in tr.values():
                paths.update(path.tolist())
                cap += int((steps == 99).sum())
    missing = [T.PATHS[p] for p in T.PATHS if paths[p] == 0]
    assert not missing, missing
    assert cap > 0 and rejected > 0, (cap, rejected)
