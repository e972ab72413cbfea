"""CPU: the edge-case plans of tests/plan_edges.py, before any GPU time is spent on them.
  * census: every case builds, reaches the branches it lists, and together the cases reach every branch in BRANCHES (the
    SM-count-dependent ones are asserted by the GPU test from the real engine's labels);
  * perfect kernel: on the small cases, the per-op checker walk of tests/test_plan_ops_checker.py (memory poisoned in front
    of every op) passes every op, so the contracts themselves handle 1-frame utterances, 1-row tiles, empty SimAM slices and
    1-frame context segments."""
import os
import sys
import tempfile

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import plan_edges as pe  # noqa: E402
import plan_interp as pi  # noqa: E402
from test_plan_ops_checker import initial_state, walk  # noqa: E402
from wespeaker_b200.models import from_synthetic  # noqa: E402


def _trace(case):
    name, prec, B, T, n_frames, opts, _ = pe.EDGE_CASES[case]
    m = from_synthetic(name, 0, precision=prec)
    for k, v in opts.items():
        m.set_option(k, v)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "plan.wspt")
        m.plan_trace(path, B, T, n_frames is not None)
        return pi.load_trace(path)


@pytest.fixture(scope="module")
def reached():
    return {case: pe.case_branches(_trace(case)[0]["ops"], pe.EDGE_CASES[case][4]) for case in pe.EDGE_CASES}


def test_every_case_reaches_its_branches(reached):
    bad = {case: sorted((pe.EDGE_CASES[case][6] - pe.DEVICE_ONLY) - got) for case, got in reached.items()}
    bad = {c: m for c, m in bad.items() if m}
    assert not bad, f"edge cases no longer reaching the branches they are there for: {bad}"


def test_every_branch_is_reached(reached):
    listed = set().union(*(c[6] for c in pe.EDGE_CASES.values()))
    assert listed <= pe.BRANCHES, sorted(listed - pe.BRANCHES)
    got = set().union(*reached.values())
    lost = sorted(pe.BRANCHES - pe.DEVICE_ONLY - got)
    assert not lost, f"branches no edge case reaches any more: {lost}"
    assert pe.DEVICE_ONLY <= listed     # the GPU test asserts these


# the cases small enough to walk in fp64 on the CPU
def _small(name, B, T, n_frames):
    if name.startswith(("ResNet", "ERes2Net", "Gemini", "SimAM")):      # 2-D maps: 80 frequency rows at the stem
        return B * T <= (140 if n_frames is not None else 48)
    return B * T <= 300


SMALL = [c for c, (name, _, B, T, n_frames, _, _) in pe.EDGE_CASES.items() if _small(name, B, T, n_frames)]


@pytest.mark.parametrize("case", SMALL)
def test_perfect_kernel_passes_every_edge_op(case):
    meta, blob = _trace(case)
    n_frames = pe.EDGE_CASES[case][4]
    B, T = meta["B"], meta["T"]
    feats = np.random.default_rng(3).standard_normal((B, T, meta["feat_dim"]))
    if n_frames is not None:
        for b, n in enumerate(n_frames):
            feats[b, n:] = 1e4 * np.random.default_rng(b).standard_normal((T - n, meta["feat_dim"]))
    _, verdicts = walk(meta, initial_state(meta, blob, feats, n_frames))
    for i, (op, (worst, fails)) in enumerate(zip(meta["ops"], verdicts)):
        assert not fails, f"op {i}: {fails}"
        assert worst <= 1.0, (i, op["label"], worst)
