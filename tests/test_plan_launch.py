"""CPU: over the edge-case plans of tests/plan_edges.py, every op whose kernel or geometry the host chooses names that choice
in its trace ("launch"), and every geometry field a tensor-core op's label prints equals the one in "launch": the label and
the trace are written from the record the op is launched from, so the plan checkers can read the trace alone."""
import os
import sys
import tempfile

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import plan_edges as pe  # noqa: E402
import plan_interp as pi  # noqa: E402
from wespeaker_b200.models import from_synthetic  # noqa: E402

TENSOR_CORE = ("conv", "conv3x3", "res2_fused", "astp_fused", "cam_dense")
KERNEL_CHOICE = ("tstats", "astp_stats", "linear")
# label field -> launch field
LABEL_FIELDS = {"cl": "cl", "grid": "grid", "bn": "bn", "st": "nstages", "caseB": "case_b", "nb": "nb", "n_mt": "n_mt", "R": "R",
                "g": "g"}


@pytest.fixture(scope="module")
def plans():
    out = {}
    for case, (name, prec, B, T, n_frames, opts, _) in pe.EDGE_CASES.items():
        m = from_synthetic(name, 0, precision=prec)
        for k, v in opts.items():
            m.set_option(k, v)
        with tempfile.TemporaryDirectory() as d:
            path = os.path.join(d, "plan.wspt")
            m.plan_trace(path, B, T, n_frames is not None)
            out[case] = pi.load_trace(path)[0]["ops"]
    return out


def test_launch_is_traced_and_matches_the_label(plans):
    fails, kinds, fields = [], set(), set()
    for case, ops in plans.items():
        for i, op in enumerate(ops):
            kind, lab = op["trace"]["kind"], op["label"]
            if kind not in TENSOR_CORE + KERNEL_CHOICE:
                continue
            kinds.add(kind)
            g = op["trace"].get("launch")
            if not isinstance(g, dict) or (kind in KERNEL_CHOICE + ("conv",) and "kernel" not in g):
                fails.append(f"{case} op {i} ({lab}): launch {g!r}")
                continue
            if kind == "conv" and lab.split()[0] != "conv_" + g["kernel"]:
                fails.append(f"{case} op {i} ({lab}): launch kernel {g['kernel']}")
            if kind not in TENSOR_CORE:
                continue
            for f, v in (w.split("=", 1) for w in lab.split() if "=" in w):
                if f in LABEL_FIELDS:
                    fields.add(f)
                    if g.get(LABEL_FIELDS[f]) != int(v):
                        fails.append(f"{case} op {i} ({lab}): {f}={v} but launch {LABEL_FIELDS[f]}={g.get(LABEL_FIELDS[f])}")
    assert not fails, "\n".join(fails[:20])
    assert kinds == set(TENSOR_CORE + KERNEL_CHOICE), sorted(set(TENSOR_CORE + KERNEL_CHOICE) - kinds)
    assert fields == set(LABEL_FIELDS), sorted(set(LABEL_FIELDS) - fields)
