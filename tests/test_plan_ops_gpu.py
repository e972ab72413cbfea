"""Every op of the real launch plans, checked on the GPU against its fp64 contract (tests/plan_interp.py) evaluated on the
op's own device inputs.  A real engine with plan_trace = 1 traces its plan with device addresses; the plan runs one op at a
time, and after each op:
  * values: every element the op wrote is within  ulp(|ref|, stored dtype) + c * u32 * E  of the contract's unrounded fp64
    result ref, E the contract's error scale (sqrt(K) * |x| |W| for the GEMM-like ops carried through the epilogue, the
    reduction length times the statistic's magnitude for the statistics ops; derivations with each contract);
  * containment: no byte of any allocation (weights included) outside the op's declared outputs changed;
  * 3xTF32 lo twins: each written lo twin is v - tf32_trunc(v) of the stored v, bit for bit.
Before each op, every element it declares written and its contract does not read is poisoned (NaN; -1 in frame counts), so
an output the kernel leaves unwritten fails instead of passing on whatever the buffer held; NaN in the contract must be NaN
in the kernel's output and nowhere else.  Errors cannot accumulate from op to op, so a failure names the op, the element
and the kernel path (the op label).  After the last op the eager embedding must equal the CUDA-graph replay bit for bit
(masked plans: replayed with longer frame counts first, then the case's own), the real engine's trace must be the
plan-check engine's trace up to allocation numbering, so the CPU plan-arithmetic tests check the plans the GPU runs, and
the plan must reach the ops and geometry branches (tests/plan_edges.py) its case is there for, the SM-count-dependent ones
included.
The worst error / bound ratio of each op kind and precision is printed (pytest -s)."""
import json
import os
import sys
import tempfile
import time

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import plan_edges as pe  # noqa: E402
import plan_interp as pi  # noqa: E402
from wespeaker_b200.models import from_synthetic  # noqa: E402

pytestmark = pytest.mark.gpu

# (model, precision, B, T, frame counts of a masked batch or None, engine options, op kinds, conv kernels and cluster N tiles
# it must reach)
CASES = {
    "ecapa1024_bf16_wide": ("ECAPA_TDNN_c1024", "bf16", 96, 200, None, {}, {"conv", "conv_tc3", "bn=256", "se_gate"}),
    "ecapa1024_bf16_T300": ("ECAPA_TDNN_c1024", "bf16", 2, 300, None, {}, {"res2_fused", "astp_fused", "scale_residual", "linear"}),
    "ecapa_glob512_fp16": ("ECAPA_TDNN_GLOB_c512", "fp16", 3, 203, None, {}, {"conv", "res2_fused", "astp_fused"}),
    "ecapa_glob512_tf32": ("ECAPA_TDNN_GLOB_c512", "tf32", 3, 203, None, {}, {"conv", "astp_stats", "tstats"}),
    "ecapa_glob512_tf32x3": ("ECAPA_TDNN_GLOB_c512", "tf32x3", 3, 203, None, {}, {"conv", "astp_stats"}),
    "ecapa512_bf16_unfused": ("ECAPA_TDNN_c512", "bf16", 2, 200, None, {"res2_fused": 0, "astp_fused": 0, "se_colsum": 0},
                              {"conv", "astp_stats", "se_gate"}),
    "resnet34_fp16": ("ResNet34", "fp16", 2, 99, None, {}, {"stem", "conv3x3", "tstats", "linear"}),
    "resnet50_bf16": ("ResNet50", "bf16", 2, 64, None, {}, {"stem", "conv3x3", "conv", "tstats"}),
    "resnet34_tf32x3": ("ResNet34", "tf32x3", 2, 99, None, {}, {"conv", "tstats"}),
    "campplus_bf16_layer": ("CAMPPlus", "bf16", 2, 260, None, {"cam_block": 0}, {"cam_dense", "conv"}),
    "campplus_bf16_block": ("CAMPPlus", "bf16", 2, 260, None, {"cam_block": 1}, {"cam_dense", "conv", "tstats"}),
    "campplus_fp16_unfused": ("CAMPPlus", "fp16", 1, 1100, None, {}, {"cam_gate", "bnrelu", "conv"}),
    "xvec_fp32": ("XVEC", "fp32", 2, 200, None, {}, {"conv_simt", "tstats", "linear"}),
    "xvec_bf16": ("XVEC", "bf16", 2, 200, None, {}, {"conv", "tstats"}),
    "eres2net_fp16": ("ERes2Net34_Base", "fp16", 2, 99, None, {}, {"aff_combine", "conv3x3"}),
    "res2net_bf16": ("Res2Net34_Base", "bf16", 2, 99, None, {}, {"conv", "tstats"}),
    "simam34_bf16": ("SimAM_ResNet34_ASP", "bf16", 2, 99, None, {}, {"simam_stats", "simam_apply", "astp_fused", "conv3x3"}),
    "gemini60_fp16": ("Gemini_DF_ResNet60", "fp16", 2, 99, None, {}, {"dwconv3x3", "tstats"}),
    "gemini60_fp16_masked": ("Gemini_DF_ResNet60", "fp16", 4, 200, [200, 163, 64, 17], {}, {"lens_derive", "dwconv3x3"}),
    "ecapa512_bf16_masked": ("ECAPA_TDNN_c512", "bf16", 4, 200, [200, 163, 64, 17], {}, {"lens_derive", "res2_fused", "astp_fused"}),
    "resnet34_fp16_masked": ("ResNet34", "fp16", 4, 200, [200, 163, 64, 17], {}, {"lens_derive", "zero_tail", "conv3x3"}),
    "campplus_bf16_masked": ("CAMPPlus", "bf16", 4, 200, [200, 163, 64, 17], {}, {"lens_derive", "cam_dense"}),
}
CASES.update(pe.EDGE_CASES)     # geometry edges: tile tails, chunk edges, 1-frame utterances (branch keys of plan_edges)
WORST = {}      # (kind, precision) -> worst error / bound ratio over the cases run


def _canonical(meta):
    """the trace with every address written as allocation number (order of first reference) + offset"""
    allocs = sorted((a, n) for a, n in meta["allocs"])
    starts = [a for a, _ in allocs]
    names = {}

    def addr(v):
        i = int(np.searchsorted(starts, v, side="right")) - 1
        if i < 0 or not (allocs[i][0] <= v < allocs[i][0] + max(allocs[i][1], 1)):
            return v
        base = allocs[i][0]
        names.setdefault(base, len(names))
        return f"A{names[base]}+{v - base}"

    def walk(x, key=None):
        if isinstance(x, dict):
            return {k: walk(v, k) for k, v in x.items() if k not in ("label", "launch")}
        if isinstance(x, list):
            return [walk(v) for v in x]
        if isinstance(x, int) and not isinstance(x, bool) and x >= 1 << 32:
            return addr(x)
        return x
    head = walk({k: meta[k] for k in ("feats_in", "emb", "lens", "B", "T", "act_es")})
    return head, walk(meta["ops"]), [op["label"] for op in meta["ops"]]


@pytest.mark.parametrize("case", list(CASES))
def test_plan_ops_match_contracts(case):
    name, prec, B, T, n_frames, opts, need = CASES[case]
    t0 = time.time()
    m = from_synthetic(name, 0, precision=prec)
    for k, v in opts.items():
        m.set_option(k, v)
    m.set_option("plan_trace", 1)
    m.to("cuda:0")
    masked = n_frames is not None
    g = torch.Generator().manual_seed(7)
    feats = torch.randn(B, T, m.feat_dim, generator=g)
    if masked:
        for b, n in enumerate(n_frames):
            feats[b, n:] = 1e4 * torch.randn(T - n, m.feat_dim, generator=g)     # garbage behind each utterance's end
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "plan.wspt")
        m.device_trace(path, B, T, masked)
        meta, _ = pi.load_trace(path)
        m.plan_trace(path, B, T, masked)
        meta_check, _ = pi.load_trace(path)
    live = pi.device_memory(meta, feats, n_frames)
    torch.cuda.synchronize()

    fails, seen = [], pe.case_branches(meta["ops"], n_frames)
    for i, op in enumerate(meta["ops"]):
        kind, g = op["trace"]["kind"], op["trace"].get("launch", {})
        seen.add(kind)
        if kind == "conv":
            seen.add("conv_" + g["kernel"])
            if g["kernel"] == "tc3":
                seen.add(f"bn={g['bn']}")
        exp = pi.expect_op(meta, op, live, tf32_cut=prec == "tf32")
        pi.poison(exp, live)         # what the op declares written and does not read: NaN (-1 in frame counts)
        before = {a: t.clone() for a, t in live.items()}
        m.run_ops(B, T, masked, i, i + 1)
        torch.cuda.synchronize()
        worst, f = pi.compare_op(exp, before, live)
        WORST[(kind, prec)] = max(WORST.get((kind, prec), 0.0), worst)
        fails += [f"op {i}: {x}" for x in f]
        del before
    assert not fails, "\n".join(fails[:20])
    missing = need - seen
    assert not missing, f"{case}: the plan no longer reaches {sorted(missing)}"

    eager = live[max(a for a in live if a <= meta["emb"])]
    off = meta["emb"] - max(a for a in live if a <= meta["emb"])
    eager = eager[off:off + B * m.embed_dim * 4].clone().view(torch.float32).reshape(B, m.embed_dim)
    if masked:      # a replay with other (longer) frame counts first: nothing of it may survive into the next one
        m.embed_padded(feats.cuda(), [T] * B)
        graph = m.embed_padded(feats.cuda(), n_frames)
    else:
        graph = m.embed(feats.cuda())
    same = torch.equal(eager.view(torch.int32), graph.view(torch.int32))      # bit for bit, NaN for NaN
    assert same, f"eager plan differs from its CUDA-graph replay: {(eager - graph).abs().nan_to_num(float('inf')).max().item()}"

    head, ops, labels = _canonical(meta)
    head_c, ops_c, labels_c = _canonical(meta_check)
    assert head == head_c and ops == ops_c, f"{case}: the real engine's plan differs from the plan-check engine's"
    lab_diff = [(a, b) for a, b in zip(labels, labels_c) if a != b]
    print(f"\n{case}: {len(meta['ops'])} ops, {time.time() - t0:.1f} s; labels differing from plan-check "
          f"(SM-count-dependent launch shapes): {len(lab_diff)}{' e.g. ' + str(lab_diff[0]) if lab_diff else ''}")
    print(case, json.dumps({f"{k}/{p}": round(v, 4) for (k, p), v in sorted(WORST.items()) if p == prec}))
