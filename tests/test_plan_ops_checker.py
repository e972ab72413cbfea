"""The per-op checker (plan_interp.check_op) can fail: on plan-check traces (no device), a "perfect kernel" that rounds
each contract's fp64 result once to the op's storage dtype passes every op of the plan, and each injected kernel fault -
a dropped tap in one 128-position tile, a row copied from its neighbour at a tile edge, an omitted ragged k-block, a
residual added twice, one Res2 link fed an unrounded s_i, one ASTP chunk's softmax weights left at the chunk's own max, a
32-channel store past Cout - is flagged on the op that has it, and on no earlier op."""
import copy
import os
import sys
import tempfile

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import plan_interp as pi  # noqa: E402
from wespeaker_b200.models import from_synthetic  # noqa: E402


def initial_state(meta, blob, feats, n_frames=None):
    """raw bytes of every allocation before the plan's first op: weights in their storage dtype, the features (and frame
    counts), zeros elsewhere"""
    act = pi.act_dtype(meta)
    blobs = {a: blob[o:o + n].astype(np.float64) for a, o, n in meta["blobs"]}
    raw = {}
    for a, n in meta["allocs"]:
        buf = np.zeros(n, np.uint8)
        if a in blobs and len(blobs[a]):
            es = n // len(blobs[a])
            b = pi.encode(blobs[a], es, act)
            buf[:b.size] = b
        raw[a] = buf
    mem = pi.RawMemory(meta, {a: torch.from_numpy(v) for a, v in raw.items()})

    def put(addr, vals, is_int):
        base, _ = mem._find(addr)
        b = pi.encode(np.asarray(vals, np.float64).reshape(-1), 4, act, is_int)
        raw[base][addr - base:addr - base + b.size] = b
    put(meta["feats_in"], feats, False)
    if n_frames is not None:
        put(meta["lens"], n_frames, True)
    return {a: torch.from_numpy(v) for a, v in raw.items()}


def perfect(meta, state, tr):
    """the perfect kernel: the contract in fp64, rounded to the storage dtype wherever the kernels store (or, inside the fused
    Res2 and CAM++ kernels, keep) a 16-bit value"""
    ref = pi.RawMemory(meta, state)
    prev, pi.ROUND = pi.ROUND, ref.act if ref.act != "fp32" else None
    try:
        pi.run_op(ref, tr, meta)
    finally:
        pi.ROUND = prev
    return pi.perfect_outputs(meta, state, ref), ref


def trace_of(name, prec, B, T, masked=False):
    m = from_synthetic(name, 0, precision=prec)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "plan.wspt")
        m.plan_trace(path, B, T, masked)
        return pi.load_trace(path)


@pytest.fixture(scope="module")
def ecapa():
    meta, blob = trace_of("ECAPA_TDNN_c512", "bf16", 2, 300)
    feats = np.random.default_rng(0).standard_normal((2, 300, 80))
    states, verdicts = walk(meta, initial_state(meta, blob, feats))
    return meta, states, verdicts


@pytest.fixture(scope="module")
def resnet():
    meta, blob = trace_of("ResNet34", "fp16", 1, 40)
    feats = np.random.default_rng(1).standard_normal((1, 40, 80))
    states, verdicts = walk(meta, initial_state(meta, blob, feats))
    return meta, states, verdicts


def walk(meta, state, poisoned=True, stop=None):
    """run the plan with the perfect kernel, checking every op (on memory poisoned the way tests/test_plan_ops_gpu.py
    poisons it, unless poisoned=False); returns the state in front of each op and what the checker said about each
    (asserted in test_perfect_kernel_passes_every_op).  stop: the number of ops to run."""
    states, verdicts = [], []
    for op in meta["ops"][:stop]:
        exp = pi.expect_op(meta, op, state)
        if poisoned:
            state = pi.poison(exp, {a: t.clone() for a, t in state.items()})
        states.append(state)
        after, _ = perfect(meta, state, op["trace"])
        verdicts.append(pi.compare_op(exp, state, after))
        state = after
    return states, verdicts


def first_op(meta, pred):
    for i, op in enumerate(meta["ops"]):
        if pred(op["trace"], op["label"]):
            return i
    raise AssertionError("the plan no longer has an op of the shape this fault targets")


def flagged(meta, i, state, after):
    worst, fails = pi.check_op(meta, meta["ops"][i], state, after)
    assert fails, f"fault in op {i} ({meta['ops'][i]['label']}) not flagged (worst ratio {worst:.3g})"
    assert all(f.startswith(meta["ops"][i]["label"]) for f in fails)
    return fails


def rows_region(tr):
    """(address, es, ld, C) of a conv's output, rows = flattened positions"""
    return tr["out"], tr["es"], tr["out_ld"], tr["Cout"]


def splice_rows(state_after, src_raw, addr, es, ld, C, rows, src_rows=None):
    """copy output rows `src_rows` (default: the same rows) of src_raw into rows `rows` of state_after"""
    out = {a: t.clone() for a, t in state_after.items()}
    base = max(a for a in out if a <= addr)
    dst = out[base].numpy()
    src = src_raw[base].numpy()
    off = addr - base
    for r, s in zip(rows, src_rows if src_rows is not None else rows):
        dst[off + r * ld * es:off + (r * ld + C) * es] = src[off + s * ld * es:off + (s * ld + C) * es]
    out[base] = torch.from_numpy(dst)
    return out


def test_perfect_kernel_passes_every_op(ecapa, resnet):
    for meta, _, verdicts in (ecapa, resnet):
        for op, (worst, fails) in zip(meta["ops"], verdicts):
            assert not fails, fails
            assert worst <= 1.0, (op["label"], worst)
    kinds = {op["trace"]["kind"] for op in ecapa[0]["ops"]}
    assert {"conv", "res2_fused", "astp_fused", "se_gate", "scale_residual", "linear"} <= kinds, kinds
    assert {"conv3x3", "stem", "tstats"} <= {op["trace"]["kind"] for op in resnet[0]["ops"]}


def test_dropped_tap_in_one_tile_is_flagged(ecapa):
    meta, states, _ = ecapa
    i = first_op(meta, lambda tr, lab: tr["kind"] == "conv" and len(tr["taps"]) >= 3 and tr["B"] * tr["F"] * tr["T"] >= 256)
    tr = meta["ops"][i]["trace"]
    good, _ = perfect(meta, states[i], tr)
    tr2 = copy.deepcopy(tr)
    tr2["taps"] = tr2["taps"][:len(tr2["taps"]) // 2] + tr2["taps"][len(tr2["taps"]) // 2 + 1:]
    bad, _ = perfect(meta, states[i], tr2)
    flagged(meta, i, states[i], splice_rows(good, bad, *rows_region(tr), range(128, 256)))


def test_row_from_neighbour_at_tile_edge_is_flagged(ecapa):
    meta, states, _ = ecapa
    i = first_op(meta, lambda tr, lab: tr["kind"] == "conv" and tr["B"] * tr["F"] * tr["T"] >= 256)
    tr = meta["ops"][i]["trace"]
    good, _ = perfect(meta, states[i], tr)
    flagged(meta, i, states[i], splice_rows(good, good, *rows_region(tr), [128], [127]))


def test_omitted_ragged_k_block_is_flagged(ecapa):
    meta, states, _ = ecapa
    i = first_op(meta, lambda tr, lab: tr["kind"] == "conv" and tr["Ktot"] % 64 != 0)
    tr = meta["ops"][i]["trace"]
    K, Cout, es = tr["Ktot"], tr["Cout"], tr["es"]
    st = {a: t.clone() for a, t in states[i].items()}
    base = max(a for a in st if a <= tr["W"])
    w = st[base].numpy()
    for o in range(Cout):      # the kernel that skips the last k-block sees zeros there
        row = tr["W"] - base + o * K * es
        w[row + (K // 64) * 64 * es:row + K * es] = 0
    bad, _ = perfect(meta, st, tr)
    flagged(meta, i, states[i], bad)


def test_residual_added_twice_in_one_tile_is_flagged(resnet):
    meta, states, _ = resnet
    i = first_op(meta, lambda tr, lab: tr["kind"] == "conv3x3" and tr["res"] is not None)
    tr = meta["ops"][i]["trace"]
    good, ref = perfect(meta, states[i], tr)
    o = tr["out"]
    v = ref.view(o, 2).copy()
    flat = v.reshape(-1, o["C"])
    flat[:128] += ref.view(tr["res"], 2).reshape(-1, o["C"])[:128]
    bad = {a: t.clone() for a, t in good.items()}
    base = max(a for a in bad if a <= o["p"])
    buf = bad[base].numpy()
    enc = pi.encode(flat[:128].reshape(-1), 2, ref.act).reshape(128, o["C"] * 2)
    for r in range(128):
        s = o["p"] - base + r * o["ld"] * 2
        buf[s:s + o["C"] * 2] = enc[r]
    flagged(meta, i, states[i], bad)


def test_unrounded_res2_link_is_flagged(ecapa):
    meta, states, _ = ecapa
    i = first_op(meta, lambda tr, lab: tr["kind"] == "res2_fused")
    tr = meta["ops"][i]["trace"]
    good, ref = perfect(meta, states[i], tr)
    got = pi.RawMemory(meta, good)
    w8, dil, k = tr["w8"], tr["dil"], 3
    x = ref.view(tr["x"], 2)[:, 0]
    sp = got.view(tr["out"], 2)[:, 0]
    W7 = ref.vec(tr["W7"], 7 * w8 * 3 * w8, 2).reshape(7, w8, 3, w8)
    bias, scale, shift = (ref.vec(tr[n], 7 * w8).reshape(7, w8) for n in ("bias", "scale", "shift"))
    s = sp[..., (k - 1) * w8:k * w8] + x[..., k * w8:(k + 1) * w8]          # s_k left unrounded
    spk = np.maximum(pi._dil_conv1d(s, W7[k], dil) + bias[k], 0.0) * scale[k] + shift[k]
    bad = {a: t.clone() for a, t in good.items()}
    o = tr["out"]
    base = max(a for a in bad if a <= o["p"])
    buf = bad[base].numpy()
    enc = pi.encode(spk.reshape(-1), 2, ref.act).reshape(-1, w8 * 2)
    for r in range(enc.shape[0]):
        st = o["p"] - base + (r * o["ld"] + k * w8) * 2
        buf[st:st + w8 * 2] = enc[r]
    flagged(meta, i, states[i], bad)


def test_astp_chunk_left_at_its_own_max_is_flagged(ecapa):
    meta, states, _ = ecapa
    i = first_op(meta, lambda tr, lab: tr["kind"] == "astp_fused" and tr["x"]["T"] > 256)
    tr = meta["ops"][i]["trace"]
    good, ref = perfect(meta, states[i], tr)
    x, h = ref.view(tr["x"], 2)[:, 0], ref.view(tr["h"], 2)[:, 0]
    B, T, C = x.shape
    W2 = ref.vec(tr["W2"], C * 128, 2).reshape(C, 128)
    stats = np.zeros((B, 2 * C))
    for b in range(B):
        lg = h[b] @ W2.T
        M, m1 = lg.max(axis=0), lg[256:].max(axis=0)
        a = np.exp(lg - M)
        a[256:] = np.exp(lg[256:] - m1)       # the second 256-frame chunk is never rescaled to the running max
        a /= a.sum(axis=0)
        mean = (a * x[b]).sum(axis=0)
        var = (a * x[b] ** 2).sum(axis=0) - mean ** 2
        stats[b] = np.concatenate([mean, np.sqrt(np.maximum(var, tr["eps"]))])
    bad = {a: t.clone() for a, t in good.items()}
    base = max(a for a in bad if a <= tr["stats"])
    buf = bad[base].numpy()
    enc = pi.encode(stats.reshape(-1), 4, ref.act)
    buf[tr["stats"] - base:tr["stats"] - base + enc.size] = enc
    flagged(meta, i, states[i], bad)


def test_store_past_cout_is_flagged(ecapa):
    meta, states, _ = ecapa
    i = first_op(meta, lambda tr, lab: tr["kind"] == "res2_fused")
    tr = meta["ops"][i]["trace"]
    good, _ = perfect(meta, states[i], tr)
    bad = {a: t.clone() for a, t in good.items()}
    o = tr["out"]
    base = max(a for a in bad if a <= o["p"])
    buf = bad[base].numpy()
    s = o["p"] - base + (5 * o["ld"] + 7 * tr["w8"]) * 2      # 32 channels past the 7 groups it owns, in row 5
    buf[s:s + 32 * 2] ^= 0x5A
    fails = flagged(meta, i, states[i], bad)
    assert any("outside its declared outputs" in f for f in fails)


def _rows(tr_view, b, f, t):
    """byte offset (from the view's address) and length of output row (b, f, t) of a channels-last View"""
    o = tr_view
    return ((b * o["F"] + f) * o["T"] + t) * o["ld"] * 2, o["C"] * 2


def test_nan_contract_element_does_not_hide_its_region(resnet):
    """a NaN the contract computes (here from a NaN input element) must not make the rest of the output region a no-op
    check: an element far out of bound next to it is flagged, and so is a finite value where the contract is NaN"""
    meta, states, _ = resnet
    i = first_op(meta, lambda tr, lab: tr["kind"] == "tstats")
    tr = meta["ops"][i]["trace"]
    st = {a: t.clone() for a, t in states[i].items()}
    x = tr["x"]
    base = max(a for a in st if a <= x["p"])
    st[base].numpy()[x["p"] - base:x["p"] - base + 2] = np.frombuffer(np.float16(np.nan).tobytes(), np.uint8)
    good, _ = perfect(meta, st, tr)
    ob = max(a for a in good if a <= tr["out"])
    out = good[ob].numpy()[tr["out"] - ob:].view(np.float32)
    assert np.isnan(out[0]) and np.isfinite(out[1])
    assert not pi.check_op(meta, meta["ops"][i], st, good)[1]
    far = {a: t.clone() for a, t in good.items()}
    far[ob].numpy()[tr["out"] - ob:].view(np.float32)[1] *= 1.01
    flagged(meta, i, st, far)
    finite = {a: t.clone() for a, t in good.items()}
    finite[ob].numpy()[tr["out"] - ob:].view(np.float32)[0] = 0.0
    flagged(meta, i, st, finite)


def test_skipped_padding_rows_fail_only_on_poisoned_memory():
    """a masked conv3x3 that never writes the zero rows behind an utterance's end passes on zero-initialised memory (zero
    is the right answer there) and fails once the op's outputs are poisoned in front of it"""
    meta, blob = trace_of("ResNet34", "fp16", 2, 40, masked=True)
    n_frames = [40, 13]
    feats = np.random.default_rng(4).standard_normal((2, 40, 80))
    i = first_op(meta, lambda tr, lab: tr["kind"] == "conv3x3" and tr["lens"])
    state = walk(meta, initial_state(meta, blob, feats, n_frames), poisoned=False, stop=i + 1)[0][i]
    op = meta["ops"][i]
    tr = op["trace"]
    o = tr["out"]
    lens = pi.RawMemory(meta, state).vec(tr["lens"], 2).astype(int)
    assert lens[1] < o["T"]

    def skip_padding(before, after):
        bad = {a: t.clone() for a, t in after.items()}
        base = max(a for a in bad if a <= o["p"])
        for f in range(o["F"]):
            for t in range(lens[1], o["T"]):
                off, n = _rows(o, 1, f, t)
                s = o["p"] - base + off
                bad[base].numpy()[s:s + n] = before[base].numpy()[s:s + n]
        return bad
    good, _ = perfect(meta, state, tr)
    assert not pi.check_op(meta, op, state, skip_padding(state, good))[1]
    exp = pi.expect_op(meta, op, state)
    poisoned = pi.poison(exp, {a: t.clone() for a, t in state.items()})
    good, _ = perfect(meta, poisoned, tr)
    assert not pi.compare_op(exp, poisoned, good)[1]
    worst, fails = pi.compare_op(exp, poisoned, skip_padding(poisoned, good))
    assert fails and all(f.startswith(op["label"]) for f in fails), (worst, fails)


def test_unwritten_one_row_time_tile_is_flagged():
    """T = 257 runs the 3x3 kernel in 128-row time tiles, the last one a single row: leaving it unwritten is flagged"""
    meta, blob = trace_of("ResNet34", "fp16", 1, 257)
    i = first_op(meta, lambda tr, lab: tr["kind"] == "conv3x3" and tr["out"]["T"] == 257 and tr["launch"]["n_mt"] == 1)
    feats = np.random.default_rng(5).standard_normal((1, 257, 80))
    state = walk(meta, initial_state(meta, blob, feats), stop=i + 1)[0][i]
    tr = meta["ops"][i]["trace"]
    good, _ = perfect(meta, state, tr)
    o = tr["out"]
    bad = {a: t.clone() for a, t in good.items()}
    base = max(a for a in bad if a <= o["p"])
    for f in range(o["F"]):
        off, n = _rows(o, 0, f, 256)
        s = o["p"] - base + off
        bad[base].numpy()[s:s + n] = state[base].numpy()[s:s + n]
    assert not pi.check_op(meta, meta["ops"][i], state, good)[1]
    flagged(meta, i, state, bad)


def test_se_gate_reads_the_column_sums_its_conv_wrote():
    """A 16-bit ECAPA plan at T >= 128 squeezes SE from the column sums the preceding conv's epilogue writes: the se_gate
    trace names that buffer, and its contract declares the read."""
    meta, blob = trace_of("ECAPA_TDNN_c512", "bf16", 2, 200)
    ops = [op["trace"] for op in meta["ops"]]
    gates = [i for i, tr in enumerate(ops) if tr["kind"] == "se_gate"]
    assert gates
    for i in gates:
        conv = next(tr for tr in reversed(ops[:i]) if tr["kind"] == "conv")
        assert conv["colsum"] and ops[i]["colsum"] == conv["colsum"]
        mem = pi.Memory(meta, blob)
        pi.run_op(mem, ops[i], meta)
        assert any(addr == conv["colsum"] for addr, *_ in mem.reads)
