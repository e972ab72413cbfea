"""CPU: host logic, the C-ABI library (loads, exports every declared symbol, fails loudly without a GPU),
Kaldi IO, the nn.Module-shaped wrapper, and the world_size-2 gloo path of the multi-GPU gather."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from wespeaker_b200 import kaldi_io, lib, parallel, synthetic as syn
from wespeaker_b200.models import B200SpeakerModel, from_synthetic, get_speaker_model

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    L = lib.load()
    hdr = open(os.path.join(ROOT, "include", "wespeaker_b200.h")).read()
    declared = set(re.findall(r"\b(ws_[a-z0-9_]+)\s*\(", hdr))
    assert declared, "no declarations parsed"
    assert declared == set(lib.EXPORTED_SYMBOLS), declared ^ set(lib.EXPORTED_SYMBOLS)
    for name in declared:
        assert hasattr(L, name), name
    assert L.ws_version() >= 100
    assert L.ws_fbank_num_frames(32000) == 198 and L.ws_fbank_num_frames(399) == 0 and L.ws_fbank_num_frames(400) == 1


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_no_cpu_fallback():
    m = from_synthetic("ECAPA_TDNN_c512")
    with pytest.raises(lib.B200Error):
        m(torch.zeros(1, 200, 80))
    from wespeaker_b200.plda import TwoCovPLDA
    p = TwoCovPLDA.from_arrays(**syn.make_plda(256))
    with pytest.raises(lib.B200Error):
        p.transform_batch(np.zeros((2, 256), np.float32))


def test_wrapper_state_dict_contract():
    ctor = get_speaker_model("ResNet34")
    m = ctor(feat_dim=80, embed_dim=256, pooling_func="TSTP", two_emb_layer=False)
    assert isinstance(m, torch.nn.Module) and isinstance(m, B200SpeakerModel)
    sd = {k: torch.from_numpy(np.asarray(v)) for k, v in syn.make_state_dict("ResNet34", 0).items()}
    r = m.load_state_dict(sd)
    assert r.missing_keys == [] and r.unexpected_keys == []
    assert list(m.state_dict().keys()) == list(sd.keys())
    bad = dict(sd)
    bad["projection.weight"] = torch.zeros(10, 256)
    del bad["seg_1.bias"]
    with pytest.raises(RuntimeError):
        m.load_state_dict(bad, strict=True)
    r = m.load_state_dict(bad, strict=False)  # checkpoint.py:66-85 semantics
    assert r.missing_keys == ["seg_1.bias"] and r.unexpected_keys == ["projection.weight"]
    bad2 = dict(sd)
    bad2["seg_1.weight"] = torch.zeros(3, 3)
    with pytest.raises(RuntimeError):
        m.load_state_dict(bad2, strict=False)
    assert m.to("cpu").eval() is m
    with pytest.raises(ValueError):
        get_speaker_model("ReDimNetB0")   # a family outside SURVEY.md section 8


def test_kaldi_vector_roundtrip(tmp_path):
    ark, scp = str(tmp_path / "xvector.ark"), str(tmp_path / "xvector.scp")
    rng = np.random.default_rng(0)
    vecs = {f"utt{i}": rng.standard_normal(192).astype(np.float32) for i in range(5)}
    with kaldi_io.VectorWriter(ark, scp) as w:
        for k, v in vecs.items():
            w(k, v)
    back = kaldi_io.read_vec_scp_file(scp)
    assert list(back) == list(vecs)
    for k in vecs:
        assert np.array_equal(back[k], vecs[k])
    assert [k for k, _ in kaldi_io.load_ark(ark)] == list(vecs)
    raw = open(ark, "rb").read()
    assert raw.startswith(b"utt0 \0BFV \4" + (192).to_bytes(4, "little"))


def test_shard_helpers():
    assert parallel.shard_indices(10, 1, 4) == [1, 5, 9]
    assert parallel.shard_rows(10, 3, 4) == (9, 10) and parallel.shard_rows(10, 0, 4) == (0, 3)
    x = torch.arange(6.0).view(3, 2)
    assert parallel.gather_embeddings(x, 3) is x  # world size 1: identity


_WORKER = r"""
import os, sys, torch
sys.path.insert(0, {root!r})
from wespeaker_b200 import parallel
import torch.distributed as dist
rank, world, _ = parallel.init_from_env("gloo")
N, E = 7, 4
full = torch.arange(N * E, dtype=torch.float32).view(N, E)
mine = full[parallel.shard_indices(N, rank, world)]
out = parallel.gather_embeddings(mine, N)
assert torch.equal(out, full), (rank, out)
lo, hi = parallel.shard_rows(N, rank, world)
tot = torch.tensor([float(hi - lo)]); dist.all_reduce(tot); assert tot.item() == N
assert parallel.max_over_ranks(float(rank)) == world - 1
parallel.barrier()
print("OK", rank)
"""


def test_gather_embeddings_gloo_world2(tmp_path):
    script = tmp_path / "w.py"
    script.write_text(_WORKER.format(root=ROOT))
    procs = []
    for r in range(2):
        env = dict(os.environ, RANK=str(r), WORLD_SIZE="2", LOCAL_RANK=str(r), MASTER_ADDR="127.0.0.1",
                   MASTER_PORT="29533")
        procs.append(subprocess.Popen([sys.executable, str(script)], env=env, stdout=subprocess.PIPE,
                                      stderr=subprocess.STDOUT, text=True))
    outs = [p.communicate(timeout=180)[0] for p in procs]
    for p, o in zip(procs, outs):
        assert p.returncode == 0 and "OK" in o, o


def test_speaker_register_recognize_similarity_host_logic(monkeypatch, capsys):
    """`cli/speaker.py:180-211` host logic (no GPU involved: extract_embedding is replaced by a lookup table)."""
    from wespeaker_b200.speaker import Speaker
    table = {"a.wav": torch.tensor([1.0, 0.0, 0.0]), "b.wav": torch.tensor([0.0, 2.0, 0.0]),
             "q.wav": torch.tensor([0.6, 0.8, 0.0]), "silence.wav": None}
    spk = Speaker(model=object())
    monkeypatch.setattr(spk, "extract_embedding", lambda p: table[p])
    assert spk.cosine_similarity(table["a.wav"], table["a.wav"]) == pytest.approx(1.0)
    assert spk.cosine_similarity(table["a.wav"], table["b.wav"]) == pytest.approx(0.5)       # cos 0 -> 0.5
    assert spk.compute_similarity("a.wav", "q.wav") == pytest.approx((0.6 + 1.0) / 2)
    assert spk.compute_similarity("a.wav", "silence.wav") == 0.0                              # None embedding
    spk.register("alice", "a.wav")
    spk.register("bob", "b.wav")
    spk.register("alice", "b.wav")                                                            # ignored, with the reference's message
    assert "already registered" in capsys.readouterr().out
    assert torch.equal(spk.table["alice"], table["a.wav"])
    r = spk.recognize("q.wav")
    assert r["name"] == "bob" and r["confidence"] == pytest.approx((0.8 + 1.0) / 2)
    assert Speaker(model=object()).recognize.__self__.table == {}


def test_kaldi_matrix_formats_and_random_chunk(tmp_path):
    """Kaldi matrix reader (`kaldiio.load_mat` analogue used by data_type=feat): FM / DM exactly, CM2 / CM3 / CM (compressed
    matrix, compressed-matrix.h) against the values the format defines; get_random_chunk against processor.py:315-347."""
    import random
    import struct
    from wespeaker_b200 import kaldi_io
    from wespeaker_b200.extract import get_random_chunk
    rng = np.random.default_rng(0)
    m = rng.standard_normal((7, 5)).astype(np.float32)
    with kaldi_io.MatrixWriter(str(tmp_path / "m.ark"), str(tmp_path / "m.scp")) as w:
        loc = w("key1", m)
        loc2 = w("key2", 2 * m)
    assert np.array_equal(kaldi_io.load_mat(loc), m) and np.array_equal(kaldi_io.load_mat(loc2), 2 * m)
    assert np.array_equal(kaldi_io.load_mat(str(tmp_path / "m.ark")), m)          # bare ark: first matrix
    hdr = lambda tok, r, c: b"\0B" + tok + b"\4" + struct.pack("<i", r) + b"\4" + struct.pack("<i", c)  # noqa: E731
    (tmp_path / "d.ark").write_bytes(hdr(b"DM ", 7, 5) + m.astype("<f8").tobytes())
    assert np.array_equal(kaldi_io.load_mat(str(tmp_path / "d.ark")), m)
    vmin, vrange = float(m.min()), float(m.max() - m.min())
    q16 = np.round((m - vmin) / vrange * 65535).astype("<u2")
    (tmp_path / "c2.ark").write_bytes(b"\0BCM2 " + struct.pack("<ffii", vmin, vrange, 7, 5) + q16.tobytes())
    assert np.abs(kaldi_io.load_mat(str(tmp_path / "c2.ark")) - m).max() <= vrange / 65535
    q8 = np.round((m - vmin) / vrange * 255).astype("u1")
    (tmp_path / "c3.ark").write_bytes(b"\0BCM3 " + struct.pack("<ffii", vmin, vrange, 7, 5) + q8.tobytes())
    assert np.abs(kaldi_io.load_mat(str(tmp_path / "c3.ark")) - m).max() <= vrange / 255
    # CM: per-column percentile headers; bytes 0 / 64 / 192 / 255 decode to the 0th / 25th / 75th / 100th percentile values
    ph = np.array([[0, 16384, 49152, 65535]] * 5, dtype="<u2")
    codes = np.array([[0, 64, 192, 255, 32, 128, 224]] * 5, dtype="u1")           # (cols, rows): column-major bytes
    (tmp_path / "c1.ark").write_bytes(b"\0BCM " + struct.pack("<ffii", -1.0, 2.0, 7, 5) + ph.tobytes() + codes.tobytes())
    got = kaldi_io.load_mat(str(tmp_path / "c1.ark"))
    p = -1.0 + 2.0 * ph[0].astype(np.float64) / 65535
    want = [p[0], p[1], p[2], p[3], p[0] + (p[1] - p[0]) * 32 / 64, p[1] + (p[2] - p[1]) * 64 / 128, p[2] + (p[3] - p[2]) * 32 / 63]
    assert got.shape == (7, 5) and np.abs(got[:, 0] - np.array(want)).max() < 1e-6 and np.array_equal(got[:, 0], got[:, 4])
    # chunks: long input -> a window at the generator's start; short input -> tiled then cut
    x = np.arange(1000)
    r1, r2 = random.Random(3), random.Random(3)
    s0 = r2.randint(0, 1000 - 300)
    assert np.array_equal(get_random_chunk(x, 300, r1), x[s0:s0 + 300])
    assert np.array_equal(get_random_chunk(np.arange(7), 17, r1), np.tile(np.arange(7), 3)[:17])
    f = rng.standard_normal((5, 4))
    assert np.array_equal(get_random_chunk(f, 12, r1), np.tile(f, (3, 1))[:12])


def test_resample_oracle_matches_torchaudio_goldens():
    """oracle/resample_np.py (restated torchaudio sinc resampler) against outputs of torchaudio.transforms.Resample itself
    (tests/golden/make_golden_resample.py): the call the reference makes in processor.py:258-259 / cli/speaker.py:158-159."""
    from oracle import resample_np
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "resample.npz"))
    for tag in ("8k_16k", "44k1_16k", "48k_16k", "22k05_16k", "16k_8k"):
        o, n = (int(v) for v in g[f"{tag}_rates"])
        x, y = g[f"{tag}_x"], g[f"{tag}_y"]
        r = resample_np.resample(x, o, n)
        assert r.shape == y.shape
        assert np.abs(r - y).max() <= 1e-5 * np.abs(y).max(), tag



# ------------------------------------------------------------------------------------------ plan-check engine (no device)
PLAN_CASES = [("ECAPA_TDNN_c1024", "bf16", 256, 200), ("ECAPA_TDNN_c512", "tf32x3", 256, 200), ("ECAPA_TDNN_GLOB_c512", "fp32", 3, 301),
              ("ResNet34", "fp16", 64, 200), ("ResNet18", "tf32x3", 2, 99), ("ResNet50", "bf16", 2, 99), ("ResNet101", "fp32", 1, 64),
              ("CAMPPlus", "bf16", 64, 200), ("CAMPPlus", "fp32", 2, 998), ("XVEC", "bf16", 3, 200)]


@pytest.mark.parametrize("name,prec,B,T", PLAN_CASES)
def test_plan_check_builds_every_family_without_a_device(name, prec, B, T):
    """ws_engine_create_plan_check: the whole weight-ingest + plan-building path (key names, shapes, folding, kernel envelopes,
    tensor-map rules) runs on a host without a GPU; nothing is computed."""
    m = from_synthetic(name, precision=prec)
    ops = m.plan_check(B, T)
    assert len(ops) >= 5 and all(isinstance(n, str) and n for n, _ in ops)
    gflop = sum(f for _, f in ops) / B / 1e9
    assert gflop > 0.5, (name, gflop)                      # the conv / GEMM ops carry their algorithmic FLOPs
    if name == "ECAPA_TDNN_c1024" and prec == "bf16":      # SURVEY section 8(d): 5.14 GFLOP per 200-frame utterance
        assert abs(gflop - 5.14) < 0.05, gflop
        assert any(n.startswith("conv_tc3") and "K=3072 N=1536" in n for n, _ in ops)
        assert sum(n.startswith("res2_fused") for n, _ in ops) == 3 and sum(n.startswith("astp_fused") for n, _ in ops) == 1
    if name == "ResNet34" and prec == "fp16":
        assert sum(n.startswith("conv3x3") for n, _ in ops) >= 24   # layers 1-3 on the halo-resident kernel


def test_plan_check_reports_missing_and_misshaped_tensors_and_never_computes():
    m = from_synthetic("ResNet34", precision="fp16")
    del m._sd["layer2.0.shortcut.0.weight"]
    del m._sd["layer3.1.bn1.running_var"]
    with pytest.raises(lib.B200Error, match="layer3.1.bn1.running_var"):
        m.plan_check(2, 100)
    # a plan-check engine refuses every compute entry point
    import ctypes as C
    L = lib.load()
    h = lib.c_engine_p()
    lib.check(L.ws_engine_create_plan_check(b"XVEC", b"bf16", 80, 512, C.byref(h)), "create")
    try:
        assert L.ws_engine_forward_host(h, None, 1, 200, None) != 0
        buf = np.zeros((1, 200, 80), np.float32)
        out = np.zeros((1, 512), np.float32)
        assert L.ws_engine_forward_host(h, buf.ctypes.data, 1, 200, out.ctypes.data) != 0
        assert b"plan-check engine" in L.ws_last_error()
    finally:
        L.ws_engine_destroy(h)


def test_tc_version_selects_the_persistent_kernel_and_refuses_1():
    """tc_version 2 puts every tensor-core conv on the persistent kernel, 3 (the default) adds weight-sharing clusters on the
    large layers.  1 named the one-tile-per-CTA kernel, which is gone: the option and ws_conv's use_tc = 1 are errors."""
    import ctypes as C
    labels = {}
    for v in (2, 3):
        m = from_synthetic("ECAPA_TDNN_c512", precision="bf16")
        m.set_option("tc_version", v)
        labels[v] = [n for n, _ in m.plan_check(128, 200)]
    assert any(n.startswith("conv_tc2") for n in labels[2]) and not any(n.startswith("conv_tc3") for n in labels[2])
    assert any(n.startswith("conv_tc3") for n in labels[3])
    m = from_synthetic("ECAPA_TDNN_c512", precision="bf16")
    m.set_option("tc_version", 1)
    with pytest.raises(lib.B200Error, match="one-tile-per-CTA"):
        m.plan_check(2, 200)
    L = lib.load()
    d = lib.ConvDesc()
    d.use_tc = 1
    assert L.ws_conv(C.byref(d), None) != 0
    assert b"one-tile-per-CTA" in L.ws_last_error()


@pytest.mark.parametrize("name,prec,B,T", [("ResNet34", "fp16", 2, 99), ("ResNet34", "tf32x3", 1, 40), ("ResNet50", "bf16", 1, 64),
                                          ("XVEC", "bf16", 2, 40)])
def test_plan_arithmetic_matches_oracle_on_the_host(name, prec, B, T, tmp_path):
    """ws_engine_plan_trace + tests/plan_interp.py: the launch plan (BN folding, merged shortcut K ranges, strided convs as
    parity planes, the halo-resident 3x3 ops with in-place residuals, TSTP index order, folded segment layers) re-evaluated on
    the host equals the oracle; the kernels executing the same plan are checked on the GPU."""
    from oracle import models_torch
    from plan_interp import run_plan
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    m = from_synthetic(name, precision=prec)
    path = str(tmp_path / "plan.bin")
    m.plan_trace(path, B, T)
    feats = syn.make_feats(B, T, 80, seed=5)
    emb, meta = run_plan(path, feats)
    ref = models_torch.forward(name, syn.make_state_dict(name, 0), feats).numpy()
    rel = np.linalg.norm(emb - ref, axis=1) / np.linalg.norm(ref, axis=1)
    assert rel.max() < 1e-5, rel
