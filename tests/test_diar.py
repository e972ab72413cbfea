"""Diarization (wespeaker_b200.diar, ws_diar.cu, Speaker.diarize).

CPU part: the numpy oracle and the host-side sub-segment tables against goldens produced by the reference's own
subsegment / cluster / merge_segments (tests/golden/make_golden_diar.py), plan builds at the window length, argument errors.
GPU part: the ragged fbank, the window kernel and the Laplacian kernels through the C ABI against the oracle and the
goldens, the device clusterer, and Speaker.diarize end to end on a synthetic recording."""
import os
import wave

import numpy as np
import pytest
import torch

from oracle import diar_np
from wespeaker_b200 import diar, frontend, lib
from wespeaker_b200.models import SUPPORTED_MODELS, from_synthetic
from wespeaker_b200.speaker import Speaker

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "diar.npz"))
gpu = pytest.mark.gpu
SEGS = [tuple(s) for s in G["segments_s"]]
KEPT = [k for k, (b, e) in enumerate(SEGS) if e - b >= 0.255]


def _seg_id(b, e):
    return "{:08d}-{:08d}".format(int(b * 1000), int(e * 1000))


def _padded(table, cols=16):
    """The golden per-segment 'fbank' matrices laid out as the ragged fbank launch would: [B][max_frames][cols]."""
    buf = np.full((len(table.row_offset), table.max_frames, cols), np.nan, dtype=np.float32)
    starts = {int(SEGS[k][0] * 16000): k for k in KEPT}
    k, s0 = None, None
    for r, (off, n) in enumerate(zip(table.row_offset, table.row_frames)):
        if int(off) in starts:
            k, s0 = starts[int(off)], int(off)
        f0 = (int(off) - s0) // 160
        buf[r, :n] = G[f"fbank_{k}"][f0:f0 + n]
    return buf


# ------------------------------------------------------------------------------------------------- CPU: oracle pinned
def test_oracle_subsegment_matches_reference():
    ids, wins = [], []
    for k in KEPT:
        i, w = diar_np.subsegment(G[f"fbank_{k}"], _seg_id(*SEGS[k]))
        ids += i
        wins += w
    assert ids == [str(s) for s in G["subseg_ids"]]
    assert np.array_equal(np.stack(wins), G["subseg_windows"])


@pytest.mark.parametrize("tag", ["small", "large"])
def test_oracle_cluster_matches_reference(tag):
    labels, k, eig, lap = diar_np.cluster(G[f"emb_{tag}"])
    assert lap.dtype == np.float32 and np.array_equal(lap, G[f"lap_{tag}"])
    assert np.abs(eig[:32] - G[f"eig_{tag}"]).max() < 1e-3          # the reference's come from fp32 LAPACK
    assert k == int(G[f"num_spks_{tag}"])
    assert diar_np.same_partition(labels, G[f"labels_{tag}"])


def test_trivial_cluster_and_merge_match_reference():
    assert np.array_equal(diar_np.cluster(G["emb_tiny"])[0], G["labels_tiny"])
    assert np.array_equal(diar.cluster(G["emb_tiny"]), G["labels_tiny"])      # m <= 2 never reaches the device
    seq = [(b, e, int(la)) for b, e, la in G["merge_in"]]
    want = [("rec", b, e, int(la)) for b, e, la in G["merge_out"]]
    assert diar_np.merge_segments("rec", seq) == want
    assert diar.merge_segments({"rec": seq}) == want
    assert diar.merge_segments({"a": [], "b": seq[:1]}) == [("b",) + seq[0]]


@pytest.mark.parametrize("cap", [None, 64, 1024])
def test_subsegment_table_matches_reference(cap):
    t = diar.subsegment_table(SEGS, max_row_frames=cap)
    assert t.ids == [str(s) for s in G["subseg_ids"]]
    assert t.max_frames == (1705 if cap is None else min(cap, 1705)) and t.row_frames.max() == t.max_frames
    assert len(t.row_offset) == (len(KEPT) if cap is None else sum(-(-(len(G[f"fbank_{k}"])) // cap) for k in KEPT))
    flat = _padded(t).reshape(-1, 16)
    diar.check_tables(t.win_row0, t.win_len, len(flat))
    got = np.stack([flat[r0 + np.arange(150) % n] for r0, n in zip(t.win_row0, t.win_len)])
    assert np.array_equal(got, G["subseg_windows"])                 # NaN padding rows are never gathered
    assert [len(G[f"fbank_{k}"]) for k in KEPT] == t.seg_len.tolist()
    for s, k in enumerate(KEPT):
        assert np.array_equal(flat[t.seg_row0[s]:t.seg_row0[s] + t.seg_len[s]], G[f"fbank_{k}"])


def test_subsegment_table_clips_at_the_recording_end_and_refuses_segments_outside_it():
    t = diar.subsegment_table([(0.0, 3.0)], num_samples=40000)      # 2.5 s of audio: 248 frames, seg_length 300
    assert t.seg_len.tolist() == [248] and t.win_len.tolist() == [150, 150, 98]
    with pytest.raises(ValueError):
        diar.subsegment_table([(0.0, 3.0)], num_samples=20000)      # the last window would have no row
    with pytest.raises(ValueError):
        diar.subsegment_table([(5.0, 6.0)], num_samples=30000)


@pytest.mark.parametrize("B", [256, 1])
@pytest.mark.parametrize("name", SUPPORTED_MODELS)
def test_every_model_builds_a_plan_at_the_window_length(name, B):
    """Diarization feeds the engine [B][150][80] windows: a full chunk and a 1-window tail, for every model in the table."""
    assert len(from_synthetic(name, precision="bf16").plan_check(B, 150)) > 0


def test_argument_errors(tmp_path):
    sp = Speaker(model=from_synthetic("ECAPA_TDNN_c512"))
    with pytest.raises(NotImplementedError, match="VAD"):
        sp.diarize("missing.wav")
    assert sp.diarize("missing.wav", segments=[]) == []
    ids, embs = diar.extract_subsegment_embeddings(sp.model, torch.zeros(16000), [(0.0, 0.1)])   # below min_duration
    assert ids == [] and tuple(embs.shape) == (0, 192)
    with pytest.raises(ValueError, match="16384"):
        diar.cluster(np.zeros((16385, 4), np.float32))
    with pytest.raises(ValueError, match="outside"):
        diar.check_tables([0, 10], [150, 150], 159)
    with pytest.raises(ValueError):
        diar.check_tables([0], [0], 10)
    seg = tmp_path / "segments"
    seg.write_text("rec-0 rec 0.50 1.75\nrec-1 rec 2.0 3.0\nseg other 0 1\n")
    assert diar.read_segments(str(seg)) == {"rec": [("rec-0", 0.5, 1.75), ("rec-1", 2.0, 3.0)], "other": [("seg", 0.0, 1.0)]}
    out = tmp_path / "x.rttm"
    sp.make_rttm([("rec", 0.5, 1.125, 2)], str(out))
    assert out.read_text() == "SPEAKER rec 1 0.500 0.625 <NA> <NA> 2 <NA> <NA>\n"
    assert diar.subseg_times("00014000-00031070-00000075-00000225") == (14.75, 16.25)


def test_diar_needs_gpu_and_fails_loudly():
    if torch.cuda.is_available():
        pytest.skip("CPU-only check")
    with pytest.raises(lib.B200Error):
        diar.cluster(G["emb_small"])
    with pytest.raises(lib.B200Error):
        diar.windows(torch.zeros(10, 80), [0], [10])


# ------------------------------------------------------------------------------------------------- GPU
@gpu
@pytest.mark.parametrize("cap", [None, 64])
def test_gpu_fbank_ragged_equals_each_segment_alone(cap):
    """fbank once per segment, segments at odd sample offsets, long ones split into rows: nothing changes, bit for bit."""
    rng = np.random.default_rng(3)
    wav = torch.from_numpy((rng.standard_normal(16000 * 8) * 3000).astype(np.float32)).cuda()
    segs = [(0.0131, 0.4), (0.50007, 2.73), (3.0, 3.9999), (4.2, 7.99)]
    t = diar.subsegment_table(segs, num_samples=wav.numel(), max_row_frames=cap)
    feats = diar.fbank_ragged(wav, t.row_offset, t.row_frames, t.max_frames).reshape(-1, 80)
    for s, (b, e) in enumerate(segs):
        alone = frontend.fbank_batch(wav[None, int(b * 16000):int(e * 16000)])[0]
        assert alone.shape[0] == t.seg_len[s]
        assert torch.equal(feats[t.seg_row0[s]:t.seg_row0[s] + t.seg_len[s]], alone)
    with pytest.raises(ValueError):
        diar.fbank_ragged(wav, [wav.numel() - 500], [2], 2)


@gpu
@pytest.mark.parametrize("cap", [None, 64])
def test_gpu_windows_match_oracle(cap):
    t = diar.subsegment_table(SEGS, max_row_frames=cap)
    feats = torch.from_numpy(np.nan_to_num(_padded(t))).cuda()
    want = G["subseg_windows"]
    assert np.array_equal(diar.windows(feats, t.win_row0, t.win_len, cmn="none").cpu().numpy(), want)
    got = diar.windows(feats, t.win_row0, t.win_len, cmn="window").cpu().numpy()
    assert np.abs(got - diar_np.window_cmn(want)).max() <= 1e-5
    means = diar.col_means(feats, t.seg_row0, t.seg_len)
    seg_mean = np.stack([G[f"fbank_{k}"].astype(np.float64).mean(axis=0) for k in KEPT])
    assert np.abs(means.cpu().numpy() - seg_mean).max() <= 1e-5
    got = diar.windows(feats, t.win_row0, t.win_len, cmn="segment", seg_mean=means, win_seg=t.win_seg).cpu().numpy()
    assert np.abs(got - (want - seg_mean[t.win_seg][:, None, :].astype(np.float32))).max() <= 1e-5


@gpu
def test_gpu_windows_edge_lengths_and_refused_tables():
    rng = np.random.default_rng(5)
    x = rng.standard_normal((400, 80)).astype(np.float32)
    feats = torch.from_numpy(x).cuda()
    row0, length = [7, 250, 0, 399], [1, 150, 149, 1]
    got = diar.windows(feats, row0, length, cmn="window").cpu().numpy()
    want = diar_np.window_cmn(np.stack([x[r + np.arange(150) % n] for r, n in zip(row0, length)]))
    assert np.abs(got - want).max() <= 1e-5
    got = diar.windows(feats, [0, 100], [100, 100], window_fs=200, cmn="none").cpu().numpy()   # another window length
    assert np.array_equal(got[1], np.concatenate([x[100:200], x[100:200]]))
    with pytest.raises(ValueError):
        diar.windows(feats, [300], [101])
    # the kernel itself skips an entry outside the buffer (zeros, no read) if a caller hands it one
    L = lib.load()
    r0 = torch.tensor([390, 0, -1], dtype=torch.int32).cuda()
    ln = torch.tensor([20, 0, 5], dtype=torch.int32).cuda()
    out = torch.full((3, 150, 80), 7.0, device="cuda")
    lib.check(L.ws_diar_windows(feats.data_ptr(), 400, 80, r0.data_ptr(), ln.data_ptr(), 3, 150, 1, None, None, 0,
                                out.data_ptr(), lib.cur_stream_ptr(0)), "ws_diar_windows")
    assert float(out.abs().max()) == 0.0


@gpu
@pytest.mark.parametrize("tag", ["small", "large"])
def test_gpu_laplacian_and_cluster_match_reference(tag):
    emb = G[f"emb_{tag}"]
    lap = diar.laplacian(emb)
    assert lap.dtype == torch.float64 and np.array_equal(lap.cpu().numpy(), G[f"lap_{tag}"].astype(np.float64))
    tiled = diar.laplacian(torch.from_numpy(emb).cuda(), tile_bytes=4 * len(emb) * 37)     # ragged last row tile
    assert torch.equal(tiled, lap)
    eig = torch.linalg.eigvalsh(lap)[:32].cpu().numpy()
    assert np.abs(eig - G[f"eig_{tag}"]).max() < 1e-3
    labels = diar.cluster(torch.from_numpy(emb).cuda())
    assert len(set(labels.tolist())) == int(G[f"num_spks_{tag}"])
    assert diar_np.same_partition(labels, G[f"labels_{tag}"])
    assert np.array_equal(labels, diar.cluster(emb)) and labels[0] == 0                     # clusters numbered by first appearance
    assert len(set(diar.cluster(emb, num_spks=2).tolist())) == 2


@gpu
def test_gpu_laplacian_ties_go_to_the_lowest_columns():
    emb = np.eye(4, dtype=np.float32)[[0, 1, 1, 1, 2, 2, 3, 0, 1, 2, 3, 3, 0]]     # rows with many exactly equal cosines
    lap = diar.laplacian(emb).cpu().numpy()
    cos = emb @ emb.T
    keep = diar.keep_per_row(len(emb))
    adj = np.zeros_like(cos)
    for i in range(len(emb)):
        adj[i, np.argsort(-cos[i], kind="stable")[:keep]] = 1.0                    # stable: the lowest columns win ties
    sym = 0.5 * (adj + adj.T)
    np.fill_diagonal(sym, 0.0)
    assert np.array_equal(lap, np.diag(sym.sum(axis=1)) - sym)


def _recording(seed=0):
    """Three sources (seeded noise through different one-pole / resonant filters) taking turns with gaps."""
    from scipy.signal import lfilter
    rng = np.random.default_rng(seed)
    filt = [([1.0], [1.0, -0.9]), ([1.0, -0.95], [1.0]), ([1.0], [1.0, -1.2, 0.8])]
    turns = [(0.40, 3.10, 0), (3.60, 5.35, 1), (5.90, 10.20, 2), (10.50, 11.30, 0), (11.80, 30.00, 1), (30.40, 33.00, 2),
             (33.20, 33.40, 0)]
    pcm = rng.standard_normal(16000 * 34) * 5.0
    for b, e, s in turns:
        n = int(e * 16000) - int(b * 16000)
        y = lfilter(*filt[s], rng.standard_normal(n))
        pcm[int(b * 16000):int(e * 16000)] = 4000.0 * y / np.abs(y).max()
    return np.round(pcm).astype(np.int16), [(b, e) for b, e, _ in turns]


@gpu
@pytest.mark.parametrize("name,prec,tol", [("ECAPA_TDNN_c512", "tf32x3", 1e-4), ("ResNet34", "fp16", 1e-2)])
def test_gpu_speaker_diarize_matches_the_pipeline_assembled_from_oracle_pieces(tmp_path, name, prec, tol):
    """Speaker.diarize against the same pipeline put together on the host: fbank of each segment alone, oracle
    sub-segmentation and window CMN, the model on the stacked windows (batches of 32), oracle Laplacian and eigengap rule,
    oracle merging.  Random-weight models do not separate the sources, so the partition is not stable under the embedding
    tolerance and is not compared across the two k-means implementations: asserted instead are the windows (5e-5), the
    embeddings (the precision's bar), >= 99 % agreement of the Laplacian's edges, equal num_spks where the Laplacians are
    identical, and the merged segments (1e-6 s) for the device labels."""
    pcm, segs = _recording()
    path = str(tmp_path / "rec.wav")
    with wave.open(path, "wb") as w:
        w.setnchannels(1)
        w.setsampwidth(2)
        w.setframerate(16000)
        w.writeframes(pcm.tobytes())
    model = from_synthetic(name, precision=prec)
    sp = Speaker(model=model)
    got = sp.diarize(path, "rec", segs)
    assert got and all(u == "rec" and e > b for u, b, e, _ in got)
    assert got[0][1] == 0.4 and abs(got[-1][2] - 33.0) < 1e-9          # the 0.2 s turn is below min_duration

    wav = torch.from_numpy(pcm.astype(np.float32)).cuda()
    ids, embs, wins = diar.extract_subsegment_embeddings(model, wav, segs, return_windows=True)
    o_ids, o_wins = [], []
    for b, e in segs:
        if e - b < 0.255:
            continue
        fb = frontend.fbank_batch(wav[None, int(b * 16000):int(e * 16000)])[0].cpu().numpy()
        i, w = diar_np.subsegment(fb, _seg_id(b, e))
        o_ids += i
        o_wins += w
    o_wins = diar_np.window_cmn(np.stack(o_wins))
    assert ids == o_ids and np.abs(wins.cpu().numpy() - o_wins).max() <= 5e-5   # log-mel values near 20, two fp32 sum orders
    x = torch.from_numpy(o_wins).cuda()
    o_embs = torch.cat([model.embed(x[i:i + 32]) for i in range(0, len(x), 32)]).cpu().numpy()
    e = embs.cpu().numpy()
    assert (np.linalg.norm(e - o_embs, axis=1) / np.linalg.norm(o_embs, axis=1)).max() <= tol

    lap = diar.laplacian(embs).cpu().numpy()
    o_lap = diar_np.laplacian(o_embs).astype(np.float64)
    off = ~np.eye(len(e), dtype=bool)
    assert (lap[off] == o_lap[off]).mean() >= 0.99
    labels = diar.cluster(embs)
    if np.array_equal(lap, o_lap):
        assert len(set(labels.tolist())) == diar_np.num_speakers(np.linalg.eigvalsh(o_lap))
    want = diar_np.merge_segments("rec", [(*diar_np.subseg_times(s), int(la)) for s, la in zip(o_ids, labels)])
    assert len(got) == len(want)
    for (_, b0, e0, l0), (_, b1, e1, l1) in zip(got, want):
        assert abs(b0 - b1) <= 1e-6 and abs(e0 - e1) <= 1e-6 and l0 == l1
