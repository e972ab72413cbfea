"""Speaker diarization of one recording on the GPU - mirror of `wespeaker/cli/speaker.py:213-289` with the recipe's pieces
(`wespeaker/diar/extract_emb.py:55-83`, `spectral_clusterer.py:33-87`, `make_rttm.py:47-70`, `make_fbank.py:39-49`).

Speech segments are an input (the reference finds them with silero VAD, whose weights are a download).  Per recording:
one ragged fbank launch over all segments (`ws_fbank_ragged`), one launch that cuts, cyclically tiles and mean-normalises
every sub-segment window (`ws_diar_windows`), the engine's forward on the `[W][window_fs][80]` windows, the pruned-affinity
Laplacian on the device (`ws_diar_laplacian`), then `torch.linalg.eigh` in fp64, the eigengap rule and a seeded k-means.
The clusterer is the reference's spectral one (its CLI imports the umap / hdbscan one instead).  No CPU fallback.
"""
from __future__ import annotations

from collections import OrderedDict, namedtuple

import numpy as np
import torch

from . import lib as _lib

FRAME_LEN, FRAME_SHIFT = 400, 160      # samples: the 25 ms / 10 ms frames of ws_fbank.cu at 16 kHz
MAX_EMBEDDINGS = 16384                 # WS_DIAR_MAX_M: a dense m x m fp64 Laplacian is 2 GB there

SubsegTable = namedtuple("SubsegTable", "ids row_offset row_frames max_frames win_row0 win_len win_seg seg_row0 seg_len")


def subsegment_table(segments, sample_rate: int = 16000, window_fs: int = 150, period_fs: int = 75, frame_shift: int = 10,
                     min_duration: float = 0.255, num_samples: int | None = None, max_row_frames: int | None = 1024):
    """Host-side plan of one recording: `segments` = [(begin_s, end_s)] -> SubsegTable of
    ids         sub-segment ids "{begin_ms:08d}-{end_ms:08d}-{begin_frame:08d}-{end_frame:08d}" (extract_emb.py:55-83; the
                frame range is counted on seg_length = (end_ms - begin_ms) // frame_shift, 2 more than the fbank has frames)
    row_offset  int64 [B], row_frames int32 [B]: the rows of the ragged fbank launch (first sample, frame count).  A segment
                with more than max_row_frames frames is split into several rows, which leaves its frames unchanged
                (every frame depends on its own 400 samples only) and bounds the padded [B][max_frames][80] buffer
    win_row0    int32 [W], win_len int32 [W]: window w is rows [row0, row0 + len) of the flat [B * max_frames][80] buffer,
                tiled cyclically to window_fs rows; len is clipped at the fbank's true frame count
    win_seg     int32 [W] segment of each window; seg_row0 / seg_len int32 [S]: each kept segment's rows in the flat buffer.
    Segments shorter than min_duration are dropped (cli/speaker.py:230); num_samples clips segments at the recording's end
    as slicing the waveform does."""
    kept = []
    for begin, end in segments:
        if end - begin < min_duration:
            continue
        s0, s1 = int(begin * sample_rate), int(end * sample_rate)
        if num_samples is not None:
            s0, s1 = min(s0, num_samples), min(s1, num_samples)
        n = s1 - s0
        frames = 0 if n < FRAME_LEN else 1 + (n - FRAME_LEN) // FRAME_SHIFT
        if frames == 0:
            raise ValueError(f"segment ({begin}, {end}) has no fbank frame inside the recording")
        kept.append((int(begin * 1000), int(end * 1000), s0, frames))
    cap = max_row_frames if max_row_frames else max((k[3] for k in kept), default=0)
    max_frames = min(cap, max((k[3] for k in kept), default=0))
    ids, row_offset, row_frames, win_row0, win_len, win_seg, seg_row0, seg_len = [], [], [], [], [], [], [], []
    for s, (b_ms, e_ms, s0, frames) in enumerate(kept):
        # rows of a split segment are full (max_frames frames) up to the last, so its frames are contiguous in the flat buffer
        first_row = len(row_offset) * max_frames
        for f0 in range(0, frames, cap):
            row_offset.append(s0 + FRAME_SHIFT * f0)
            row_frames.append(min(cap, frames - f0))
        seg_row0.append(first_row)
        seg_len.append(frames)
        seg_length = (e_ms - b_ms) // frame_shift
        begins = [0] if seg_length <= window_fs else range(0, seg_length - window_fs + period_fs, period_fs)
        for wb in begins:
            we = min(wb + window_fs, seg_length)
            rows = min(we, frames) - wb
            if rows <= 0:
                raise ValueError(f"segment ({b_ms} ms, {e_ms} ms) runs past the end of the recording")
            ids.append(f"{b_ms:08d}-{e_ms:08d}-{wb:08d}-{we:08d}")
            win_row0.append(first_row + wb)
            win_len.append(rows)
            win_seg.append(s)
    i32 = lambda v: np.asarray(v, dtype=np.int32)   # noqa: E731
    return SubsegTable(ids, np.asarray(row_offset, dtype=np.int64), i32(row_frames), int(max_frames), i32(win_row0),
                       i32(win_len), i32(win_seg), i32(seg_row0), i32(seg_len))


def check_tables(row0, length, total_rows: int):
    """Refuse (row0, len) tables that leave the [0, total_rows) feature buffer before they reach the device."""
    row0, length = np.asarray(row0, dtype=np.int64), np.asarray(length, dtype=np.int64)
    if row0.shape != length.shape or row0.ndim != 1:
        raise ValueError("row0 and len tables must be 1-D and of equal length")
    if row0.size and (row0.min() < 0 or length.min() <= 0 or (row0 + length).max() > total_rows):
        raise ValueError(f"window table points outside the {total_rows}-row feature buffer")


def _cuda(device=None) -> torch.device:
    if not torch.cuda.is_available():
        raise _lib.B200Error("wespeaker_b200.diar needs a CUDA device (no CPU fallback)")
    return torch.device("cuda", torch.cuda.current_device() if device is None else device)


def _dev_i32(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)).to(dev)


def fbank_ragged(pcm: torch.Tensor, row_offset, row_frames, max_frames: int, window_type: str = "hamming") -> torch.Tensor:
    """1-D CUDA waveform (int16, or float in int16 range) -> [B][max_frames][80] fp32 log-mel, no CMN; row b holds
    row_frames[b] frames starting at sample row_offset[b] (rows behind that are not written)."""
    if not pcm.is_cuda or pcm.dim() != 1:
        raise _lib.B200Error("fbank_ragged needs a 1-D CUDA waveform (no CPU fallback)")
    is_i16 = 1 if pcm.dtype == torch.int16 else 0
    pcm = pcm.contiguous() if is_i16 else pcm.float().contiguous()
    off, frm = np.asarray(row_offset, dtype=np.int64), np.asarray(row_frames, dtype=np.int32)
    B = off.size
    if B and (off.min() < 0 or frm.min() <= 0 or frm.max() > max_frames
              or (off + FRAME_SHIFT * (frm.astype(np.int64) - 1) + FRAME_LEN).max() > pcm.numel()):
        raise ValueError("fbank row table reaches outside the waveform")
    feats = torch.empty((B, max_frames, 80), dtype=torch.float32, device=pcm.device)
    if B == 0 or max_frames == 0:
        return feats
    off_d, frm_d = torch.from_numpy(off).to(pcm.device), torch.from_numpy(frm).to(pcm.device)
    idx = pcm.device.index
    with torch.cuda.device(idx):
        _lib.check(_lib.load().ws_fbank_ragged(pcm.data_ptr(), is_i16, pcm.numel(), off_d.data_ptr(), frm_d.data_ptr(),
                                               int(max_frames), B, window_type.encode(), feats.data_ptr(),
                                               _lib.cur_stream_ptr(idx)), "ws_fbank_ragged")
    return feats


def col_means(feats: torch.Tensor, row0, length) -> torch.Tensor:
    """Mean of rows [row0[s], row0[s] + len[s]) of the flat [rows][F] CUDA buffer `feats` -> [S][F]."""
    flat = feats.reshape(-1, feats.shape[-1])
    check_tables(row0, length, flat.shape[0])
    S = len(row0)
    out = torch.empty((S, flat.shape[1]), dtype=torch.float32, device=flat.device)
    idx = flat.device.index
    r0, ln = _dev_i32(row0, flat.device), _dev_i32(length, flat.device)
    with torch.cuda.device(idx):
        _lib.check(_lib.load().ws_diar_col_means(flat.data_ptr(), flat.shape[0], flat.shape[1], r0.data_ptr(), ln.data_ptr(), S,
                                                 out.data_ptr(), _lib.cur_stream_ptr(idx)), "ws_diar_col_means")
    return out


def windows(feats: torch.Tensor, row0, length, window_fs: int = 150, cmn: str = "window", seg_mean: torch.Tensor | None = None,
            win_seg=None) -> torch.Tensor:
    """Gather + cyclic tiling + CMN of sub-segment windows: `feats` is a CUDA fp32 buffer whose last dimension is the
    feature dimension (rows are counted over all leading dimensions); returns [W][window_fs][F].  cmn: "window" (the mean of
    the tiled window, cli/speaker.py:110-112), "segment" (seg_mean[win_seg[w]], make_fbank.py:85-86) or "none"."""
    if cmn not in ("window", "segment", "none"):
        raise ValueError(f"cmn must be 'window', 'segment' or 'none', not {cmn!r}")
    if not feats.is_cuda or feats.dtype != torch.float32:
        raise _lib.B200Error("diar.windows needs a CUDA float32 feature buffer (no CPU fallback)")
    flat = feats.contiguous().reshape(-1, feats.shape[-1])
    check_tables(row0, length, flat.shape[0])
    W, F = len(row0), flat.shape[1]
    out = torch.empty((W, window_fs, F), dtype=torch.float32, device=flat.device)
    if W == 0:
        return out
    dev, idx = flat.device, flat.device.index
    r0, ln = _dev_i32(row0, dev), _dev_i32(length, dev)
    sm_ptr = so_ptr = None
    S = 0
    if cmn == "segment":
        seg_mean = seg_mean.contiguous()
        S = seg_mean.shape[0]
        ws_ = np.asarray(win_seg, dtype=np.int32)
        if ws_.shape != (W,) or ws_.min() < 0 or ws_.max() >= S or tuple(seg_mean.shape) != (S, F):
            raise ValueError("win_seg / seg_mean do not match the window table")
        so = _dev_i32(ws_, dev)
        sm_ptr, so_ptr = seg_mean.data_ptr(), so.data_ptr()
    with torch.cuda.device(idx):
        _lib.check(_lib.load().ws_diar_windows(flat.data_ptr(), flat.shape[0], F, r0.data_ptr(), ln.data_ptr(), W,
                                               int(window_fs), int(cmn == "window"), sm_ptr, so_ptr, S, out.data_ptr(),
                                               _lib.cur_stream_ptr(idx)), "ws_diar_windows")
    return out


def extract_subsegment_embeddings(model, pcm: torch.Tensor, segments, sample_rate: int = 16000, window_secs: float = 1.5,
                                  period_secs: float = 0.75, frame_shift: int = 10, min_duration: float = 0.255,
                                  batch_size: int = 256, cmn: str = "window", window_type: str = "hamming",
                                  max_row_frames: int | None = 1024, return_windows: bool = False):
    """`cli/speaker.py:224-251` for one recording: waveform (N,) or (1, N) (int16, or float in int16 range) and speech
    segments [(begin_s, end_s)] -> (sub-segment ids, embeddings [m][E] CUDA tensor).  fbank runs once per segment; the
    embeddings do not depend on batch_size."""
    if sample_rate != 16000 or frame_shift != 10:
        raise NotImplementedError("the fbank kernel is built for 16 kHz audio and a 10 ms frame shift")
    if getattr(model, "feat_dim", 80) != 80:
        raise NotImplementedError("diarization runs on the 80-bin fbank")
    window_fs, period_fs = int(window_secs * 1000) // frame_shift, int(period_secs * 1000) // frame_shift
    pcm = pcm[0] if pcm.dim() == 2 else pcm
    table = subsegment_table(segments, sample_rate, window_fs, period_fs, frame_shift, min_duration, pcm.numel(), max_row_frames)
    if not table.ids:
        empty = torch.empty((0, model.embed_dim), dtype=torch.float32, device=pcm.device)
        return ([], empty, torch.empty((0, window_fs, 80), device=pcm.device)) if return_windows else ([], empty)
    pcm = pcm.to(pcm.device if pcm.is_cuda else _cuda())
    feats = fbank_ragged(pcm, table.row_offset, table.row_frames, table.max_frames, window_type)
    seg_mean = col_means(feats, table.seg_row0, table.seg_len) if cmn == "segment" else None
    wins = windows(feats, table.win_row0, table.win_len, window_fs, cmn, seg_mean, table.win_seg)
    embs = torch.cat([model.embed(wins[i:i + batch_size]) for i in range(0, wins.shape[0], batch_size)])
    return (table.ids, embs, wins) if return_windows else (table.ids, embs)


# ------------------------------------------------------------------------------------------------- spectral clustering
def keep_per_row(m: int, p: float = 0.01) -> int:
    """How many entries of each affinity row survive pruning (spectral_clusterer.py:39-44: the m - n largest)."""
    n = max(m - 10, 2) if m < 1000 else int((1.0 - p) * m)
    return m - n


def laplacian(embeddings, p: float = 0.01, device=None, tile_bytes: int = 1 << 28) -> torch.Tensor:
    """[m][E] embeddings (CUDA tensor or numpy) -> the m x m fp64 Laplacian of the pruned, symmetrised cosine affinity, on the
    device (spectral_clusterer.py:35-56)."""
    m = len(embeddings)
    if m > MAX_EMBEDDINGS:
        raise ValueError(f"{m} embeddings: more than {MAX_EMBEDDINGS} need a sparse eigensolver, not a dense m x m Laplacian")
    if m < 2:
        raise ValueError("the Laplacian needs at least 2 embeddings")
    if isinstance(embeddings, torch.Tensor) and embeddings.is_cuda:
        x = embeddings.detach().float().contiguous()
    else:
        x = torch.from_numpy(np.ascontiguousarray(np.asarray(embeddings), dtype=np.float32)).to(_cuda(device))
    dev, idx = x.device, x.device.index
    L = _lib.load()
    D = x.shape[1]
    unit = torch.empty((m, D), dtype=torch.float64, device=dev)
    rows = max(1, min(m, tile_bytes // (4 * m)))
    work = torch.empty((rows, m), dtype=torch.float32, device=dev)
    adj = torch.empty((m, m), dtype=torch.uint8, device=dev)
    lap = torch.empty((m, m), dtype=torch.float64, device=dev)
    with torch.cuda.device(idx):
        s = _lib.cur_stream_ptr(idx)
        _lib.check(L.ws_score_unit_rows(x.data_ptr(), m, D, None, unit.data_ptr(), None, s), "ws_score_unit_rows")
        _lib.check(L.ws_diar_laplacian(unit.data_ptr(), m, D, keep_per_row(m, p), work.data_ptr(), rows, adj.data_ptr(),
                                       lap.data_ptr(), s), "ws_diar_laplacian")
    return lap


def num_speakers(eig_values, num_spks=None, min_num_spks: int = 1, max_num_spks: int = 20) -> int:
    """The eigengap rule of spectral_clusterer.py:58-63 on ascending eigenvalues."""
    if num_spks is None:
        num_spks = int(np.argmax(np.diff(np.asarray(eig_values)[:max_num_spks + 1]))) + 1
    return max(int(num_spks), min_num_spks)


def kmeans(data: torch.Tensor, k: int, seed: int = 0, n_init: int = 10, max_iter: int = 300) -> torch.Tensor:
    """Seeded k-means++ / Lloyd on the rows of `data` (any device), best inertia of n_init starts -> int64 labels.  The
    same seed gives the same labels; the reference's k_means (random_state=None) gives the same partition on separable
    data and no particular label values."""
    m = data.shape[0]
    if k <= 1:
        return torch.zeros(m, dtype=torch.int64, device=data.device)
    gen = torch.Generator().manual_seed(seed)
    best, best_inertia = None, None
    for _ in range(n_init):
        centers = data[torch.randint(m, (1,), generator=gen)]
        for _ in range(1, k):
            d2 = torch.cdist(data, centers).pow(2).min(dim=1).values
            u = torch.rand((), generator=gen, dtype=torch.float64).item() * float(d2.sum())
            nxt = int(torch.searchsorted(torch.cumsum(d2, 0), torch.tensor(u, dtype=d2.dtype, device=d2.device)).clamp(max=m - 1))
            centers = torch.cat([centers, data[nxt:nxt + 1]])
        labels = None
        for _ in range(max_iter):
            new = torch.cdist(data, centers).argmin(dim=1)
            if labels is not None and torch.equal(new, labels):
                break
            labels = new
            sums = torch.zeros_like(centers).index_add_(0, labels, data)
            counts = torch.bincount(labels, minlength=k).to(data.dtype)[:, None]
            centers = torch.where(counts > 0, sums / counts.clamp(min=1), centers)   # an emptied cluster keeps its centre
        inertia = float((data - centers[labels]).pow(2).sum())
        if best_inertia is None or inertia < best_inertia:
            best, best_inertia = labels, inertia
    return best


def cluster(embeddings, p: float = .01, num_spks=None, min_num_spks: int = 1, max_num_spks: int = 20, seed: int = 0,
            device=None) -> np.ndarray:
    """`spectral_clusterer.cluster` (its signature plus the seed): [m][E] embeddings (CUDA tensor or numpy) -> numpy int
    labels, numbered in order of first appearance.  The Laplacian is built by ws_diar.cu; its eigendecomposition is
    torch.linalg.eigh in fp64 on the device."""
    m = len(embeddings)
    if m <= 2:
        return np.zeros(m, dtype=np.int64)
    lap = laplacian(embeddings, p, device)
    eig_values, eig_vectors = torch.linalg.eigh(lap)
    k = num_speakers(eig_values[:max_num_spks + 1].cpu().numpy(), num_spks, min_num_spks, max_num_spks)
    labels = kmeans(eig_vectors[:, :k].contiguous(), k, seed).cpu().numpy()
    # number the clusters by first appearance: label values then depend on the partition alone, not on which basis of a
    # repeated eigenvalue's eigenspace the solver returned
    _, first = np.unique(labels, return_index=True)
    rank = np.empty(labels.max() + 1, dtype=np.int64)
    rank[labels[np.sort(first)]] = np.arange(len(first))
    return rank[labels]


# ------------------------------------------------------------------------------------------------- segments in, RTTM out
def read_segments(segments_file: str):
    """The recipe's `segments` file (make_fbank.py:39-49; `seg utt begin_s end_s` per line) -> {utt: [(seg, begin, end)]}."""
    utt_to_segments = OrderedDict()
    with open(segments_file, "r", encoding="utf-8") as f:
        for line in f:
            seg, utt, begin, end = line.strip().split()
            utt_to_segments.setdefault(utt, []).append((seg, float(begin), float(end)))
    return utt_to_segments


def subseg_times(subseg_id: str, frame_shift: int = 10):
    """Sub-segment id -> (begin_s, end_s) in the recording (cli/speaker.py:259-263)."""
    begin_ms, _, begin_frame, end_frame = (int(v) for v in subseg_id.split("-")[-4:])
    return (begin_ms + begin_frame * frame_shift) / 1000.0, (begin_ms + end_frame * frame_shift) / 1000.0


def merge_segments(utt_to_subseg_labels):
    """{utt: [(begin, end, label)] in time order} -> [(utt, begin, end, label)] (make_rttm.py:47-70): overlapping
    neighbours with one label are joined; where the label changes inside an overlap the boundary is its midpoint."""
    merged = []
    for utt, subsegs in utt_to_subseg_labels.items():
        if len(subsegs) == 0:
            continue
        begin, end, label = subsegs[0]
        for b, e, la in subsegs[1:]:
            if b > end:
                merged.append((utt, begin, end, label))
                begin, end, label = b, e, la
            elif la == label:
                end = e
            else:
                pivot = (b + end) / 2.0
                merged.append((utt, begin, pivot, label))
                begin, end, label = pivot, e, la
        merged.append((utt, begin, end, label))
    return merged


def make_rttm(merged_segment_to_labels, outfile: str):
    """`cli/speaker.py:283-289`."""
    with open(outfile, "w", encoding="utf-8") as f:
        for utt, begin, end, label in merged_segment_to_labels:
            f.write("SPEAKER {} {} {:.3f} {:.3f} <NA> <NA> {} <NA> <NA>\n".format(utt, 1, float(begin),
                                                                                 float(end) - float(begin), label))
