"""numpy restatement of the reference's diarization arithmetic (test oracle, CPU):
sub-segmentation with its seg_length-vs-frame-count quirk and cyclic tiling (`wespeaker/diar/extract_emb.py:55-83`), window
and segment CMN (`cli/speaker.py:110-112`, `diar/make_fbank.py:85-86`), the spectral clusterer's fp32 affinity / pruning /
Laplacian and eigengap rule (`diar/spectral_clusterer.py:33-87`) and segment merging (`diar/make_rttm.py:47-70`).
Pinned on the reference's own functions by tests/golden/make_golden_diar.py."""
import numpy as np
import scipy.linalg


def num_frames(num_samples: int) -> int:
    return 0 if num_samples < 400 else 1 + (num_samples - 400) // 160


def subsegment(fbank, seg_id, window_fs=150, period_fs=75, frame_shift=10):
    """(T, F) fbank of one segment "…{begin_ms}-{end_ms}" -> (sub-segment ids, list of (window_fs, F) windows).  Window
    bounds are counted on seg_length = (end_ms - begin_ms) // frame_shift (T + 2 for a kaldi fbank); the rows actually
    there, fbank[begin:min(end, T)], are repeated cyclically up to window_fs rows."""
    begin_ms, end_ms = (int(v) for v in seg_id.split("-")[-2:])
    seg_length = (end_ms - begin_ms) // frame_shift
    begins = [0] if seg_length <= window_fs else list(range(0, seg_length - window_fs + period_fs, period_fs))
    ids, wins = [], []
    for b in begins:
        e = min(b + window_fs, seg_length)
        rows = fbank[b:e]
        ids.append("{}-{:08d}-{:08d}".format(seg_id, b, e))
        wins.append(rows[np.arange(window_fs) % len(rows)])
    return ids, wins


def window_cmn(windows):
    """(W, window_fs, F) -> minus each window's own mean over its (tiled) rows."""
    windows = np.asarray(windows, dtype=np.float32)
    return windows - windows.mean(axis=1, keepdims=True)


def laplacian(embeddings, p=0.01):
    """fp32 throughout, as the reference: S = (1 + cos) / 2; per row the m - n largest -> 1, the rest -> 0; symmetrise;
    clear the diagonal; diag(row sums) - matrix."""
    x = np.asarray(embeddings)
    x = x / np.linalg.norm(x, axis=1, keepdims=True)
    sim = 0.5 * (1.0 + np.dot(x, x.T))
    m = sim.shape[0]
    n = max(m - 10, 2) if m < 1000 else int((1.0 - p) * m)
    order = np.argsort(sim, axis=1)
    pruned = np.zeros_like(sim)
    np.put_along_axis(pruned, order[:, n:], 1.0, axis=1)
    sym = 0.5 * (pruned + pruned.T)
    np.fill_diagonal(sym, 0.0)
    return np.diag(np.abs(sym).sum(axis=1)) - sym


def num_speakers(eig_values, num_spks=None, min_num_spks=1, max_num_spks=20):
    if num_spks is None:
        num_spks = int(np.argmax(np.diff(eig_values[:max_num_spks + 1]))) + 1
    return max(num_spks, min_num_spks)


def kmeans(data, k, seed=0, n_init=10, max_iter=300):
    """Seeded k-means++ / Lloyd, best inertia of n_init starts (the reference's sklearn k_means is unseeded; compare
    partitions, not label values)."""
    rng = np.random.default_rng(seed)
    data = np.asarray(data, dtype=np.float64)
    best, best_inertia = None, None
    for _ in range(n_init):
        centers = data[[rng.integers(len(data))]]
        for _ in range(1, k):
            d2 = ((data[:, None] - centers[None]) ** 2).sum(-1).min(axis=1)
            centers = np.vstack([centers, data[rng.choice(len(data), p=d2 / d2.sum())]])
        labels = None
        for _ in range(max_iter):
            new = ((data[:, None] - centers[None]) ** 2).sum(-1).argmin(axis=1)
            if labels is not None and np.array_equal(new, labels):
                break
            labels = new
            for c in range(k):
                if (labels == c).any():
                    centers[c] = data[labels == c].mean(axis=0)
        inertia = ((data - centers[labels]) ** 2).sum()
        if best_inertia is None or inertia < best_inertia:
            best, best_inertia = labels, inertia
    return best


def cluster(embeddings, p=0.01, num_spks=None, min_num_spks=1, max_num_spks=20, seed=0):
    """-> (labels, num_spks, eigenvalues, Laplacian)."""
    m = len(embeddings)
    if m <= 2:
        return np.zeros(m, dtype=np.int64), 1, None, None
    lap = laplacian(embeddings, p)
    eig_values, eig_vectors = scipy.linalg.eigh(lap.astype(np.float64))
    k = num_speakers(eig_values, num_spks, min_num_spks, max_num_spks)
    labels = np.zeros(m, dtype=np.int64) if k == 1 else kmeans(eig_vectors[:, :k], k, seed)
    return labels, k, eig_values, lap


def same_partition(a, b) -> bool:
    """Two labelings name the same partition (label values are arbitrary)."""
    a, b = np.asarray(a), np.asarray(b)
    if a.shape != b.shape:
        return False
    pairs = set(zip(a.tolist(), b.tolist()))
    return len(pairs) == len(set(a.tolist())) == len(set(b.tolist()))


def subseg_times(subseg_id, frame_shift=10):
    begin_ms, _, begin_frame, end_frame = (int(v) for v in subseg_id.split("-")[-4:])
    return (begin_ms + begin_frame * frame_shift) / 1000.0, (begin_ms + end_frame * frame_shift) / 1000.0


def merge_segments(utt, subsegs):
    """[(begin, end, label)] in time order -> [(utt, begin, end, label)]: neighbours that touch or overlap and share a label
    are joined; a label change inside an overlap puts the boundary at the overlap's midpoint; a gap closes the segment."""
    out = []
    if not subsegs:
        return out
    cur_b, cur_e, cur_l = subsegs[0]
    for b, e, la in subsegs[1:]:
        if b <= cur_e and la == cur_l:
            cur_e = e
            continue
        cut = cur_e if b > cur_e else (b + cur_e) / 2.0
        out.append((utt, cur_b, cut, cur_l))
        cur_b, cur_e, cur_l = (b if b > cur_e else cut), e, la
    out.append((utt, cur_b, cur_e, cur_l))
    return out
