"""Generate tests/golden/diar.npz by running the REAL reference diarization code.

Runs only where $WESPEAKER_REFERENCE names a checkout of wenet-e2e/wespeaker.  `wespeaker/diar/extract_emb.py:55-83`
(subsegment), `wespeaker/diar/spectral_clusterer.py:33-87` (cluster) and `wespeaker/diar/make_rttm.py:47-70`
(merge_segments) are imported with the package __init__ bypassed and `kaldiio`, `onnxruntime`, `tqdm` stubbed (none is
installed here or needed by these functions).  `cluster`'s steps are nested closures, so the Laplacian it hands to
`scipy.linalg.eigh` and the eigenvalues it gets back are recorded by wrapping that one function while `cluster` runs;
everything computed is the reference's own code.
"""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.path.join(os.environ["WESPEAKER_REFERENCE"], "wespeaker")
WINDOW_FS, PERIOD_FS, FRAME_SHIFT = 150, 75, 10


def _import_reference():
    for pkg, path in [("wespeaker", REF), ("wespeaker.diar", REF + "/diar"), ("wespeaker.utils", REF + "/utils")]:
        m = types.ModuleType(pkg)
        m.__path__ = [path]
        sys.modules[pkg] = m
    for name in ("kaldiio", "onnxruntime"):
        sys.modules[name] = types.ModuleType(name)
    tq = types.ModuleType("tqdm")
    tq.tqdm = lambda it, *a, **k: it
    sys.modules["tqdm"] = tq
    import wespeaker.diar.extract_emb as extract_emb
    import wespeaker.diar.make_rttm as make_rttm
    import wespeaker.diar.spectral_clusterer as spectral_clusterer
    return extract_emb, spectral_clusterer, make_rttm


def _same_partition(a, b):
    pairs = set(zip(np.asarray(a).tolist(), np.asarray(b).tolist()))
    return len(pairs) == len(set(np.asarray(a).tolist())) == len(set(np.asarray(b).tolist()))


def _boundary_gap(emb, p=0.01):
    """Smallest distance, over the rows, between the last kept and the first dropped fp32 similarity."""
    x = emb / np.linalg.norm(emb, axis=1, keepdims=True)
    s = np.sort(0.5 * (1.0 + np.dot(x, x.T)), axis=1)
    m = len(emb)
    n = max(m - 10, 2) if m < 1000 else int((1.0 - p) * m)
    return float((s[:, n] - s[:, n - 1]).min())


def _embeddings(rng, m, spk, dim, noise):
    centres = rng.standard_normal((spk, dim)).astype(np.float32)
    who = rng.integers(0, spk, m)
    return (centres[who] + noise * rng.standard_normal((m, dim))).astype(np.float32)


def main():
    extract_emb, spectral, make_rttm = _import_reference()
    import scipy.linalg
    rng = np.random.default_rng(11)
    out = {}

    # ---- sub-segmentation: seg_length below, equal to and one above window_fs; ending on a period boundary; long (>= 20
    # windows); below min_duration (dropped by the caller, cli/speaker.py:230, and absent from the reference's output)
    segs_ms = [(500, 1400), (2000, 3500), (4000, 5510), (6000, 9000), (10000, 12340), (13000, 13200), (14000, 31070)]
    out["segments_s"] = np.array([(b / 1000.0, e / 1000.0) for b, e in segs_ms], dtype=np.float64)
    ids, wins = [], []
    for k, (b, e) in enumerate(segs_ms):
        seg_length = (e - b) // FRAME_SHIFT
        fbank = rng.standard_normal((seg_length - 2, 16)).astype(np.float32) * 3 + 7   # 16 columns keep the file small
        out[f"fbank_{k}"] = fbank
        if (e - b) / 1000.0 < 0.255:
            continue
        i, w = extract_emb.subsegment(fbank, "{:08d}-{:08d}".format(b, e), WINDOW_FS, PERIOD_FS, FRAME_SHIFT)
        ids += i
        wins += w
    out["subseg_ids"] = np.array(ids)
    out["subseg_windows"] = np.stack(wins)

    # ---- clustering: m = 2 (trivial branch), m = 120 / 3 speakers, m = 1100 / 5 speakers (the m >= 1000 pruning branch)
    real_eigh = scipy.linalg.eigh
    # Ties at the pruning boundary have no defined order in np.argsort, so each set is redrawn until the last kept and the
    # first dropped similarity of every row are apart by `gap`: 1e-5 for the small set; 2e-6 (some 30 fp32 ulps) for the
    # large one, whose 1100 rows of 1100 similarities lie too densely for more
    for tag, m, spk, gap in (("tiny", 2, 1, 0.0), ("small", 120, 3, 1e-5), ("large", 1100, 5, 2e-6)):
        for _ in range(200):
            emb = _embeddings(rng, m, spk, 32, 0.35)
            if m <= 2 or _boundary_gap(emb) > gap:
                break
        else:
            raise RuntimeError(f"no {tag} embedding set with a pruning-boundary gap above {gap}")
        seen = {}

        def recording_eigh(M, *a, **k):
            seen["lap"] = np.array(M, copy=True)
            w, v = real_eigh(M, *a, **k)
            seen["eig"] = np.array(w, copy=True)
            return w, v

        scipy.linalg.eigh = recording_eigh
        try:
            runs = [np.asarray(spectral.cluster(emb)) for _ in range(5)]
        finally:
            scipy.linalg.eigh = real_eigh
        assert all(_same_partition(runs[0], r) for r in runs[1:]), tag
        out[f"emb_{tag}"] = emb
        out[f"labels_{tag}"] = runs[0].astype(np.int64)
        if m > 2:
            out[f"lap_{tag}"] = seen["lap"]
            out[f"eig_{tag}"] = seen["eig"][:32]
            out[f"num_spks_{tag}"] = np.int64(len(set(runs[0].tolist())))
            assert out[f"num_spks_{tag}"] == spk, (tag, out[f"num_spks_{tag}"])

    # ---- merging: overlaps with and without a label change, a gap, a single trailing sub-segment
    seq = [(0.0, 1.5, 0), (0.75, 2.25, 0), (1.5, 3.0, 1), (2.25, 3.75, 1), (5.0, 5.9, 1), (6.0, 7.5, 2), (6.75, 8.25, 0),
           (7.5, 8.4, 0), (9.0, 9.3, 2)]
    out["merge_in"] = np.array(seq, dtype=np.float64)
    merged = make_rttm.merge_segments({"rec": seq})
    out["merge_out"] = np.array([(b, e, la) for _, b, e, la in merged], dtype=np.float64)

    np.savez_compressed(os.path.join(HERE, "diar.npz"), **out)
    print({k: (v.shape, v.dtype) for k, v in out.items()})


if __name__ == "__main__":
    main()
