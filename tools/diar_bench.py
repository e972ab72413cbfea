"""Where the time of one recording's diarization goes on one GPU: seeded synthetic recordings of 5, 20 and 60 minutes (60 %
speech, segments of 1-15 s), ResNet34 fp16 and ECAPA-TDNN-512 bf16.  Every (B, 150) plan the run uses is warmed first; each
stage is then timed as its Python entry point runs it (the upload of its index tables included) with CUDA events closed by a
synchronise (median of --repeats): ragged fbank, ws_diar_windows, the
engine forward over all windows, ws_diar_laplacian (unit rows included), torch.linalg.eigh, k-means.

For the two bandwidth kernels the bytes are counted from shapes - windows: every window's source rows read once plus
W * 150 * 80 * 4 written; Laplacian stage: the fp32 cosine tiles written and read, m * m adjacency bytes written and read
twice, m * m fp64 written and read once - and given over the stage's time as a share of the H100 SXM data sheet's 3.35 TB/s
of HBM bandwidth ("hbm_share": the Laplacian stage also contains the fp64 GEMM, so its figure is a lower bound for the
kernels alone).  The card's name and power limit are read in the same run (a query; nothing is set).

    python tools/diar_bench.py [--out DIR] [--minutes 5 20 60] [--repeats 3]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from wespeaker_b200 import diar  # noqa: E402
from wespeaker_b200.models import from_synthetic  # noqa: E402

HBM_PEAK = 3.35e12
BATCH = 256


def device_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        name, power = [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")]
    except Exception:
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def recording(minutes, seed):
    """int16-range noise and speech segments [(begin_s, end_s)] covering 60 % of it in pieces of 1-15 s."""
    rng = np.random.default_rng(seed)
    total = minutes * 60.0
    segs, t = [], 0.0
    while True:
        dur = float(rng.uniform(1.0, 15.0))
        gap = dur * (0.4 / 0.6) * float(rng.uniform(0.5, 1.5))
        if t + gap + dur > total:
            break
        segs.append((round(t + gap, 3), round(t + gap + dur, 3)))
        t += gap + dur
    pcm = (rng.standard_normal(int(total * 16000)) * 2000).astype(np.float32)
    return torch.from_numpy(pcm).cuda(), segs


def timed(fn, repeats):
    ms, out = [], None
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms)), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="diar_bench_out")
    ap.add_argument("--minutes", type=int, nargs="+", default=[5, 20, 60])
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("diar_bench needs a CUDA device")
    os.makedirs(a.out, exist_ok=True)
    gpu, power = device_info()
    print(f"device: {gpu}, power limit {power}")
    results = []
    for name, prec in (("ResNet34", "fp16"), ("ECAPA_TDNN_c512", "bf16")):
        model = from_synthetic(name, 0, precision=prec).to("cuda:0")
        for minutes in a.minutes:
            pcm, segs = recording(minutes, seed=minutes)
            t = diar.subsegment_table(segs, num_samples=pcm.numel())
            W = len(t.ids)
            feats = diar.fbank_ragged(pcm, t.row_offset, t.row_frames, t.max_frames)
            wins = diar.windows(feats, t.win_row0, t.win_len)
            for b in {min(BATCH, W), W % BATCH} - {0}:                      # warm every (B, 150) plan
                model.embed(wins[:b])
            embed = lambda: torch.cat([model.embed(wins[i:i + BATCH]) for i in range(0, W, BATCH)])   # noqa: E731
            embs = embed()
            lap = diar.laplacian(embs)
            vals, vecs = torch.linalg.eigh(lap)
            k = max(2, diar.num_speakers(vals[:21].cpu().numpy()))          # noise has no speakers: time k-means at k >= 2
            ms = {}
            ms["fbank"], _ = timed(lambda: diar.fbank_ragged(pcm, t.row_offset, t.row_frames, t.max_frames), a.repeats)
            ms["windows"], _ = timed(lambda: diar.windows(feats, t.win_row0, t.win_len), a.repeats)
            ms["forward"], _ = timed(embed, a.repeats)
            ms["laplacian"], _ = timed(lambda: diar.laplacian(embs), a.repeats)
            ms["eigh"], _ = timed(lambda: torch.linalg.eigh(lap), a.repeats)
            ms["kmeans"], _ = timed(lambda: diar.kmeans(vecs[:, :k].contiguous(), k), a.repeats)
            total = sum(ms.values())
            win_bytes = (int(t.win_len.sum()) + W * 150) * 80 * 4
            rows = max(1, min(W, (1 << 28) // (4 * W)))
            lap_bytes = W * W * (4 * 2 + 1 * 3 + 8 * 3) + W * embs.shape[1] * 8 * (1 + -(-W // rows))
            res = dict(model=name, precision=prec, minutes=minutes, device=gpu, power_limit=power, segments=len(segs),
                       fbank_rows=len(t.row_offset), max_frames=t.max_frames, windows=W, kmeans_k=k,
                       ms={k_: round(v, 3) for k_, v in ms.items()}, total_ms=round(total, 2),
                       windows_per_s=round(W / total * 1e3, 1), audio_s_per_wall_s=round(minutes * 60.0 / total * 1e3, 1),
                       windows_gb=round(win_bytes / 1e9, 4), windows_hbm_share=round(win_bytes / (ms["windows"] * 1e-3) / HBM_PEAK, 4),
                       laplacian_gb=round(lap_bytes / 1e9, 4),
                       laplacian_hbm_share=round(lap_bytes / (ms["laplacian"] * 1e-3) / HBM_PEAK, 4))
            print(json.dumps(res), flush=True)
            results.append(res)
            del feats, wins, embs, lap, vals, vecs
            torch.cuda.empty_cache()
        del model
    with open(os.path.join(a.out, "diar_bench.json"), "w") as f:
        json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
