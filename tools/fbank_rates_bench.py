"""Time the fbank kernel (csrc/ws_fbank.cu, through ws_fbank_at, no CMN) at the SRE recipes' 8 kHz configurations and at
16 kHz, with CUDA events over many launches; the bytes it must move (PCM in + features out) over that time as a share of the
H100 SXM data-sheet 3.35 TB/s; and ResNet34 fp16 utterances per second through extract_from_wav (fbank + CMN + forward) at
8 kHz / 64 bins against 16 kHz / 80 bins.  The card's name and power limit are read in the same run.

Workloads: 256 utterances of 2 s (a batched extraction) and 16 of 60 s (long recordings), float32 PCM in int16 range.
Usage: python tools/fbank_rates_bench.py [--reps R] [--out file.json]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from wespeaker_b200 import frontend, lib  # noqa: E402
from wespeaker_b200.models import from_synthetic  # noqa: E402

PEAK_BPS = 3.35e12
CONFIGS = [(8000, 40), (8000, 64), (8000, 80), (16000, 64), (16000, 80)]
SHAPES = [(256, 2.0), (16, 60.0)]


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"


def time_ms(fn, reps):
    for _ in range(3):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("fbank_rates_bench needs a CUDA device")
    L = lib.load()
    st = lib.cur_stream_ptr(0)
    res = {"card": card(), "fbank": [], "extract": []}
    g = torch.Generator(device="cuda").manual_seed(0)
    for B, secs in SHAPES:
        for sr, nb in CONFIGS:
            N = int(sr * secs)
            wav = (torch.randn((B, N), device="cuda", generator=g) * 3000.0).contiguous()
            T = frontend.num_frames(N, sr)
            feats = torch.empty((B, T, nb), device="cuda")

            def run():
                lib.check(L.ws_fbank_at(wav.data_ptr(), 0, N, N, B, b"hamming", sr, nb, 0, feats.data_ptr(), st), "ws_fbank_at")
            ms = time_ms(run, args.reps)
            nbytes = B * N * 4 + B * T * nb * 4
            row = {"B": B, "seconds": secs, "sample_rate": sr, "bins": nb, "kernel_ms": round(ms, 4),
                   "GBps": round(nbytes / ms / 1e6, 1), "share_of_3.35TBps": round(nbytes / ms / 1e-3 / PEAK_BPS, 3)}
            res["fbank"].append(row)
            print(json.dumps(row), flush=True)
    for sr, nb in ((8000, 64), (16000, 80)):
        m = from_synthetic("ResNet34", 0, precision="fp16", feat_dim=nb)
        B = 256
        wav = (torch.randn((B, 2 * sr), device="cuda", generator=g) * 3000.0).contiguous()
        ms = time_ms(lambda: m.extract_from_wav(wav, sample_rate=sr), max(5, args.reps // 5))
        row = {"model": "ResNet34", "precision": "fp16", "B": B, "seconds": 2.0, "sample_rate": sr, "bins": nb,
               "ms_per_batch": round(ms, 3), "utt_per_s": round(B / ms * 1e3, 1)}
        res["extract"].append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps({"card": res["card"]}))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
