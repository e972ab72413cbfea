"""SimAM_ResNet34_ASP throughput on one GPU (fp16 and bf16, B = 64 x 200 frames, from device features and from wav), the
per-op breakdown of the plan (ws_engine_profile_ops: CUDA events between ops, no graph) and the SimAM kernels' share of it.

SimAM bytes are counted from the block shapes: the statistics op reads y once, the apply op reads y and the shortcut and writes
the output (the fp32 partials / statistics are negligible).  Achieved bandwidth = those bytes over the SimAM ops' summed
event times, against the H100 SXM data sheet's 3.35 TB/s.  The device name and power limit are read in the same run.

    python tools/simam_bench.py [--steps 20] [--warmup 5] [--batch 64] [--frames 200]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from wespeaker_b200 import lib, synthetic as syn  # noqa: E402
from wespeaker_b200.models import from_synthetic  # noqa: E402

NAME = "SimAM_ResNet34_ASP"
HBM_PEAK = 3.35e12


def device_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        name, power = [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")]
    except Exception:
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def simam_bytes(B, T, es, in_planes=64, feat_dim=80):
    """bytes the SimAM ops of one forward move: per block, stats read y, apply reads y + shortcut and writes the output"""
    total, F, Tl = 0, feat_dim, T
    for li, nb in enumerate(syn.SIMAM_NAMES[NAME]):
        if li > 0:
            F, Tl = (F - 1) // 2 + 1, (Tl - 1) // 2 + 1
        total += nb * 4 * B * F * Tl * (in_planes << li) * es
    return total


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--frames", type=int, default=200)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("simam_bench needs a CUDA device")
    B, T = a.batch, a.frames
    gpu, power = device_info()
    print(f"device: {gpu}, power limit {power}")
    L = lib.load()
    feats = torch.from_numpy(syn.make_feats(B, T, 80, seed=1)).cuda()
    wavs = torch.from_numpy(syn.make_wavs(B, (T - 1) * 160 + 400, seed=2)).cuda()
    for prec in ("fp16", "bf16"):
        m = from_synthetic(NAME, 0, precision=prec).to("cuda:0")
        ms_feat = timed(lambda: m.embed(feats), a.steps, a.warmup)
        ms_wav = timed(lambda: m.extract_from_wav(wavs), a.steps, a.warmup)
        buf = (C.c_float * 4096)()
        n = L.ws_engine_profile_ops(m._engine, B, T, 10, buf, 4096)
        assert n > 0, L.ws_last_error()
        t = np.array(buf[:n])
        fl = C.c_double(0.0)
        names, flops = [], 0.0
        for i in range(n):
            nm = L.ws_engine_plan_op_name(m._engine, B, T, i, C.byref(fl))
            names.append(nm.decode() if nm else "?")
            flops += fl.value
        by_kind = {}
        for nm, ms in zip(names, t):
            k = nm.split(" ")[0]
            by_kind[k] = by_kind.get(k, 0.0) + float(ms)
        sim_ms = by_kind.get("simam_stats", 0.0) + by_kind.get("simam_apply", 0.0)
        nbytes = simam_bytes(B, T, 2)
        res = dict(model=NAME, precision=prec, batch=B, frames=T, device=gpu, power_limit=power,
                   ms_per_step_feats=round(ms_feat, 3), utt_per_s_feats=round(B / ms_feat * 1e3, 1),
                   ms_per_step_wav=round(ms_wav, 3), utt_per_s_wav=round(B / ms_wav * 1e3, 1),
                   op_sum_ms=round(float(t.sum()), 3), conv_gflop_per_utt=round(flops / B / 1e9, 2),
                   simam_stats_ms=round(by_kind.get("simam_stats", 0.0), 3), simam_apply_ms=round(by_kind.get("simam_apply", 0.0), 3),
                   simam_share_of_op_sum=round(sim_ms / float(t.sum()), 3), simam_gb=round(nbytes / 1e9, 3),
                   simam_tb_per_s=round(nbytes / (sim_ms * 1e-3) / 1e12, 3),
                   simam_frac_of_hbm_peak=round(nbytes / (sim_ms * 1e-3) / HBM_PEAK, 3),
                   op_ms_by_kind={k: round(v, 3) for k, v in sorted(by_kind.items(), key=lambda kv: -kv[1])})
        print(json.dumps(res))
        del m
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
