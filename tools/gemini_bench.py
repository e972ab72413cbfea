"""Gemini_DF_ResNet114 throughput on one GPU (fp16 and bf16, B = 64 x 200 frames, from device features and from wav), the
per-op breakdown of the plan (ws_engine_profile_ops: CUDA events between ops, no graph), the depthwise 3x3 ops' share of it,
and the standalone depthwise kernel on the stage-3 shape (B = 64, F = 10, T = 100, C = 512, fp16).

Depthwise bytes are counted from the block shapes: each op reads its 4x-expanded input once and writes its output once (the
fp32 weights are negligible).  Achieved bandwidth = those bytes over the ops' summed event times, against the H100 SXM data
sheet's 3.35 TB/s.  The device name and power limit are read in the same run.

    python tools/gemini_bench.py [--steps 20] [--warmup 5] [--batch 64] [--frames 200]
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

NAME = "Gemini_DF_ResNet114"
HBM_PEAK = 3.35e12
STRIDE_T = (1, 2, 1, 1)


def device_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        name, power = [s.strip() for s in r.stdout.strip().splitlines()[0].split(",")]
    except Exception:
        name, power = torch.cuda.get_device_name(0), "unknown"
    return name, power


def dwconv_bytes(B, T, es, feat_dim=80):
    """bytes the depthwise ops of one forward move: per block, the 4 dim-channel map read once and written once"""
    total, F, Tl = 0, feat_dim, T
    for i, nb in enumerate(syn.GEMINI_NAMES[NAME]):
        F, Tl = (F - 1) // 2 + 1, (Tl - 1) // STRIDE_T[i] + 1
        total += nb * 2 * B * F * Tl * 4 * syn.GEMINI_DIMS[i + 1] * es
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


def standalone_kernel(L, steps):
    """ws_dwconv on the stage-3 shape, fp16, timed with CUDA events over `steps` launches"""
    B, F, T, Cc = 64, 10, 100, 512
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(B, F, T, Cc, device="cuda", generator=g).half()
    out = torch.empty_like(x)
    w = torch.randn(Cc, 3, 3, device="cuda", generator=g) / 3
    sh = torch.randn(Cc, device="cuda", generator=g)
    d = lib.DwConvDesc()
    d.x, d.x_ld, d.B, d.F, d.T, d.C = x.data_ptr(), Cc, B, F, T, Cc
    d.lens, d.w, d.shift, d.out, d.out_ld, d.out_lo, d.dtype = None, w.data_ptr(), sh.data_ptr(), out.data_ptr(), Cc, None, 2
    st = torch.cuda.current_stream().cuda_stream

    def run():
        lib.check(L.ws_dwconv(C.byref(d), C.c_void_p(st)), "ws_dwconv")
    ms = timed(run, steps, 10)
    nbytes = 2 * x.numel() * 2
    return dict(shape=f"B{B} F{F} T{T} C{Cc} fp16", us=round(ms * 1e3, 2), tb_per_s=round(nbytes / (ms * 1e-3) / 1e12, 3),
                frac_of_hbm_peak=round(nbytes / (ms * 1e-3) / HBM_PEAK, 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--frames", type=int, default=200)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gemini_bench needs a CUDA device")
    B, T = a.batch, a.frames
    gpu, power = device_info()
    print(f"device: {gpu}, power limit {power}")
    L = lib.load()
    print(json.dumps(dict(standalone_dwconv3x3=standalone_kernel(L, 200), device=gpu, power_limit=power)))
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
        names = []
        for i in range(n):
            nm = L.ws_engine_plan_op_name(m._engine, B, T, i, C.byref(fl))
            names.append(nm.decode() if nm else "?")
        by_kind = {}
        for nm, ms in zip(names, t):
            k = nm.split(" ")[0]
            by_kind[k] = by_kind.get(k, 0.0) + float(ms)
        dw_ms = by_kind.get("dwconv3x3", 0.0)
        nbytes = dwconv_bytes(B, T, 2)
        res = dict(model=NAME, precision=prec, batch=B, frames=T, device=gpu, power_limit=power,
                   ms_per_step_feats=round(ms_feat, 3), utt_per_s_feats=round(B / ms_feat * 1e3, 1),
                   ms_per_step_wav=round(ms_wav, 3), utt_per_s_wav=round(B / ms_wav * 1e3, 1),
                   op_sum_ms=round(float(t.sum()), 3), dwconv_ms=round(dw_ms, 3),
                   dwconv_share_of_op_sum=round(dw_ms / float(t.sum()), 3), dwconv_gb=round(nbytes / 1e9, 3),
                   dwconv_tb_per_s=round(nbytes / (dw_ms * 1e-3) / 1e12, 3),
                   dwconv_frac_of_hbm_peak=round(nbytes / (dw_ms * 1e-3) / HBM_PEAK, 3),
                   op_ms_by_kind={k: round(v, 3) for k, v in sorted(by_kind.items(), key=lambda kv: -kv[1])})
        print(json.dumps(res))
        del m
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
