#!/usr/bin/env python
"""Per-tile fixed cost of the 256-wide 16-bit conv-GEMM: the time a tile spends outside its k-loop (epilogue, tile switch).

Times ws_conv (CUDA events, operands rotated so that every launch misses L2, as tools/gemm_tile_sweep.py does) for a
bf16 1x1 conv over 51 200 positions (B=256, T=200) with N = 1024 output channels and K in {256, 512, 1024, 2048, 3072},
in clusters of two CTAs (use_tc=3), for two epilogues:
    bias + ReLU
    bias + ReLU + BN + SE column sums
Every launch runs 128 x 256 tiles; the persistent schedule covers the 200 x 4 cluster tiles in
rounds = ceil(800 / clusters) rounds, with the resident cluster count taken from ws_tc3_max_clusters(2).  A least-squares
fit of time per round = a + b * (K / 64) gives the fixed cost a per tile and the cost b per 64-wide k-block.

    python tools/gemm_epilogue_cost.py [--iters 40] [--json OUT]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B, T, N, CL = 256, 200, 1024, 2
KS = (256, 512, 1024, 2048, 3072)
VARIANTS = (("bias+relu", False), ("bias+relu+bn+colsum", True))


def device_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "nvidia-smi: no output"
    except (OSError, subprocess.TimeoutExpired) as ex:
        return f"nvidia-smi unavailable ({ex})"


def time_conv(L, lib, torch, cin, colsum, iters):
    dev = torch.device("cuda", 0)
    st = lib.cur_stream_ptr()
    npos = B * T
    per = npos * (cin + N) * 2
    nbuf = max(2, int(2 * 126e6 // per) + 1)   # > 2x the 50 MB L2 between two uses of one buffer
    g = torch.Generator(device=dev).manual_seed(cin)
    xs = [torch.randn(B, 1, T, cin, device=dev, generator=g).to(torch.bfloat16) for _ in range(nbuf)]
    outs = [torch.empty(B, 1, T, N, device=dev, dtype=torch.bfloat16) for _ in range(nbuf)]
    w = (torch.randn(N, cin, device=dev, generator=g) / cin ** 0.5).to(torch.bfloat16)
    bias = 0.1 * torch.randn(N, device=dev, generator=g)
    scale = 0.5 + torch.rand(N, device=dev, generator=g)
    shift = 0.1 * torch.randn(N, device=dev, generator=g)
    cs = torch.zeros(2 * ((npos + 63) // 64), N, device=dev)
    descs = []
    for x, o in zip(xs, outs):
        d = lib.ConvDesc()
        d.x, d.B, d.F, d.T, d.Cin, d.x_ld = x.data_ptr(), B, 1, T, cin, cin
        d.w, d.Cout, d.kf, d.kt = w.data_ptr(), N, 1, 1
        d.dil_f = d.dil_t = d.stride_f = d.stride_t = 1
        d.bias, d.act1, d.out, d.out_ld, d.dtype = bias.data_ptr(), 1, o.data_ptr(), N, 1
        d.use_tc = 3
        if colsum:
            d.scale, d.shift, d.colsum = scale.data_ptr(), shift.data_ptr(), cs.data_ptr()
        descs.append(d)
    for i in range(5):
        lib.check(L.ws_conv(C.byref(descs[i % nbuf]), st), "ws_conv")
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(iters):
        lib.check(L.ws_conv(C.byref(descs[i % nbuf]), st), "ws_conv")
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    del xs, outs
    torch.cuda.empty_cache()
    return ms


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--iters", type=int, default=40)
    ap.add_argument("--json", help="also write the rows and fits to this file")
    a = ap.parse_args()
    import torch
    sys.path.insert(0, ROOT)
    from wespeaker_b200 import lib
    if not torch.cuda.is_available():
        raise SystemExit("gemm_epilogue_cost: needs a CUDA device")
    L = lib.load()
    fn = L.ws_tc3_max_clusters
    fn.restype, fn.argtypes = C.c_int, [C.c_int]
    torch.cuda.init()
    ncl = fn(CL)
    if ncl <= 0:
        raise SystemExit("gemm_epilogue_cost: ws_tc3_max_clusters failed")
    cluster_tiles = (B * T + 128 * CL - 1) // (128 * CL) * (N // 256)
    rounds = (cluster_tiles + ncl - 1) // ncl
    print(f"device: {device_info()}")
    print(f"bf16 1x1 conv, {B * T} positions, N={N}, 128x256 tiles, CL={CL}: {cluster_tiles} cluster tiles over "
          f"{ncl} resident clusters = {rounds} rounds; {a.iters} launches each, operands rotated past L2\n")
    print("| epilogue | K | ms | TFLOP/s | us per round |\n|---|---|---|---|---|")
    rows, fits = [], []
    for name, colsum in VARIANTS:
        us = []
        for k in KS:
            ms = time_conv(L, lib, torch, k, colsum, a.iters)
            per_round = 1e3 * ms / rounds
            us.append(per_round)
            tf = 2.0 * B * T * k * N / (ms * 1e-3) / 1e12
            rows.append(dict(epilogue=name, K=k, ms=ms, tflops=tf, us_per_round=per_round))
            print(f"| {name} | {k} | {ms:.4f} | {tf:.0f} | {per_round:.2f} |", flush=True)
        kb = np.array(KS, dtype=np.float64) / 64
        b, a0 = np.polyfit(kb, np.array(us), 1)
        share = a0 / (a0 + 16 * b)
        fits.append(dict(epilogue=name, a_us=a0, b_us=b, a_share_k1024=share))
    print()
    for f in fits:
        print(f"{f['epilogue']}: a = {f['a_us']:.2f} us per tile, b = {f['b_us']:.3f} us per 64-wide k-block, "
              f"a's share at K=1024: {100 * f['a_share_k1024']:.1f} %")
    print(f"\ndevice after: {device_info()}")
    if a.json:
        with open(a.json, "w") as f:
            json.dump(dict(device=device_info(), clusters=ncl, rounds=rounds, rows=rows, fits=fits), f, indent=1)


if __name__ == "__main__":
    main()
