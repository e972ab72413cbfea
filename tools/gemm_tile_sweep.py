#!/usr/bin/env python
"""Rate of the persistent conv-GEMM against its L2 -> SM operand traffic, on the headline workload's two dense 1x1 shapes.

Times ws_conv (CUDA events, operands rotated so that every launch misses L2, as bench.time_dominant_kernel does) for
ECAPA-TDNN-1024 bf16 at B=256, T=200 (51 200 positions):
    1024 -> 1024, bias + ReLU              (se_res2block.0)
    1024 -> 1024, bias + ReLU + BN + SE column sums  (se_res2block.2)
    3072 -> 1536, bias + ReLU              (conv)
under every tile setting the code can select: cluster size CL = 1 (use_tc=2), 2 and 4 (use_tc=3, WS_TC3_CL) and N-tile
caps WS_TC2_MAX_BN = 64, 128, 256, each setting in a subprocess of its own.

Per run it prints ms per launch, TFLOP/s, and the operand bytes each launch pulls from L2 computed from shapes:
tiles x (128 + bn / CL) x K x 2 B (each CTA loads its 128-position A tile and 1/CL of the bn-row weight tile, which TMA
multicasts to the cluster).  If the rate follows bytes per FLOP, TFLOP/s x bytes/FLOP (the implied TB/s) stays flat.

    python tools/gemm_tile_sweep.py [--iters 30] [--bn 64,128,256] [--json OUT]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B, T = 256, 200
SHAPES = [("1024->1024 relu", 1024, 1024, False), ("1024->1024 relu+bn+colsum", 1024, 1024, True),
          ("3072->1536 relu", 3072, 1536, False)]


def device_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30)
        return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "nvidia-smi: no output"
    except (OSError, subprocess.TimeoutExpired) as ex:
        return f"nvidia-smi unavailable ({ex})"


def child(cl, iters):
    import ctypes as C
    import torch
    sys.path.insert(0, ROOT)
    from wespeaker_b200 import lib
    L = lib.load()
    dev = torch.device("cuda", 0)
    st = lib.cur_stream_ptr()
    npos = B * T
    res = []
    for name, cin, cout, colsum in SHAPES:
        per = npos * (cin + cout) * 2
        nbuf = max(2, int(2 * 126e6 // per) + 1)
        g = torch.Generator(device=dev).manual_seed(cin + cout)
        xs = [torch.randn(B, 1, T, cin, device=dev, generator=g).to(torch.bfloat16) for _ in range(nbuf)]
        outs = [torch.empty(B, 1, T, cout, device=dev, dtype=torch.bfloat16) for _ in range(nbuf)]
        w = (torch.randn(cout, cin, device=dev, generator=g) / cin ** 0.5).to(torch.bfloat16)
        bias = 0.1 * torch.randn(cout, device=dev, generator=g)
        scale = 0.5 + torch.rand(cout, device=dev, generator=g)
        shift = 0.1 * torch.randn(cout, device=dev, generator=g)
        cs = torch.zeros(2 * ((npos + 63) // 64), cout, device=dev)
        descs = []
        for x, o in zip(xs, outs):
            d = lib.ConvDesc()
            d.x, d.B, d.F, d.T, d.Cin, d.x_ld = x.data_ptr(), B, 1, T, cin, cin
            d.w, d.Cout, d.kf, d.kt = w.data_ptr(), cout, 1, 1
            d.dil_f = d.dil_t = d.stride_f = d.stride_t = 1
            d.bias, d.act1, d.out, d.out_ld, d.dtype = bias.data_ptr(), 1, o.data_ptr(), cout, 1
            d.use_tc = 2 if cl == 1 else 3
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
        res.append(dict(shape=name, K=cin, N=cout, ms=e0.elapsed_time(e1) / iters))
        del xs, outs
        torch.cuda.empty_cache()
    print(json.dumps(res))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--bn", default="64,128,256", help="WS_TC2_MAX_BN values to sweep")
    ap.add_argument("--json", help="also write the rows to this file")
    ap.add_argument("--child-cl", type=int, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.child_cl:
        child(a.child_cl, a.iters)
        return
    print(f"device: {device_info()}")
    print(f"ECAPA-TDNN-1024 bf16 1x1 convs over {B * T} positions, {a.iters} launches each, operands rotated past L2\n")
    print("| shape | CL | bn cap | ms | TFLOP/s | L2->SM MB | mB/FLOP | implied TB/s |\n|---|---|---|---|---|---|---|---|")
    rows = []
    for cl in (1, 2, 4):
        for bn in (int(v) for v in a.bn.split(",")):
            env = dict(os.environ, WS_TC2_MAX_BN=str(bn))
            env.pop("WS_TC3_CL", None)
            if cl == 4:
                env["WS_TC3_CL"] = "4"
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child-cl", str(cl), "--iters", str(a.iters)],
                               env=env, capture_output=True, text=True, cwd=ROOT)
            if r.returncode != 0:
                print(f"| CL={cl} bn<={bn} failed: {r.stderr.strip().splitlines()[-1:]} |")
                continue
            for x in json.loads(r.stdout.strip().splitlines()[-1]):
                # every swept shape has Cout % 256 == 0 and takes the widest tile the cap allows
                ebn = min(bn, 256)
                flops = 2.0 * B * T * x["K"] * x["N"]
                tiles = (B * T + 127) // 128 * (x["N"] // ebn)
                nbytes = tiles * (128 + ebn / cl) * x["K"] * 2
                x.update(cl=cl, bn=ebn, tflops=flops / (x["ms"] * 1e-3) / 1e12, l2_bytes=nbytes,
                         mb_per_flop=1e3 * nbytes / flops, tbps=nbytes / (x["ms"] * 1e-3) / 1e12)
                rows.append(x)
                print(f"| {x['shape']} | {cl} | {ebn} | {x['ms']:.3f} | {x['tflops']:.0f} | {nbytes / 1e6:.0f} | "
                      f"{x['mb_per_flop']:.1f} | {x['tbps']:.2f} |", flush=True)
    print(f"\ndevice after: {device_info()}")
    if a.json:
        with open(a.json, "w") as f:
            json.dump(dict(device=device_info(), rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
