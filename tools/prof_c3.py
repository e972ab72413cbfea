"""Time the halo-resident 3x3 conv (ws_conv, use_tc=4) at several shapes in ONE process.
usage: prof_c3.py "B F T C" ... [--tc 4,3]"""
import os, sys, ctypes as C
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from wespeaker_b200 import lib
args = sys.argv[1:]
tcs = [4]
shapes = []
i = 0
while i < len(args):
    if args[i] == "--tc": tcs = [int(x) for x in args[i + 1].split(",")]; i += 2
    else: shapes.append(tuple(int(x) for x in args[i].split())); i += 1
if not shapes:
    shapes = [(64, 80, 200, 32), (64, 40, 100, 64), (64, 20, 50, 128)]
dev = torch.device("cuda:0")
tdt = torch.float16
L = lib.load()
st = lib.cur_stream_ptr()


def run(B, F, T, Cc, use_tc, with_res, n=10):
    nb = 3
    xs = [torch.randn(B, F, T, Cc, device=dev).to(tdt) for _ in range(nb)]
    rs = [torch.randn(B, F, T, Cc, device=dev).to(tdt) for _ in range(nb)]
    os_ = [torch.empty(B, F, T, Cc, device=dev, dtype=tdt) for _ in range(nb)]
    w = (torch.randn(Cc, 9 * Cc, device=dev) / (9 * Cc) ** 0.5).to(tdt)
    bias = torch.zeros(Cc, device=dev)
    ds = []
    for x, r, o in zip(xs, rs, os_):
        d = lib.ConvDesc()
        d.x, d.B, d.F, d.T, d.Cin, d.x_ld = x.data_ptr(), B, F, T, Cc, Cc
        d.w, d.Cout, d.kf, d.kt = w.data_ptr(), Cc, 3, 3
        d.dil_f = d.dil_t = d.stride_f = d.stride_t = d.pad_f = d.pad_t = 1
        d.bias, d.act1, d.act2, d.out, d.out_ld, d.dtype, d.use_tc = bias.data_ptr(), 0 if with_res else 1, 1 if with_res else 0, o.data_ptr(), Cc, 2, use_tc
        if with_res:
            d.res, d.res_ld = r.data_ptr(), Cc
        ds.append(d)
    for i in range(3):
        lib.check(L.ws_conv(C.byref(ds[i % nb]), st), "ws_conv")
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(n):
        lib.check(L.ws_conv(C.byref(ds[i % nb]), st), "ws_conv")
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


for (B, F, T, Cc) in shapes:
    fl = 2.0 * B * F * T * 9 * Cc * Cc
    for tc in tcs:
        for with_res in (0, 1):
            ms = run(B, F, T, Cc, tc, with_res)
            by = B * F * T * Cc * 2 * (3 if with_res else 2)
            print(f"conv3x3 B{B} F{F} T{T} C{Cc} use_tc={tc} res={with_res}: {ms*1e3:.1f} us, {fl/ms/1e9:.0f} TFLOP/s, "
                  f"{by/ms/1e6:.0f} GB/s algorithmic", flush=True)
