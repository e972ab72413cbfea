"""CUDA-event timing of conv shapes through ws_conv (no profiler), with the default N tile and with WS_TC2_MAX_BN=128."""
import ctypes as C, os, sys, itertools
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from wespeaker_b200 import lib

def time_conv(B, T, cin, cout, k, dil, use_tc, code=1, iters=10, res=False):
    tdt = {0: torch.float32, 1: torch.bfloat16, 2: torch.float16}[code]
    dev = torch.device("cuda")
    per = B * T * (cin + cout) * (2 if code else 4)
    nbuf = max(2, int(2 * 126e6 // per) + 1)
    nbuf = min(nbuf, 6)
    xs = [torch.randn(B, 1, T, cin, device=dev).to(tdt) for _ in range(nbuf)]
    outs = [torch.empty(B, 1, T, cout, device=dev, dtype=tdt) for _ in range(nbuf)]
    rs = torch.randn(B, 1, T, cout, device=dev).to(tdt) if res else None
    w = (torch.randn(cout, k * cin, device=dev) / (k * cin) ** 0.5).to(tdt)
    bias = torch.zeros(cout, device=dev)
    L = lib.load(); descs = []
    for x, o in zip(xs, outs):
        d = lib.ConvDesc()
        d.x, d.B, d.F, d.T, d.Cin, d.x_ld = x.data_ptr(), B, 1, T, cin, cin
        d.w, d.Cout, d.kf, d.kt = w.data_ptr(), cout, 1, k
        d.dil_f = d.stride_f = d.stride_t = 1; d.dil_t = dil; d.pad_t = dil * (k - 1) // 2
        d.bias, d.act1, d.out, d.out_ld, d.dtype, d.use_tc = bias.data_ptr(), 1, o.data_ptr(), cout, code, use_tc
        if res: d.res, d.res_ld = rs.data_ptr(), cout
        descs.append(d)
    st = lib.cur_stream_ptr()
    for i in range(3): lib.check(L.ws_conv(C.byref(descs[i % nbuf]), st), "ws_conv")
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(iters): lib.check(L.ws_conv(C.byref(descs[i % nbuf]), st), "ws_conv")
    e1.record(); torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    return ms, 2.0 * B * T * k * cin * cout / (ms * 1e-3) / 1e12

shapes = {"cc1024": (256, 200, 1024, 1024, 1, 1), "big": (256, 200, 3072, 1536, 1, 1), "res2": (256, 200, 128, 128, 3, 2),
          "layer1": (256, 200, 80, 1024, 5, 1), "astp2": (256, 200, 128, 1536, 1, 1)}
if __name__ == "__main__":
    which = sys.argv[1].split(",") if len(sys.argv) > 1 else list(shapes)
    for name in which:
        B, T, ci, co, k, d = shapes[name]
        for tcv in (2, 3):
            for knobs in ({}, {"WS_TC2_MAX_BN": "128"}):
                os.environ.pop("WS_TC2_MAX_BN", None)
                os.environ.update(knobs)
                ms, tf = time_conv(B, T, ci, co, k, d, tcv, res=(name == "res2"))
                print(f"{name:8s} tc{tcv} {str(knobs):34s} {ms*1e3:8.1f} us {tf:7.1f} TF/s", flush=True)
