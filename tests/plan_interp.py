"""Host re-evaluation of a launch plan written by ws_engine_plan_trace (plan-check engine: no device, nothing computed by
the library).  TEST INFRASTRUCTURE: it checks the plan BUILDER's arithmetic - BN folding, channel padding, torch.cat /
torch.split as channel slices, shortcut convs merged as K ranges, strided convs as parity planes, tap offsets, residuals,
activations - against the oracle on the CPU; the CUDA kernels that execute the same plan are checked on the GPU.

Memory model: every placeholder allocation becomes a flat float64 array indexed in ELEMENTS (address offset / element size of
the tensor's dtype in the plan); values are never rounded, so a bf16 plan and an fp32 plan both reproduce the oracle to
floating-point accuracy.  The fused kernels (Res2 chain, ASTP tail, CAM++ dense block, SE gate) are re-evaluated from their
documented contracts (ws_host.h).  Length-masked plans are modelled too: rows behind an utterance's end are conv padding and
every statistic runs over the utterance's own frames."""
import json
import struct

import numpy as np


def load_trace(path):
    with open(path, "rb") as f:
        assert f.read(6) == b"WSPT1\n"
        (n,) = struct.unpack("<Q", f.read(8))
        meta = json.loads(f.read(n).decode())
        blob = np.frombuffer(f.read(), dtype="<f4")
    return meta, blob


class Memory:
    def __init__(self, meta, blob):
        self.allocs = sorted((a, n) for a, n in meta["allocs"])
        self.starts = np.array([a for a, _ in self.allocs], dtype=np.uint64)
        self.bufs = {}      # base address -> (float64 array, element size)
        self.writes = []    # (address, element size, shape, element strides) of every region an op's contract writes
        self.reads = []     # (address, element size, shape, element strides) of every region an op's contract reads
        self.blobs = {a: blob[o:o + n].astype(np.float64) for a, o, n in meta["blobs"]}

    def _find(self, addr):
        i = int(np.searchsorted(self.starts, np.uint64(addr), side="right")) - 1
        assert i >= 0, addr
        base, nbytes = self.allocs[i]
        assert base <= addr < base + max(nbytes, 1), (addr, base, nbytes)
        return base, nbytes

    def array(self, addr, es):
        """(flat array, element offset) of the allocation holding `addr`, elements of `es` bytes."""
        base, nbytes = self._find(addr)
        if base in self.blobs:              # weights: fp32 source values, whatever the plan's storage dtype
            assert (addr - base) % es == 0
            return self.blobs[base], (addr - base) // es
        if base not in self.bufs:
            self.bufs[base] = (np.zeros(nbytes // es, dtype=np.float64), es)
        arr, es0 = self.bufs[base]
        assert es0 == es and (addr - base) % es == 0, (addr, es0, es)
        return arr, (addr - base) // es

    def vec(self, addr, n, es=4):
        """n elements at addr; es is the size the operand is stored in (weights in the activation dtype: 2 in 16-bit plans)"""
        if not addr:
            return None
        self.reads.append((addr, es, (n,), (1,)))
        arr, off = self.array(addr, es)
        return arr[off:off + n]

    def read(self, addr, es, shape, strides):
        """declare a region the contract reads without going through strided / view (in-place ops)"""
        self.reads.append((addr, es, tuple(shape), tuple(strides)))

    def strided(self, addr, es, shape, strides, write=False):
        if write:
            self.writes.append((addr, es, tuple(shape), tuple(strides), None, False))
        else:
            self.reads.append((addr, es, tuple(shape), tuple(strides)))
        return self.region(addr, es, shape, strides, write)

    def region(self, addr, es, shape, strides, writeable=True):
        """array over a region, recorded as neither read nor written"""
        arr, off = self.array(addr, es)
        need = off + sum((s - 1) * st for s, st in zip(shape, strides)) + 1
        assert need <= arr.size, (addr, shape, strides, arr.size)
        return np.lib.stride_tricks.as_strided(arr[off:], shape=shape, strides=[st * 8 for st in strides], writeable=writeable)

    def side(self, addr):
        """declare the rest of addr's allocation as an op's scratch / side output: it may change, its values are not checked
        here (the SE column sums and the split-K partials are checked through the ops that consume them)"""
        if addr:
            base, nbytes = self._find(addr)
            self.writes.append((addr, 4, ((base + nbytes - addr) // 4,), (1,), None, True))

    def view(self, v, es, write=False):
        """channels-last View {p,B,F,T,C,ld} -> array (B,F,T,C)."""
        B, F, T, C, ld = v["B"], v["F"], v["T"], v["C"], v["ld"]
        if write and v.get("plo"):     # 3xTF32: the op also writes the fp32 lo twin, same layout
            self.writes.append((v["plo"], 4, (B, F, T, C), (F * T * ld, T * ld, ld, 1), v["p"], False))
        return self.strided(v["p"], es, (B, F, T, C), (F * T * ld, T * ld, ld, 1), write)


ROUND = None   # None: exact re-evaluation; "bf16" / "fp16": emulate the plan's 16-bit storage (activations and conv weights
               # rounded where the kernels round them) to PREDICT the 16-bit paths' distance from the oracle


def _tf32_trunc(a):
    return (np.ascontiguousarray(a, dtype=np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def tf32x3_matmul(x, Wt):
    """The engine's 3xTF32 product x @ Wt as the tensor core sees it (ROUND = "tf32x3" or "tf32x3_trunc_lo"): operands are
    truncated to tf32; x_lo * W_hi + x_hi * W_lo + x_hi * W_hi with lo = the residual rounded to the nearest tf32 (the engine's
    ws_tf32_lo) or, for comparison, left to the hardware's truncation."""
    def split(a):
        a32 = np.ascontiguousarray(a, dtype=np.float32)
        hi = _tf32_trunc(a32)
        d = a32 - hi
        lo = ((d.view(np.uint32) + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32) if ROUND == "tf32x3" else _tf32_trunc(d)
        return hi.astype(np.float64), lo.astype(np.float64)
    xh, xl = split(x)
    wh, wl = split(Wt)
    return xl @ wh + xh @ wl + xh @ wh


def rnd(x, es):
    if ROUND in ("tf32x3", "tf32x3_trunc_lo"):
        return np.asarray(x, np.float32).astype(np.float64) if es == 4 else x   # fp32 storage
    if ROUND is None or es != 2:
        return x
    import torch
    dt = torch.bfloat16 if ROUND == "bf16" else torch.float16
    return torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).to(dt).to(torch.float32).numpy().astype(np.float64)


def act(x, code):
    if code == 0:
        return x
    if code == 1:
        return np.maximum(x, 0.0)
    if code == 2:
        return np.tanh(x)
    if code == 3:
        return 1.0 / (1.0 + np.exp(-x))
    if code == 4:
        return np.clip(x, 0.0, 20.0)
    if code == 5:
        return x / (1.0 + np.exp(-x))
    raise NotImplementedError(code)


def shifted(src, df, dt, F, T):
    """src (B,Fs,Ts,C) -> (B,F,T,C): out[b,f,t] = src[b,f+df,t+dt], zero outside the source extents."""
    B, Fs, Ts, C = src.shape
    out = np.zeros((B, F, T, C))
    f0, f1 = max(0, -df), min(F, Fs - df)
    t0, t1 = max(0, -dt), min(T, Ts - dt)
    if f1 > f0 and t1 > t0:
        out[:, f0:f1, t0:t1] = src[:, f0 + df:f1 + df, t0 + dt:t1 + dt]
    return out


def _act_gain(code):
    """how much the activation can amplify an error of its input (SiLU's slope reaches 1.0998)"""
    return {3: 0.25, 5: 1.1}.get(code, 1.0)


def run_conv(mem, tr):
    """Returns {output address: E}: the error scale of each output element, sum over the reduction of sqrt(K) * |x| |W| (+ |bias|),
    carried through the epilogue (the checker's bound is ulp(out) + c * u32 * E)."""
    es = tr["es"]
    B, F, T, Cout, K = tr["B"], tr["F"], tr["T"], tr["Cout"], tr["Ktot"]   # (colsum, the fused SE squeeze, is a side output)
    W = rnd(mem.vec(tr["W"], Cout * K, es).reshape(Cout, K), es)
    if getattr(mem, "tf32_cut", False):     # single-pass tf32 tensor cores: the operands as the tensor core cuts them
        W = _tf32_trunc(W).astype(np.float64)
    srcs = [mem.strided(s["p"], es, (s["B"], s["F"], s["T"], s["C"]), (s["sB"], s["sF"], s["sT"], 1)) for s in tr["src"]]
    acc = np.zeros((B, F, T, Cout))
    mag = np.zeros((B, F, T, Cout))
    for si, c0, dt, df, wk, nch in tr["taps"]:
        x = shifted(srcs[si][..., c0:c0 + nch], df, dt, F, T)
        if getattr(mem, "tf32_cut", False):
            x = _tf32_trunc(x).astype(np.float64)
        acc += tf32x3_matmul(x, W[:, wk:wk + nch].T) if ROUND in ("tf32x3", "tf32x3_trunc_lo") and es == 4 else x @ W[:, wk:wk + nch].T
        mag += np.abs(x) @ np.abs(W[:, wk:wk + nch].T)
    mag *= np.sqrt(K)
    if tr["bias"]:
        acc += mem.vec(tr["bias"], Cout)
        mag += np.abs(mem.vec(tr["bias"], Cout))
    if tr["rowbias"]:      # per-utterance bias row (ECAPA global-context attention)
        rb = mem.strided(tr["rowbias"], 4, (B, Cout), (tr["rowbias_ld"], 1))[:, None, None, :]
        acc += rb
        mag += np.abs(rb)
    acc = act(acc, tr["act1"])
    mag *= _act_gain(tr["act1"])
    if tr["scale"]:
        acc = acc * mem.vec(tr["scale"], Cout) + mem.vec(tr["shift"], Cout)
        mag = mag * np.abs(mem.vec(tr["scale"], Cout)) + np.abs(mem.vec(tr["shift"], Cout))
    if tr["gate"]:         # CAM context mask: gate[b][t / gate_seg][c]
        nseg, gl = tr["gate_nseg"], tr["gate_ld"]
        g = mem.strided(tr["gate"], 4, (B, nseg, Cout), (nseg * gl, gl, 1))
        acc = acc * g[:, np.arange(T) // tr["gate_seg"], :][:, None]
        mag = mag * np.abs(g[:, np.arange(T) // tr["gate_seg"], :][:, None])
    if tr["res"]:
        r = mem.view(dict(p=tr["res"], B=B, F=F, T=T, C=Cout, ld=tr["res_ld"]), es)
        acc = acc + r
        mag = mag + np.abs(r)
    pre = act(acc, tr["act2"])
    mag *= _act_gain(tr["act2"])
    acc = rnd(pre, es)
    mem.side(tr["colsum"])
    mem.view(dict(p=tr["out"], plo=tr.get("out_lo", 0), B=B, F=F, T=T, C=Cout, ld=tr["out_ld"]), es, write=True)[...] = acc
    errs = {tr["out"]: mag}
    if tr["out2"]:         # unfused Res2 chain: s_{i+1} = rnd(sp_i + x_{i+1}) from the epilogue's fp32 sp_i, not the stored one
        add2 = mem.view(dict(p=tr["add2"], B=B, F=F, T=T, C=Cout, ld=tr["add2_ld"]), es)
        mem.view(dict(p=tr["out2"], plo=tr.get("out2_lo", 0), B=B, F=F, T=T, C=Cout, ld=tr["out2_ld"]), es, write=True)[...] = rnd(pre + add2, es)
        errs[tr["out2"]] = mag + np.abs(add2)
    return errs


def run_conv3x3(mem, tr):
    es = tr["es"]
    x = mem.view(tr["x"], es)
    o = tr["out"]
    Cin, Cout, sf, st = tr["x"]["C"], o["C"], tr["sf"], tr["st"]
    W = rnd(mem.vec(tr["W"], Cout * 9 * Cin, es).reshape(Cout, 9, Cin), es)
    Fo, To = o["F"], o["T"]
    assert Fo == (x.shape[1] - 1) // sf + 1 and To == (x.shape[2] - 1) // st + 1
    acc = np.zeros((o["B"], Fo, To, Cout))
    mag = np.zeros((o["B"], Fo, To, Cout))
    for jf in range(3):
        for jt in range(3):
            full = shifted(x, jf - 1, jt - 1, x.shape[1], x.shape[2])[:, ::sf, ::st][:, :Fo, :To]   # full[b,f,t] = x[b,f+jf-1,t+jt-1]
            acc += full @ W[:, jf * 3 + jt].T
            mag += np.abs(full) @ np.abs(W[:, jf * 3 + jt].T)
    mag *= np.sqrt(9 * Cin)
    if tr["bias"]:
        acc += mem.vec(tr["bias"], Cout)
        mag += np.abs(mem.vec(tr["bias"], Cout))
    if tr["res"] is not None:
        acc = acc + mem.view(tr["res"], es)
        mag += np.abs(mem.view(tr["res"], es))
    acc = {0: acc, 1: np.maximum(acc, 0.0), 2: np.clip(acc, 0.0, 20.0)}[tr["relu"]]
    if tr["lens"]:      # length-masked batch: output rows behind an utterance's end are stored as zeros
        acc = np.where((np.arange(To)[None, :] < mem.vec(tr["lens"], o["B"])[:, None])[:, None, :, None], acc, 0.0)
    mem.view(o, es, write=True)[...] = rnd(acc, es)
    return {o["p"]: mag}


def run_stem(mem, tr, meta):
    o = tr["out"]
    B, Fd, T, C = o["B"], o["F"], o["T"], o["C"]
    feats = mem.vec(tr["feats"], B * T * Fd).reshape(B, T, Fd)
    valid = np.ones((B, T), bool)
    if tr["lens"]:      # frames behind an utterance's end are padding: read as zeros, written as zeros
        valid = np.arange(T)[None, :] < mem.vec(tr["lens"], B)[:, None]
        feats = np.where(valid[:, :, None], feats, 0.0)
    w9 = mem.vec(tr["w9"], C * 9).reshape(C, 9)
    x = feats.transpose(0, 2, 1)[..., None]                                # (B,F,T,1)
    acc = np.zeros((B, Fd, T, C))
    mag = np.zeros((B, Fd, T, C))
    for jf in range(3):
        for jt in range(3):
            acc += shifted(x, jf - 1, jt - 1, Fd, T) * w9[:, jf * 3 + jt]
            mag += np.abs(shifted(x, jf - 1, jt - 1, Fd, T) * w9[:, jf * 3 + jt])
    acc = np.where(valid[:, None, :, None], np.maximum(acc + mem.vec(tr["shift"], C), 0.0), 0.0)
    mem.view(o, tr["es"], write=True)[...] = rnd(acc, tr["es"])
    return {o["p"]: 3.0 * mag + np.abs(mem.vec(tr["shift"], C))}


def run_tstats(mem, tr):
    x = mem.view(tr["x"], tr["es"])
    B, F, T, C = x.shape
    xe = np.zeros(x.shape)          # error scale of each input element: the fused BN-ReLU's fp32 rounding
    if tr["pre_scale"]:
        xe = np.abs(x * mem.vec(tr["pre_scale"], C)) + np.abs(mem.vec(tr["pre_shift"], C))
        x = np.maximum(x * mem.vec(tr["pre_scale"], C) + mem.vec(tr["pre_shift"], C), 0.0)
    out_ld, so = tr["out_ld"], tr["std_off"]
    out = mem.strided(tr["out"], tr["out_es"], (B, out_ld), (out_ld, 1), write=True)
    lens = mem.vec(tr["lens"], B).astype(int) if tr["lens"] else np.full(B, T)   # statistics over each utterance's own frames
    err = np.zeros((B, out_ld))
    for b in range(B):
        xb = x[b, :, :lens[b]]
        n = lens[b]
        out[b, :C * F] = xb.mean(axis=1).T.reshape(C * F)                       # (F,C) -> index c*F + f
        eb = xe[b, :, :n]
        err[b, :C * F] = (n * np.abs(xb).mean(axis=1) + eb.mean(axis=1)).T.reshape(C * F)   # a sum of n terms: gamma_n
        if so >= 0:
            sd = np.sqrt(xb.var(axis=1, ddof=1) + tr["eps"])
            out[b, so:so + C * F] = sd.T.reshape(C * F)
            # var error <= n u (sum x^2) / (n - 1) whether it is summed in one pass or two; d(std) = d(var) / (2 std)
            dvar = (n * (xb * xb).sum(axis=1) + 2 * (np.abs(xb - xb.mean(axis=1, keepdims=True)) * eb).sum(axis=1)) / max(n - 1, 1)
            err[b, so:so + C * F] = (dvar / (2 * sd)).T.reshape(C * F)
    return {tr["out"]: err}


def run_linear(mem, tr):
    R, I, O = tr["R"], tr["I"], tr["O"]
    x = mem.strided(tr["in"], 4, (R, I), (tr["in_ld"], 1)).copy()
    if tr["in2"]:
        x2 = mem.strided(tr["in2"], 4, (R // tr["rows_per_b"], I), (tr["in2_ld"], 1))
        x = x + np.repeat(x2, tr["rows_per_b"], axis=0)
    W = mem.vec(tr["W"], O * I).reshape(O, I)
    y = x @ W.T
    mag = np.sqrt(I) * (np.abs(x) @ np.abs(W.T))
    if tr["bias"]:
        y = y + mem.vec(tr["bias"], O)
        mag = mag + np.abs(mem.vec(tr["bias"], O))
    mem.strided(tr["out"], 4, (R, O), (tr["out_ld"], 1), write=True)[...] = act(y, tr["act"])
    mem.side(tr.get("wsp", 0))       # split-K partial sums
    return {tr["out"]: mag * _act_gain(tr["act"])}


def run_aff_combine(mem, tr):
    es = tr["es"]
    x, y, t = mem.view(tr["x"], es), mem.view(tr["y"], es), mem.view(tr["t"], es)
    att = 1.0 + t
    mem.view(tr["out"], es, write=True)[...] = rnd(x * att + y * (2.0 - att), es)
    return {tr["out"]["p"]: 2.0 * (np.abs(x * att) + np.abs(y * (2.0 - att)))}


def run_convert(mem, tr):
    n = tr["n"]
    if tr.get("out_lo"):
        mem.writes.append((tr["out_lo"], 4, (n,), (1,), tr["out"], False))
    mem.strided(tr["out"], tr["es"], (n,), (1,), write=True)[...] = rnd(mem.vec(tr["in"], n), tr["es"])


def _dil_conv1d(x, W, dil):
    """x (B,T,Cin), W (Cout,3,Cin) tap-major, zero padding `dil` -> (B,T,Cout): sum_j x[t + (j-1)*dil] @ W[:, j].T"""
    B, T, _ = x.shape
    out = np.zeros((B, T, W.shape[0]))
    for j in range(3):
        off = (j - 1) * dil
        xs = shifted(x[:, None], 0, off, 1, T)[:, 0]
        out += xs @ W[:, j].T
    return out


def _lens(mem, tr, B, T):
    """frames per utterance of a length-masked op (clamped to [1, T]); T for every utterance in ordinary plans"""
    if not tr["lens"]:
        return np.full(B, T, dtype=int)
    return np.clip(mem.vec(tr["lens"], B).astype(int), 1, T)


def run_res2_fused(mem, tr):
    """ws_host.h make_res2_op: 7 dependent dilated k=3 convs on w8-channel groups (ecapa_tdnn.py:29-78):
    sp_i = bn(relu(conv(s_i) + bias_i)), s_0 = x_0, s_{i+1} = sp_i + x_{i+1}; out groups 0..6 = sp_0..sp_6."""
    es, w8, dil = tr["es"], tr["w8"], tr["dil"]
    xall = mem.view(tr["x"], es)[:, 0]                   # (B,T,8*w8)
    out = mem.view({**tr["out"], "C": 7 * w8}, es, write=True)     # group 7 of the block output is not this op's
    W7 = rnd(mem.vec(tr["W7"], 7 * w8 * 3 * w8, es).reshape(7, w8, 3, w8), es)
    bias, scale, shift = (mem.vec(tr[k], 7 * w8).reshape(7, w8) for k in ("bias", "scale", "shift"))
    B, T, _ = xall.shape
    lens = _lens(mem, tr, B, T)
    links = getattr(mem, "links", None)     # check link by link: s_{i+1} from the sp_i the kernel stored
    got = links.view(tr["out"], es)[:, 0] if links is not None else None
    err = np.zeros(out.shape)
    for b in range(B):       # length-masked: rows behind the utterance's end are conv padding = the utterance alone
        x = xall[b:b + 1, :lens[b]]
        s = x[..., :w8]
        out[b, 0, lens[b]:, :7 * w8] = 0.0
        for i in range(7):
            sp = rnd(np.maximum(_dil_conv1d(s, W7[i], dil) + bias[i], 0.0) * scale[i] + shift[i], es)
            out[b, 0, :lens[b], i * w8:(i + 1) * w8] = sp[0]
            mag = (np.sqrt(3 * w8) * _dil_conv1d(np.abs(s), np.abs(W7[i]), dil) + np.abs(bias[i])) * np.abs(scale[i]) + np.abs(shift[i])
            err[b, 0, :lens[b], i * w8:(i + 1) * w8] = mag[0]
            if i < 6:
                spi = got[b:b + 1, :lens[b], i * w8:(i + 1) * w8] if got is not None else sp
                s = round_to(spi + x[..., (i + 1) * w8:(i + 2) * w8], links.act) if got is not None else rnd(sp + x[..., (i + 1) * w8:(i + 2) * w8], es)
    return {tr["out"]["p"]: err}


def run_se_gate(mem, tr):
    """gate[b][c] = sigmoid(W2 relu(W1 mean_T(x[b]) + b1) + b2); W2t is W2 transposed to [H][C] (ecapa_tdnn.py:113-126).
    With colsum, the kernel sums the column sums the producing conv's epilogue wrote instead of reading x; the contract is
    still the mean of x."""
    x = mem.view(tr["x"], tr["es"])[:, 0]
    B, T, C = x.shape
    if tr["colsum"]:    # the rest of the column-sum buffer
        base, nbytes = mem._find(tr["colsum"])
        mem.read(tr["colsum"], 4, ((base + nbytes - tr["colsum"]) // 4,), (1,))
    H = tr["H"]
    W1 = mem.vec(tr["W1"], H * C).reshape(H, C)
    W2t = mem.vec(tr["W2t"], H * C).reshape(H, C)
    lens = _lens(mem, tr, B, T)
    mean = np.stack([x[b, :lens[b]].mean(axis=0) for b in range(B)])
    hid = np.maximum(mean @ W1.T + mem.vec(tr["b1"], H), 0.0)
    mem.strided(tr["gate"], 4, (B, C), (C, 1), write=True)[...] = act(hid @ W2t + mem.vec(tr["b2"], C), 3)
    dmean = np.stack([np.sqrt(lens[b]) * np.abs(x[b, :lens[b]]).mean(axis=0) for b in range(B)])
    return {tr["gate"]: _gate_err(mean, dmean, W1, mem.vec(tr["b1"], H), hid, W2t, mem.vec(tr["b2"], C))}


def _gate_err(mean, dmean, W1, b1, hid, W2t, b2):
    """error scale of sigmoid(W2 relu(W1 mean + b1) + b2): the mean's own (dmean), then each fp32 product through the
    Lipschitz constants (relu 1, sigmoid 1/4); W2t is [H][G]"""
    H, C = W1.shape
    dhid = np.sqrt(C) * (np.abs(mean) @ np.abs(W1.T)) + np.abs(b1) + dmean @ np.abs(W1.T)
    return 0.25 * (np.sqrt(H) * (np.abs(hid) @ np.abs(W2t)) + np.abs(b2) + dhid @ np.abs(W2t))


def run_scale_residual(mem, tr):
    es = tr["es"]
    x, res = mem.view(tr["x"], es), mem.view(tr["res"], es)
    B, _, T, C = x.shape
    gate = mem.strided(tr["gate"], 4, (B, C), (C, 1))
    mem.view(tr["out"], es, write=True)[...] = rnd(x * gate[:, None, None, :] + res, es)
    return {tr["out"]["p"]: 2.0 * (np.abs(x * gate[:, None, None, :]) + np.abs(res))}


def _astp(x, logits, eps=1e-7, dlogit=None):
    """pooling_layers.py:140-144: softmax over T, weighted mean and sqrt(clamp(E[x^2] - mean^2, eps)).
    With dlogit (the error scale of each logit) also returns the error scale of each statistic: fp32 sums over T frames
    (sqrt(T) u per term), a logit error d moves the weights by a relative 2 d at most, and the variance's cancellation
    E[x^2] - mean^2 is carried explicitly: d(var) <= d(E[x^2]) + 2 |mean| d(mean), d(std) = d(var) / (2 std)."""
    a = np.exp(logits - logits.max(axis=1, keepdims=True))
    a /= a.sum(axis=1, keepdims=True)
    mean = (a * x).sum(axis=1)
    ex2 = (a * x * x).sum(axis=1)
    var = ex2 - mean * mean
    std = np.sqrt(np.maximum(var, eps))
    stats = np.concatenate([mean, std], axis=1)
    if dlogit is None:
        return stats
    T = x.shape[1]
    dl = 2.0 * dlogit.max(axis=1)
    dmean = np.sqrt(T) * (a * np.abs(x)).sum(axis=1) + dl * (a * np.abs(x - mean[:, None])).sum(axis=1)
    dex2 = np.sqrt(T) * ex2 + dl * (a * np.abs(x * x - ex2[:, None])).sum(axis=1)
    dvar = dex2 + 2.0 * np.abs(mean) * dmean
    dstd = dvar / (2.0 * std)       # std >= sqrt(eps): the clamp only shrinks the error
    return stats, np.concatenate([dmean, dstd], axis=1)


def run_astp_fused(mem, tr):
    """ws_host.h make_astp_op: logits = h @ W2^T (linear2's bias cancels in the softmax over time)."""
    es = tr["es"]
    x, h = mem.view(tr["x"], es)[:, 0], mem.view(tr["h"], es)[:, 0]
    B, T, C = x.shape
    W2 = rnd(mem.vec(tr["W2"], C * 128, es).reshape(C, 128), es)
    lens = _lens(mem, tr, B, T)
    st = mem.strided(tr["stats"], 4, (B, 2 * C), (2 * C, 1), write=True)
    err = np.zeros((B, 2 * C))
    for b in range(B):
        hb = h[b:b + 1, :lens[b]]
        st[b], e = _astp(x[b:b + 1, :lens[b]], hb @ W2.T, tr["eps"], np.sqrt(128) * (np.abs(hb) @ np.abs(W2.T)))
        err[b] = e[0]
    return {tr["stats"]: err}


def run_astp_stats(mem, tr):
    es = tr["es"]
    x, lg = mem.view(tr["x"], es)[:, 0], mem.view(tr["logits"], es)[:, 0]
    B, T, C = x.shape
    lens = _lens(mem, tr, B, T)
    st = mem.strided(tr["stats"], 4, (B, 2 * C), (2 * C, 1), write=True)
    err = np.zeros((B, 2 * C))
    for b in range(B):
        lb = lg[b:b + 1, :lens[b]]
        st[b], e = _astp(x[b:b + 1, :lens[b]], lb, tr.get("eps", 1e-7), np.abs(lb))
        err[b] = e[0]
    return {tr["stats"]: err}


def run_bnrelu(mem, tr):
    es, C = tr["es"], tr["C"]
    x = mem.view(tr["x"], es)[..., :C]
    mem.view(tr["out"], es, write=True)[..., :C] = rnd(np.maximum(x * mem.vec(tr["scale"], C) + mem.vec(tr["shift"], C), 0.0), es)
    err = np.zeros(mem.view(tr["out"], es).shape)
    err[..., :C] = 2.0 * (np.abs(x * mem.vec(tr["scale"], C)) + np.abs(mem.vec(tr["shift"], C)))
    return {tr["out"]["p"]: err}


def _cam_context(h, seg_len):
    """campplus.py:108-135: mean over T + per-segment means (avg_pool1d, ceil_mode: the last segment averages its own frames),
    one context vector per segment: (B, nseg, C)."""
    B, T, C = h.shape
    nseg = (T + seg_len - 1) // seg_len
    seg = np.stack([h[:, s * seg_len:min(T, (s + 1) * seg_len)].mean(axis=1) for s in range(nseg)], axis=1)
    return h.mean(axis=1)[:, None, :] + seg


def run_cam_gate(mem, tr):
    es, H, G, L = tr["es"], tr["H"], tr["G"], tr["seg_len"]
    h = mem.view(tr["x"], es)[:, 0]
    B, T, C = h.shape
    ctx = _cam_context(h, L)
    W1 = mem.vec(tr["W1"], H * C).reshape(H, C)
    W2 = mem.vec(tr["W2"], G * H).reshape(G, H)
    hid = np.maximum(ctx @ W1.T + mem.vec(tr["b1"], H), 0.0)
    nseg = ctx.shape[1]
    mem.strided(tr["gate"], 4, (B, nseg, G), (nseg * G, G, 1), write=True)[...] = act(hid @ W2.T + mem.vec(tr["b2"], G), 3)
    dctx = np.sqrt(T) * np.abs(h).mean(axis=1)[:, None, :] + np.sqrt(L) * _cam_context(np.abs(h), L)
    return {tr["gate"]: _gate_err(ctx, dctx, W1, mem.vec(tr["b1"], H), hid, W2.T, mem.vec(tr["b2"], G))}


def run_seg_means(mem, tr):
    es, L = tr["es"], tr["seg_len"]
    h = mem.view(tr["x"], es)[:, 0]
    B, T, C = h.shape
    nseg = (T + L - 1) // L
    mem.strided(tr["mean"], 4, (B, C), (C, 1), write=True)[...] = h.mean(axis=1)
    seg = np.stack([h[:, s * L:min(T, (s + 1) * L)].mean(axis=1) for s in range(nseg)], axis=1)
    mem.strided(tr["segmean"], 4, (B, nseg, C), (nseg * C, C, 1), write=True)[...] = seg
    dseg = np.stack([np.sqrt(L) * np.abs(h[:, s * L:min(T, (s + 1) * L)]).mean(axis=1) for s in range(nseg)], axis=1)
    return {tr["mean"]: np.sqrt(T) * np.abs(h).mean(axis=1), tr["segmean"]: dseg}


def run_cam_dense(mem, tr):
    """ws_host.h make_cam_dense_op / campplus.py:86-201, per layer: h = relu(W1 relu(bn1(x[:, :cin])) + bias2) (BN2 folded into
    W1), context mask m = sigmoid(W2c relu(W1c (mean_T(h) + segmean(h)) + b1c) + b2c) per 100-frame segment,
    x[:, cin:cin+32] = (k3 dilated conv of h) * m."""
    es, L, V = tr["es"], tr["seg_len"], tr["X"]
    B, Tmax, ld = V["B"], V["T"], V["ld"]
    Xall = mem.region(V["p"], es, (B, 1, Tmax, V["C"]), (Tmax * ld, Tmax * ld, ld, 1))
    # in place over the concat buffer: reads the channels in front of its first layer (whole 128-row tiles, so every row),
    # writes each layer's 32-channel slice
    mem.read(V["p"], es, (B, Tmax, tr["layers"][0]["cin"]), (Tmax * ld, ld, 1))
    for ly in tr["layers"]:
        mem.writes.append((V["p"] + ly["cin"] * es, es, (B, Tmax, 32), (Tmax * ld, ld, 1), None, False))
    lens = _lens(mem, tr, B, Tmax)
    links = getattr(mem, "links", None)     # check layer by layer: each layer reads the slices the kernel stored
    got = links.view(tr["X"], es) if links is not None else None
    u16 = {"bf16": 2.0 ** -8, "fp16": 2.0 ** -11}.get(getattr(links, "act", None), 0.0)
    err = np.zeros(Xall.shape)
    for b in range(B):       # one utterance at a time over its own frames (what the one-CTA-per-utterance kernel does)
        T = lens[b]
        X = Xall[b:b + 1, :, :T]
        for ly in tr["layers"]:
            cin, dil = ly["cin"], ly["dil"]
            Xin = got[b:b + 1, :, :T] if got is not None else X
            xin = rnd(np.maximum(Xin[:, 0, :, :cin] * mem.vec(ly["bn1_scale"], cin) + mem.vec(ly["bn1_shift"], cin), 0.0), es)
            W1 = rnd(mem.vec(ly["W1"], 128 * cin, es).reshape(128, cin), es)
            h = rnd(np.maximum(xin @ W1.T + mem.vec(ly["bias2"], 128), 0.0), es)
            # the kernel rounds xin and h to 16 bits (one unit roundoff each) and accumulates in fp32; in units of u32
            dh = (u16 / 2.0 ** -23) * (np.abs(h) + np.abs(xin) @ np.abs(W1.T)) + np.sqrt(cin) * (np.abs(xin) @ np.abs(W1.T))
            ctx = _cam_context(h, L)                                           # (1,nseg,128)
            w1c_t = mem.vec(ly["w1c_t"], 128 * 64).reshape(128, 64)
            w2c_t = mem.vec(ly["w2c_t"], 64 * 32).reshape(64, 32)
            m = act(np.maximum(ctx @ w1c_t + mem.vec(ly["b1c"], 64), 0.0) @ w2c_t + mem.vec(ly["b2c"], 32), 3)   # (1,nseg,32)
            Wl = rnd(mem.vec(ly["Wl"], 32 * 3 * 128, es).reshape(32, 3, 128), es)
            y = _dil_conv1d(h, Wl, dil)
            seg_of_t = np.arange(T) // L
            X[:, 0, :, cin:cin + 32] = rnd(y * m[:, seg_of_t, :], es)
            # rows behind the utterance's end: zeros in the plan re-evaluation; the kernel's 128-row stores leave values there
            # that no later op reads (it works over each utterance's own frames), so the check takes what it stored
            Xall[b, 0, T:, cin:cin + 32] = got[b, 0, T:, cin:cin + 32] if got is not None else 0.0
            dy = _dil_conv1d(dh + np.sqrt(3 * 128) * np.abs(h), np.abs(Wl), dil)
            err[b, 0, :T, cin:cin + 32] = (dy * m[:, seg_of_t, :])[0] + 2.0 * np.abs(y * m[:, seg_of_t, :])[0]
    return {V["p"] + ly["cin"] * es: err[:, 0, :, ly["cin"]:ly["cin"] + 32] for ly in tr["layers"]}


def run_lens_derive(mem, tr):
    """frames per utterance behind each stride-2 level: level 0 clamped to [1, T], level k + 1 = (level k - 1) // 2 + 1"""
    B, T, levels = tr["B"], tr["T"], tr["levels"]
    mem.read(tr["lens"], 4, (B,), (1,))
    lens = mem.strided(tr["lens"], 4, (levels, B), (B, 1), write=True)
    lens[0] = np.clip(lens[0], 1, T)
    for k in range(1, levels):
        lens[k] = (lens[k - 1] - 1) // 2 + 1
    return {tr["lens"]: np.zeros((levels, B))}


def run_zero_tail(mem, tr):
    x = mem.view(tr["x"], tr["es"], write=True)
    B, F, T, C = x.shape
    lens = mem.vec(tr["lens"], B)
    v = tr["x"]
    for b in range(B):      # in place: the rows in front of the utterance's end are read (and kept), the rest written
        mem.read(v["p"] + b * F * T * v["ld"] * tr["es"], tr["es"], (F, int(min(max(lens[b], 0), T)), C), (T * v["ld"], v["ld"], 1))
    x[...] = np.where((np.arange(T)[None, :] < lens[:, None])[:, None, :, None], x, 0.0)
    return {tr["x"]["p"]: np.zeros(x.shape)}


def run_simam_stats(mem, tr):
    """ws_launch_simam_stats: stats [B][2][C] = mean, sum of centred squares / (F*T_b - 1) over each utterance's frames."""
    x = mem.view(tr["x"], tr["es"])
    B, F_, T, C = x.shape
    lens = _lens(mem, tr, B, T)
    st = mem.strided(tr["stats"], 4, (B, 2, C), (2 * C, C, 1), write=True)
    err = np.zeros((B, 2, C))
    mem.side(tr.get("partial", 0))     # per-block partial sums
    for b in range(B):
        xb = x[b, :, :lens[b]]
        n = F_ * lens[b]
        mu = xb.mean(axis=(0, 1))
        st[b, 0] = mu
        st[b, 1] = ((xb - mu) ** 2).sum(axis=(0, 1)) / (n - 1)
        err[b, 0] = n * np.abs(xb).mean(axis=(0, 1))                       # sums of n terms (gamma_n)
        err[b, 1] = n * (xb * xb).sum(axis=(0, 1)) / (n - 1)
    return {tr["stats"]: err}


def run_simam_apply(mem, tr):
    """ws_launch_simam_apply: out = relu(y * sigmoid((y - mean)^2 / (4 (var + lambda)) + 0.5) + res) at out's own strides,
    rows behind an utterance's end written as zeros."""
    es = tr["es"]
    y, res = mem.view(tr["y"], es), mem.view(tr["res"], es)
    B, F_, T, C = y.shape
    st = mem.strided(tr["stats"], 4, (B, 2, C), (2 * C, C, 1))
    mu, var = st[:, 0][:, None, None, :], st[:, 1][:, None, None, :]
    z = (y - mu) ** 2 / (4.0 * (var + tr["lambda"])) + 0.5
    o = np.maximum(y / (1.0 + np.exp(-z)) + res, 0.0)
    o = np.where((np.arange(T)[None, :] < _lens(mem, tr, B, T)[:, None])[:, None, :, None], o, 0.0)
    mem.strided(tr["out"], es, (B, F_, T, C), (tr["out_sb"], tr["out_sf"], tr["out_st"], 1), write=True)[...] = rnd(o, es)
    # a few fp32 roundings on each term; the sigmoid's slope (<= 1/4) carries the relative error of its argument z
    return {tr["out"]: 4.0 * (np.abs(y) + np.abs(res)) + np.abs(y) * (z + 2.0)}


def run_dwconv3x3(mem, tr):
    """ws_launch_dwconv3x3: out = relu(depthwise 3x3(x, w) + shift), zero padding, rows behind an utterance's end read as
    zeros and written as zeros; w and shift are fp32 (never rounded to the activation dtype)."""
    es = tr["es"]
    x = mem.view(tr["x"], es)
    B, F_, T, C = x.shape
    valid = (np.arange(T)[None, :] < _lens(mem, tr, B, T)[:, None])[:, None, :, None]
    x = np.where(valid, x, 0.0)
    w = mem.vec(tr["w"], C * 9).reshape(C, 3, 3)
    acc = np.zeros(x.shape)
    mag = np.zeros(x.shape)
    for jf in range(3):
        for jt in range(3):
            acc += shifted(x, jf - 1, jt - 1, F_, T) * w[:, jf, jt]
            mag += np.abs(shifted(x, jf - 1, jt - 1, F_, T) * w[:, jf, jt])
    out = np.where(valid, np.maximum(acc + mem.vec(tr["shift"], C), 0.0), 0.0)
    mem.view(tr["out"], es, write=True)[...] = rnd(out, es)
    return {tr["out"]["p"]: 3.0 * mag + np.abs(mem.vec(tr["shift"], C))}


EXTRA = {"simam_stats": run_simam_stats, "simam_apply": run_simam_apply, "dwconv3x3": run_dwconv3x3,
         "lens_derive": run_lens_derive, "zero_tail": run_zero_tail, "res2_fused": run_res2_fused, "se_gate": run_se_gate, "scale_residual": run_scale_residual, "astp_fused": run_astp_fused,
         "astp_stats": run_astp_stats, "bnrelu": run_bnrelu, "cam_gate": run_cam_gate, "seg_means": run_seg_means,
         "cam_dense": run_cam_dense}


def run_plan(path, feats, n_frames=None):
    """feats (B,T,feat_dim) float -> embeddings (B,embed_dim) float64 by re-evaluating the traced plan on the host.
    n_frames: per-utterance frame counts of a length-masked plan (ws_engine_forward_masked)."""
    meta, blob = load_trace(path)
    B, T, Fd, E = meta["B"], meta["T"], meta["feat_dim"], meta["embed_dim"]
    assert feats.shape == (B, T, Fd)
    mem = Memory(meta, blob)
    arr, off = mem.array(meta["feats_in"], 4)
    arr[off:off + B * T * Fd] = np.asarray(feats, np.float64).reshape(-1)
    assert (n_frames is not None) == bool(meta["lens"]), "n_frames goes with a masked plan"
    if n_frames is not None:
        arr, off = mem.array(meta["lens"], 4)
        arr[off:off + B] = np.asarray(n_frames, np.float64)
    for op in meta["ops"]:
        if op["trace"] is None:
            raise NotImplementedError("no trace for op " + op["label"])
        run_op(mem, op["trace"], meta)
    return mem.vec(meta["emb"], B * E).reshape(B, E).copy(), meta


def run_op(mem, tr, meta):
    """evaluate one op's contract on `mem`; returns {output address: error scale} (see run_conv)"""
    kind = tr["kind"]
    if kind == "conv":
        return run_conv(mem, tr)
    if kind == "conv3x3":
        return run_conv3x3(mem, tr)
    if kind == "stem":
        return run_stem(mem, tr, meta)
    if kind == "tstats":
        return run_tstats(mem, tr)
    if kind == "linear":
        return run_linear(mem, tr)
    if kind == "aff_combine":
        return run_aff_combine(mem, tr)
    if kind == "convert":
        return run_convert(mem, tr)
    if kind in EXTRA:
        return EXTRA[kind](mem, tr)
    raise NotImplementedError(kind)


# ------------------------------------------------------------------------------------------------ one op on real memory
# A real engine with the option plan_trace = 1 writes the same trace with device addresses (model.device_trace) and runs
# its plan op by op (model.run_ops).  RawMemory evaluates an op's contract on the bytes the op found in memory, decoded from
# the dtype each operand is stored in, and check_op compares every element the op wrote with that contract and checks that
# no byte outside the op's declared outputs changed.  The same checker runs on the CPU over plan-check traces (with a
# "perfect kernel" made by rounding the contract's results), which is how tests/test_plan_ops_checker.py shows it can fail.

U32 = 2.0 ** -23
_FMT = {"bf16": (7, -126), "fp16": (10, -14), "fp32": (23, -126)}


def act_dtype(meta):
    return {"bf16": "bf16", "fp16": "fp16"}.get(meta["precision"], "fp32")


def ulp(x, dt):
    """unit in the last place of |x| in dtype dt (subnormal spacing below the smallest normal)"""
    mant, emin = _FMT[dt]
    e = np.floor(np.log2(np.maximum(np.abs(x), 2.0 ** emin)))
    return 2.0 ** (e - mant)


def round_to(x, dt):
    """fp64 -> nearest value of dtype dt (round to nearest even), as fp64"""
    import torch
    t = torch.from_numpy(np.ascontiguousarray(x, dtype=np.float64))
    return t.to({"bf16": torch.bfloat16, "fp16": torch.float16, "fp32": torch.float32}[dt]).to(torch.float64).numpy()


def decode(raw, es, dt, is_int=False):
    """uint8 numpy bytes -> float64 elements"""
    if es == 4:
        return raw.view(np.int32 if is_int else np.float32).astype(np.float64)
    if dt == "fp16":
        return raw.view(np.float16).astype(np.float64)
    return (raw.view(np.uint16).astype(np.uint32) << 16).view(np.float32).astype(np.float64)


def encode(vals, es, dt, is_int=False):
    """float64 elements -> uint8 bytes in dtype (es, dt), rounded to nearest"""
    if es == 4:
        return (np.rint(vals).astype(np.int32) if is_int else vals.astype(np.float32)).view(np.uint8)
    import torch
    t = torch.from_numpy(np.ascontiguousarray(vals, dtype=np.float64)).to(torch.float16 if dt == "fp16" else torch.bfloat16)
    return t.view(torch.int16).numpy().view(np.uint8)


class RawMemory(Memory):
    """The allocations of a traced plan as raw bytes (raw: base address -> torch uint8 tensor, on any device); operands are
    decoded to float64 from the dtype they are stored in: 2-byte elements in the plan's activation dtype, 4-byte ones fp32
    except the int32 frame counts."""

    def __init__(self, meta, raw):
        super().__init__({"allocs": meta["allocs"], "blobs": []}, np.zeros(0, np.float32))
        self.raw = raw
        self.act = act_dtype(meta)
        self.int_base = self._find(meta["lens"])[0] if meta["lens"] else None
        self.tf32_cut = False
        self.links = None

    def array(self, addr, es):
        base, nbytes = self._find(addr)
        if base not in self.bufs:
            self.bufs[base] = (decode(self.raw[base].cpu().numpy()[:nbytes // es * es], es, self.act, base == self.int_base), es)
        arr, es0 = self.bufs[base]
        assert es0 == es and (addr - base) % es == 0, (addr, es0, es)
        return arr, (addr - base) // es


class _DevBytes:
    """an engine allocation as a zero-copy uint8 CUDA tensor (torch.as_tensor takes __cuda_array_interface__)"""

    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": "|u1", "data": (ptr, False), "version": 3}


def device_memory(meta, feats, n_frames=None, device="cuda:0"):
    """{base address: zero-copy uint8 CUDA tensor} over every allocation of a real engine's trace (model.device_trace), with
    the features (B,T,feat_dim) written into feats_in and, in a masked plan, the frame counts into lens.  check_op takes
    clones of these as `before` and the live tensors as `after`."""
    import torch
    live = {a: torch.as_tensor(_DevBytes(a, n), device=device) for a, n in meta["allocs"]}

    def put(addr, t):
        base = max(a for a in live if a <= addr)
        b = t.contiguous().view(torch.uint8).reshape(-1).to(device)
        live[base][addr - base:addr - base + b.numel()].copy_(b)
    put(meta["feats_in"], torch.as_tensor(feats, dtype=torch.float32))
    if n_frames is not None:
        put(meta["lens"], torch.as_tensor(n_frames, dtype=torch.int32))
    return live


def _regions(mem):
    """{base: [(element offset, es, shape, strides, hi address or None)]} of the regions an op's contract declared written"""
    out = {}
    for addr, es, shape, strides, hi, side in mem.writes:
        base, _ = mem._find(addr)
        out.setdefault(base, []).append(((addr - base) // es, es, shape, strides, hi, side))
    return out


def _elements(shape, strides, off):
    idx = np.full(tuple(shape), off, dtype=np.int64)
    for d, (n, st) in enumerate(zip(shape, strides)):
        sh = [1] * len(shape)
        sh[d] = n
        idx = idx + (np.arange(n, dtype=np.int64) * st).reshape(sh)
    return idx


def _byte_mask(t, regions):
    """bool torch tensor over the bytes of allocation tensor t: True on every byte of the regions (element offset, es,
    shape, strides, ...)"""
    import torch
    mask = torch.zeros(t.numel(), dtype=torch.bool, device=t.device)
    for off, es, shape, strides, *_ in regions:
        el = torch.from_numpy(_elements(shape, strides, off).reshape(-1)).to(t.device)
        mask[:t.numel() // es * es].view(-1, es)[el] = True
    return mask


def declared_mask(raw, regions, base):
    """bool torch tensor over the bytes of allocation `base`: True where the op may write"""
    return _byte_mask(raw[base], regions.get(base, []))


def perfect_outputs(meta, before, ref):
    """what a kernel that rounds the contract's fp64 result once to its storage dtype writes: new raw bytes"""
    after = {b: t.clone() for b, t in before.items()}
    regions = sorted(((b, *r) for b, rs in _regions(ref).items() for r in rs), key=lambda r: r[5] is not None)
    for base, off, es, shape, strides, hi, side in regions:   # hi values first: a lo twin is derived from the stored hi value
        if side:
            continue
        el = _elements(shape, strides, off).reshape(-1)
        if hi is None:
            arr, _ = ref.array(base + off * es, es)
            b = encode(arr[el], es, ref.act, base == ref.int_base).reshape(-1, es)
        else:
            hb, _ = ref._find(hi)
            hv = after[hb].numpy()[: (after[hb].numel() // 4) * 4].view(np.float32)[(hi - hb) // 4 + el - off]
            b = (hv - _tf32_trunc(hv)).astype(np.float32).view(np.uint8).reshape(-1, 4)
        buf = after[base].numpy()
        for k in range(es):
            buf[el * es + k] = b[:, k]
    return after


# error-scale factor c per op kind: bound = ulp(|ref|, output dtype) + c * u32 * E, E the contract's error scale.  Measured on
# an H100 (tests/test_plan_ops_gpu.py prints the worst error / bound per kind and precision): every kind stays at or below
# 0.5 with these.  tstats needs c = 8: its std reached 1.9x the c = 2 bound over 13-frame utterances.
C_KIND = {"conv": 2.0, "conv3x3": 2.0, "stem": 2.0, "res2_fused": 2.0, "linear": 2.0, "cam_dense": 1.0, "astp_fused": 2.0,
          "astp_stats": 2.0, "tstats": 8.0, "se_gate": 2.0, "cam_gate": 2.0, "seg_means": 2.0, "bnrelu": 1.0,
          "scale_residual": 1.0, "aff_combine": 1.0, "simam_stats": 2.0, "simam_apply": 1.0,
          "dwconv3x3": 2.0, "convert": 0.0, "zero_tail": 0.0, "lens_derive": 0.0}


LINKED = ("res2_fused", "cam_dense")    # contracts checked link by link: evaluated again on what the kernel stored


class Expectation:
    """an op's contract evaluated on the memory in front of it (expect_op): the fp64 results and error scales, the regions
    it declares written and the regions it reads"""

    def __init__(self, meta, op, ref, errs, tf32_cut):
        self.meta, self.op, self.ref, self.errs, self.tf32_cut = meta, op, ref, errs, tf32_cut
        self.regions = _regions(ref)
        self.reads = {}
        for addr, es, shape, strides in ref.reads:
            base, _ = ref._find(addr)
            if base in self.regions:
                self.reads.setdefault(base, []).append(((addr - base) // es, es, shape, strides))


def expect_op(meta, op, before, tf32_cut=False):
    """Evaluate op `op`'s contract on `before` (raw bytes in front of the op) -> Expectation."""
    tr = op["trace"]
    ref = RawMemory(meta, before)
    ref.tf32_cut = tf32_cut and tr["kind"] == "conv" and tr["launch"]["kernel"] in ("tc2", "tc3")
    errs = run_op(ref, tr, meta) or {}
    return Expectation(meta, op, ref, errs, ref.tf32_cut)


def poison(exp, state):
    """Fill every byte `exp`'s op declares written (outputs, lo twins, side outputs) and its contract does not read with
    0xFF, in place: NaN in fp32, bf16 and fp16, -1 in the int32 frame counts.  A kernel that leaves a declared output
    unwritten then leaves NaN behind instead of whatever happened to be there (zeros in fresh memory, which is the right
    answer for padding rows and ReLU'd tails)."""
    for base, regs in exp.regions.items():
        t = state[base]
        m = _byte_mask(t, regs) & ~_byte_mask(t, exp.reads.get(base, []))
        t[m] = 255
    return state


def compare_op(exp, before, after):
    """Compare what exp's op wrote (after: raw bytes once it ran) with the contract; before: the bytes it ran on.  Returns
    (worst error/bound ratio, list of failure strings naming the op, the element and the values).  NaN is a value like any
    other: NaN where the contract is NaN agrees, NaN on one side only is an infinite error."""
    meta, op = exp.meta, exp.op
    tr = op["trace"]
    kind = tr["kind"]
    got = RawMemory(meta, after)
    ref, errs = exp.ref, exp.errs
    if kind in LINKED:          # (its read regions are as they were when exp was made: only declared writes are poisoned)
        ref = RawMemory(meta, before)
        ref.links = got
        errs = run_op(ref, tr, meta) or {}
    fails, worst = [], 0.0
    out_dt = lambda es: ref.act if es == 2 else "fp32"
    for addr, es, shape, strides, hi, side in ref.writes:
        if side:
            continue
        r = ref.region(addr, es, shape, strides, False)
        g = got.region(addr, es, shape, strides, False)
        name = f"{op['label']} [{kind}] @{addr:#x}"
        if hi:                      # lo twin: bit for bit v - tf32_trunc(v) of the stored hi value
            hv = got.region(hi, 4, shape, strides, False).astype(np.float32)
            want = (hv - _tf32_trunc(hv)).astype(np.float32)
            bad = np.argwhere(want.view(np.uint32) != g.astype(np.float32).view(np.uint32))
            if len(bad):
                fails.append(f"{name}: lo twin differs from v - tf32_trunc(v) at {len(bad)} elements, first {tuple(bad[0])}")
            continue
        e = errs.get(addr)
        if e is None:
            e = np.zeros(r.shape)
        if ref.int_base is not None and ref._find(addr)[0] == ref.int_base:
            bound = np.zeros(r.shape)        # frame counts: exact
        else:
            bound = ulp(r, out_dt(es)) + C_KIND[kind] * U32 * np.broadcast_to(np.abs(e), r.shape)
        with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
            ratio = np.abs(g - r) / np.where(bound > 0, bound, 1e-300)
        same = (g == r) | (np.isnan(g) & np.isnan(r))
        ratio = np.where(same, 0.0, np.where(np.isnan(ratio), np.inf, ratio))   # NaN on one side (or in the bound): infinite
        if ratio.size:
            worst = max(worst, float(ratio.max()))
            if ratio.max() > 1.0:
                i = np.unravel_index(int(np.argmax(ratio)), ratio.shape)
                fails.append(f"{name}: {int((ratio > 1).sum())} of {ratio.size} elements out of bound, worst at {i}: "
                             f"got {g[i]!r} want {r[i]!r} bound {bound[i]:.3g} (ratio {ratio[i]:.3g})")
    for base, _ in ref.allocs:
        diff = before[base] != after[base]
        if not bool(diff.any()):
            continue
        stray = diff & ~declared_mask(before, exp.regions, base)
        if bool(stray.any()):
            i = int(stray.nonzero()[0])
            fails.append(f"{op['label']} [{kind}]: wrote {int(stray.sum())} bytes outside its declared outputs, first at "
                         f"allocation {base:#x} + {i}")
    return worst, fails


def check_op(meta, op, before, after, tf32_cut=False):
    """expect_op on `before` and compare_op with `after` (no poisoning: `before` is the memory the op ran on)"""
    return compare_op(expect_op(meta, op, before, tf32_cut), before, after)
