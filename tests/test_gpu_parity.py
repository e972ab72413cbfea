"""GPU parity tests (run on an H100: ``pytest -m gpu``).  Everything goes through the C ABI
(wespeaker_b200/lib.py -> libwespeaker_b200.so); the oracle is only the checker.

Tolerances (stated per SURVEY.md §7/§8d):
  * fp32 precision  : embeddings rel-L2 <= 1e-4 vs the reference goldens and the oracle (north_star bar)
  * tf32/bf16/fp16  : tensor-core input rounding; the reference itself drifts 4.1e-3 under bf16 autocast
                      (SURVEY §7) so the bar is rel-L2 <= 3e-2 (bf16) / 1e-2 (fp16, tf32), reported separately
  * fbank           : |log-mel error| <= 2e-3 max, 5e-5 mean vs torchaudio goldens (fp32 FFT rounding only)
  * PLDA            : |s - s_ref| <= 1e-5 * max(1, |s_ref|) vs the fp64 reference
"""
import ctypes as C
import os
import zlib

import numpy as np
import pytest
import torch

from oracle import fbank_np, models_torch, plda_np
from wespeaker_b200 import frontend, lib, synthetic as syn
from wespeaker_b200.models import from_synthetic
from wespeaker_b200.plda import TwoCovPLDA

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
class _Goldens(dict):
    """models.npz (hot-path families) + models_f4.npz (section 8(f) rank-4 families) behind the NpzFile interface."""
    @property
    def files(self):
        return list(self.keys())


G_MODELS = _Goldens()
for _f in ("models.npz", "models_f4.npz"):
    with np.load(os.path.join(HERE, "golden", _f)) as _z:
        G_MODELS.update({k: _z[k] for k in _z.files})
G_FBANK = np.load(os.path.join(HERE, "golden", "fbank.npz"))
G_PLDA = np.load(os.path.join(HERE, "golden", "plda.npz"))
DEV = "cuda:0"
DT = {"fp32": (0, torch.float32), "tf32": (0, torch.float32), "tf32x3": (0, torch.float32), "bf16": (1, torch.bfloat16),
      "fp16": (2, torch.float16)}


def tf32_lo(t):
    """v - tf32_trunc(v): the low part of the 3xTF32 split (exact in fp32)."""
    return t - (t.view(torch.int32) & ~0x1FFF).view(torch.float32)


def rel_l2(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.linalg.norm(a - b, axis=-1) / np.linalg.norm(b, axis=-1)


# ------------------------------------------------------------------------------------------ fused conv operator
def run_conv(x_cl, w, bias, scale, shift, res, prec, use_tc, kf, kt, dil, pad, stride, act1=1, act2=0):
    """x_cl (B,F,T,Cin) float32 channels-last; w torch layout (Cout,Cin,kf,kt)."""
    code, tdt = DT[prec]
    B, F, T, Cin = x_cl.shape
    Cout = w.shape[0]
    Fo = (F + 2 * pad[0] - dil[0] * (kf - 1) - 1) // stride[0] + 1
    To = (T + 2 * pad[1] - dil[1] * (kt - 1) - 1) // stride[1] + 1
    xd = x_cl.to(DEV, tdt).contiguous()
    wp = w.permute(0, 2, 3, 1).reshape(Cout, kf * kt * Cin).to(DEV, tdt).contiguous()
    out = torch.zeros((B, Fo, To, Cout), dtype=tdt, device=DEV)
    keep = [xd, wp, out]
    out_lo = None
    d = lib.ConvDesc()
    d.x, d.B, d.F, d.T, d.Cin, d.x_ld = xd.data_ptr(), B, F, T, Cin, Cin
    d.w, d.Cout, d.kf, d.kt = wp.data_ptr(), Cout, kf, kt
    d.dil_f, d.dil_t, d.pad_f, d.pad_t, d.stride_f, d.stride_t = dil[0], dil[1], pad[0], pad[1], stride[0], stride[1]
    for name, v in (("bias", bias), ("scale", scale), ("shift", shift)):
        if v is not None:
            t = v.to(DEV, torch.float32).contiguous()
            keep.append(t)
            setattr(d, name, t.data_ptr())
    if res is not None:
        r = res.to(DEV, tdt).contiguous()
        keep.append(r)
        d.res, d.res_ld = r.data_ptr(), Cout
    d.act1, d.act2, d.out, d.out_ld, d.dtype, d.use_tc = act1, act2, out.data_ptr(), Cout, code, int(use_tc)  # 0 FFMA, 2 tc, 3 tc + clusters
    if prec == "tf32x3":
        xl, wl = tf32_lo(xd).contiguous(), tf32_lo(wp).contiguous()
        out_lo = torch.zeros_like(out)
        keep += [xl, wl, out_lo]
        d.x_lo, d.w_lo, d.out_lo = xl.data_ptr(), wl.data_ptr(), out_lo.data_ptr()
    lib.check(lib.load().ws_conv(C.byref(d), None), "ws_conv")
    torch.cuda.synchronize()
    if out_lo is not None:  # the kernel must emit the exact low part of what it stored
        assert torch.equal(out_lo, tf32_lo(out))
    return out.float().cpu()


def ref_conv(x_cl, w, bias, scale, shift, res, tdt, kf, kt, dil, pad, stride, act1=1, act2=0):
    # reference in fp64 on inputs rounded to the operand dtype (isolates kernel error from input rounding)
    x = x_cl.to(tdt).double().permute(0, 3, 1, 2)
    wq = w.to(tdt).double()
    y = torch.nn.functional.conv2d(x, wq, None if bias is None else bias.double(), stride=stride, padding=pad, dilation=dil)
    if act1 == 1:
        y = torch.relu(y)
    elif act1 == 2:
        y = torch.tanh(y)
    if scale is not None:
        y = y * scale.double()[None, :, None, None] + shift.double()[None, :, None, None]
    y = y.permute(0, 2, 3, 1)
    if res is not None:
        y = y + res.to(tdt).double()
    if act2 == 1:
        y = torch.relu(y)
    return y


CONV_CASES = [
    # name, B, F, T, Cin, Cout, kf, kt, dil, pad, stride
    ("pw512", 3, 1, 198, 512, 512, 1, 1, (1, 1), (0, 0), (1, 1)),
    ("k5_80", 4, 1, 198, 80, 512, 1, 5, (1, 1), (0, 2), (1, 1)),
    ("k3_d3_w64", 5, 1, 61, 64, 64, 1, 3, (1, 3), (0, 3), (1, 1)),
    ("c3x3_32", 2, 20, 37, 32, 32, 3, 3, (1, 1), (1, 1), (1, 1)),
    ("c3x3_s2", 2, 20, 37, 32, 64, 3, 3, (1, 1), (1, 1), (2, 2)),
    ("c3x3_s21", 2, 10, 45, 32, 32, 3, 3, (1, 1), (1, 1), (2, 1)),
    ("pw_s2", 2, 20, 37, 64, 128, 1, 1, (1, 1), (0, 0), (2, 2)),
    ("k3_d2_128_32", 2, 1, 100, 128, 32, 1, 3, (1, 2), (0, 2), (1, 1)),
    ("pw_1536_nores", 2, 1, 200, 256, 1536, 1, 1, (1, 1), (0, 0), (1, 1)),
    ("pw_many_tiles", 64, 1, 200, 128, 512, 1, 1, (1, 1), (0, 0), (1, 1)),
    ("pw_1504_nores", 2, 1, 150, 512, 1504, 1, 1, (1, 1), (0, 0), (1, 1)),   # XVEC's padded width: 47 tiles of 32 channels
    ("k3_d4_c96", 3, 1, 80, 96, 96, 1, 3, (1, 4), (0, 4), (1, 1)),          # 3 tiles of 32 channels, ragged 16-bit k-blocks
    ("pw_c160_ragged", 2, 1, 130, 160, 256, 1, 1, (1, 1), (0, 0), (1, 1)),  # one ragged k-block of a 1x1 conv
    ("c3x3_dil_f2", 2, 12, 30, 64, 64, 3, 3, (2, 1), (2, 1), (1, 1)),      # dilated along F: 2-D position tiles
]


@pytest.mark.parametrize("case", CONV_CASES, ids=[c[0] for c in CONV_CASES])
@pytest.mark.parametrize("mode", ["fp32-simt", "bf16-simt", "tf32-tc2", "bf16-tc2", "fp16-tc2", "tf32x3-tc2", "bf16-tc3", "tf32-tc3",
                                  "fp16-tc3", "tf32x3-tc3"])
def test_conv_operator(case, mode):
    name, B, F, T, Cin, Cout, kf, kt, dil, pad, stride = case
    prec, path = mode.split("-")
    g = torch.Generator().manual_seed(zlib.crc32(name.encode()) % 1000)
    x = torch.randn(B, F, T, Cin, generator=g)
    w = torch.randn(Cout, Cin, kf, kt, generator=g) / np.sqrt(Cin * kf * kt)
    bias = 0.1 * torch.randn(Cout, generator=g)
    scale = 0.5 + torch.rand(Cout, generator=g)
    shift = 0.1 * torch.randn(Cout, generator=g)
    Fo = (F + 2 * pad[0] - dil[0] * (kf - 1) - 1) // stride[0] + 1
    To = (T + 2 * pad[1] - dil[1] * (kt - 1) - 1) // stride[1] + 1
    res = None if name.endswith("nores") else torch.randn(B, Fo, To, Cout, generator=g)
    if path == "tc3":
        os.environ["WS_TC3_MIN_POS"] = "1"   # force the cluster kernel on these small shapes (odd tile tails included)
    try:
        out = run_conv(x, w, bias, scale, shift, res, prec, {"simt": 0, "tc2": 2, "tc3": 3}[path], kf, kt, dil, pad,
                       stride, 1, 1)
    finally:
        os.environ.pop("WS_TC3_MIN_POS", None)
    tdt = DT[prec][1]
    ref = ref_conv(x, w, bias, scale, shift, res, tdt, kf, kt, dil, pad, stride, 1, 1)
    err = (out.double() - ref).abs().max().item()
    scale_ref = ref.abs().max().item()
    # fp32 FFMA: accumulation rounding only.  tf32: 10-bit operand mantissa.  16-bit: inputs pre-rounded, so the
    # error left is fp32 accumulation + the 16-bit output rounding.
    tol = {"fp32": 2e-5, "tf32x3": 2e-5, "tf32": 4e-3, "bf16": 1.2e-2, "fp16": 2e-3}[prec] * max(1.0, scale_ref)
    print(f"{name} {mode}: max|err|={err:.3e} (ref max {scale_ref:.2f}, tol {tol:.1e})")
    assert err <= tol, (name, mode, err, tol)



C3_CASES = [
    # name, B, F, T, C: geometry cases of the halo-resident 3x3 kernel (ws_conv3x3.cu)
    ("l1_T200_2tiles", 2, 9, 200, 32),       # ResNet layer1 shape: one utterance per slot, two M tiles, 64-byte operand rows
    ("l1_T100_1tile", 3, 7, 100, 32),
    ("l2_T100_c64", 2, 11, 100, 64),         # layer2: 128-byte rows, resident weights
    ("l3_T50_c128_nb2", 5, 20, 50, 128),     # layer3: two utterances share an M tile (odd B), streamed weights, two K panels
    ("T25_c128_nb4", 6, 10, 25, 128),        # four utterances per tile
    ("T64_c64_nb2", 3, 5, 64, 64),           # largest pitch of the side-by-side case (P = 66)
    ("T65_c32", 2, 4, 65, 32),               # smallest one-utterance-per-slot pitch
    ("T255_multibox", 1, 4, 255, 32),        # slot needs 258 rows: two 128-row boxes + the 2-row tail box
    ("T256_multibox", 1, 3, 256, 64),
    ("T300_ttiles128", 1, 5, 300, 32),       # t tiles of 128
    ("T500_ttiles256", 1, 3, 500, 32),       # t tiles of 256, ragged last tile
    ("T998_c32", 1, 6, 998, 32),             # CAM++ FCM head at 10 s
    ("F1_single_row", 2, 1, 77, 64),
    ("many_steps", 9, 40, 100, 64),          # more steps than SMs: CTAs cross utterance boundaries mid-range
]


@pytest.mark.parametrize("case", C3_CASES, ids=[c[0] for c in C3_CASES])
@pytest.mark.parametrize("prec", ["fp16", "bf16"])
@pytest.mark.parametrize("variant", ["relu", "res_relu", "plain"])
def test_conv3x3_halo_kernel(case, prec, variant):
    """use_tc = 4 routes stride-1 3x3 convs to ws_conv3x3.cu (input rows resident in a shared-memory ring, taps as
    row-shifted wgmma operand reads).  Checked against fp64 conv2d on the rounded operands, and against the generic
    conv-GEMM kernel (same operands, same fp32 accumulation: differences only from summation order)."""
    name, B, F, T, Cc = case
    g = torch.Generator().manual_seed(zlib.crc32(name.encode()) % 1000)
    x = torch.randn(B, F, T, Cc, generator=g)
    w = torch.randn(Cc, Cc, 3, 3, generator=g) / np.sqrt(9 * Cc)
    bias = 0.1 * torch.randn(Cc, generator=g)
    res = torch.randn(B, F, T, Cc, generator=g) if variant == "res_relu" else None
    act1 = 1 if variant == "relu" else 0
    act2 = 1 if variant == "res_relu" else 0
    args = (x, w, bias, None, None, res, prec)
    geo = (3, 3, (1, 1), (1, 1), (1, 1), act1, act2)
    out = run_conv(*args, 4, *geo)
    ref = ref_conv(x, w, bias, None, None, res, DT[prec][1], *geo)
    err = (out.double() - ref).abs().max().item()
    tol = {"bf16": 1.2e-2, "fp16": 2e-3}[prec] * max(1.0, ref.abs().max().item())
    print(f"conv3x3 {name} {prec} {variant}: max|err|={err:.3e} (tol {tol:.1e})")
    assert err <= tol, (name, prec, variant, err, tol)
    if B * F * T <= 20000:
        gen = run_conv(*args, 2, *geo)
        assert (out - gen).abs().max().item() <= tol


C3_STRIDED = [
    # name, B, F, T, Cin, Cout, stride_f, stride_t
    ("r34_l2", 2, 20, 50, 32, 64, 2, 2),         # ResNet layer2 conv1: both strides, channel doubling, 64-byte operand rows
    ("r34_l3", 3, 11, 37, 64, 128, 2, 2),        # odd extents
    ("r34_l4in", 2, 10, 26, 128, 128, 2, 2),     # two K panels
    ("fcm_s21", 2, 21, 150, 32, 32, 2, 1),       # CAM++ FCM: frequency-only stride
    ("fcm_s21_long", 1, 10, 600, 32, 32, 2, 1),  # t tiles
    ("s22_long", 1, 6, 700, 32, 64, 2, 2),       # stride-2 time planes with t tiles of 128 outputs
    ("s12", 2, 5, 90, 64, 64, 1, 2),
    ("many_steps_s22", 40, 20, 30, 32, 64, 2, 2),
]


@pytest.mark.parametrize("case", C3_STRIDED, ids=[c[0] for c in C3_STRIDED])
@pytest.mark.parametrize("prec", ["fp16", "bf16"])
def test_conv3x3_halo_kernel_strided(case, prec):
    """Strided variants of ws_conv3x3.cu: stride 2 along F consumes two ring rows per step; stride 2 along T reads the even
    and the shifted odd time plane of a row (two TMA views with a doubled t stride) as separate operand sub-slots."""
    name, B, F, T, Cin, Cout, sf, st = case
    g = torch.Generator().manual_seed(zlib.crc32(name.encode()) % 1000)
    x = torch.randn(B, F, T, Cin, generator=g)
    w = torch.randn(Cout, Cin, 3, 3, generator=g) / np.sqrt(9 * Cin)
    bias = 0.1 * torch.randn(Cout, generator=g)
    geo = (3, 3, (1, 1), (1, 1), (sf, st), 1, 0)
    out = run_conv(x, w, bias, None, None, None, prec, 4, *geo)
    ref = ref_conv(x, w, bias, None, None, None, DT[prec][1], *geo)
    assert tuple(out.shape) == tuple(ref.shape)
    err = (out.double() - ref).abs().max().item()
    tol = {"bf16": 1.2e-2, "fp16": 2e-3}[prec] * max(1.0, ref.abs().max().item())
    print(f"conv3x3 strided {name} {prec}: max|err|={err:.3e} (tol {tol:.1e})")
    assert err <= tol, (name, prec, err, tol)


def test_conv3x3_ring_depths_agree():
    """Ring depth only changes the pipelining (WS_C3_RING caps it): identical bits for depths 4..8."""
    g = torch.Generator().manual_seed(3)
    x = torch.randn(3, 30, 100, 32, generator=g)
    w = torch.randn(32, 32, 3, 3, generator=g) / np.sqrt(288)
    bias = 0.1 * torch.randn(32, generator=g)
    res = torch.randn(3, 30, 100, 32, generator=g)
    outs = []
    for depth in ("4", "5", "8"):
        os.environ["WS_C3_RING"] = depth
        try:
            outs.append(run_conv(x, w, bias, None, None, res, "fp16", 4, 3, 3, (1, 1), (1, 1), (1, 1), 0, 1))
        finally:
            os.environ.pop("WS_C3_RING", None)
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[0], outs[2])


@pytest.mark.parametrize("name,prec,B,T", [("ResNet34", "fp16", 3, 200), ("ResNet34", "bf16", 2, 99), ("ResNet18", "fp16", 2, 57),
                                           ("CAMPPlus", "bf16", 2, 198), ("ResNet34", "fp16", 2, 612)])
def test_conv3x3_engine_path_matches_generic_path(name, prec, B, T):
    """Whole models with the halo-resident kernel on (default) and off (`conv3x3` = 0): same operands and roundings, so the
    embeddings agree to summation-order level, and fewer launches are not the point (same count +- shortcut convs)."""
    feats = torch.from_numpy(syn.make_feats(B, T, 80, seed=9)).to(DEV)
    m1 = from_synthetic(name, 0, precision=prec)
    m1.set_option("conv3x3", 1)
    m0 = from_synthetic(name, 0, precision=prec)
    m0.set_option("conv3x3", 0)
    e1, e0 = m1.embed(feats).cpu().numpy(), m0.embed(feats).cpu().numpy()
    rel = rel_l2(e1, e0).max()
    print(f"conv3x3 on/off {name} {prec} B{B} T{T}: rel {rel:.2e}, launches {m1.last_launches()} vs {m0.last_launches()}")
    assert np.isfinite(e1).all() and rel <= 3e-3


@pytest.mark.parametrize("prec,B,T,block", [("bf16", 3, 198, 0), ("fp16", 2, 455, 0), ("bf16", 2, 98, 0), ("bf16", 1, 998, 0),
                                            ("bf16", 5, 300, 1), ("fp16", 2, 200, 1)])
def test_campplus_fused_dense_layers_match_unfused(prec, B, T, block):
    """ws_cam_dense.cu (BN-ReLU on load, 1x1 conv, context gate and dilated conv of a CAMDenseTDNNLayer in one launch; with
    `cam_block` all layers of a dense block in one launch) against the 4-launch path: same roundings of h and of the new
    channels, so the embeddings agree to summation-order level; and both against the oracle."""
    feats = torch.from_numpy(syn.make_feats(B, T, 80, seed=13))
    mf = from_synthetic("CAMPPlus", 0, precision=prec)
    mf.set_option("cam_block", block)
    mu = from_synthetic("CAMPPlus", 0, precision=prec)
    mu.set_option("cam_fused", 0)
    ef, eu = mf.embed(feats.to(DEV)).cpu().numpy(), mu.embed(feats.to(DEV)).cpu().numpy()
    ref = models_torch.forward("CAMPPlus", syn.make_state_dict("CAMPPlus", 0), feats).numpy()
    print(f"cam fused vs unfused {prec} B{B} T{T} block={block}: rel {rel_l2(ef, eu).max():.2e}; vs oracle fused {rel_l2(ef, ref).max():.2e} "
          f"unfused {rel_l2(eu, ref).max():.2e}; launches {mf.last_launches()} vs {mu.last_launches()}")
    assert np.isfinite(ef).all() and rel_l2(ef, eu).max() <= 3e-3
    assert rel_l2(ef, ref).max() <= TC_TOL[prec]
    assert mf.last_launches() < mu.last_launches() - 100


@pytest.mark.parametrize("name,prec,B,T", [("ECAPA_TDNN_c512", "bf16", 5, 200), ("ECAPA_TDNN_GLOB_c512", "fp16", 3, 203),
                                           ("ECAPA_TDNN_c1024", "bf16", 2, 256), ("ECAPA_TDNN_c512", "bf16", 3, 300),
                                           ("ECAPA_TDNN_GLOB_c512", "bf16", 2, 998), ("ECAPA_TDNN_c512", "fp16", 300, 40),
                                           ("ECAPA_TDNN_c512", "bf16", 1, 17)])
def test_ecapa_fused_astp_matches_unfused(name, prec, B, T):
    """ws_astp_fused.cu (linear2 + softmax over time + weighted mean/std in one launch, transposed logits in registers, online
    softmax over 256-frame chunks) against the linear2-launch + statistics-launch path (pooling_layers.py:119-144), and both
    against the oracle.  The fused path keeps the logits in fp32 (the unfused one rounds them to 16 bits), so the two agree
    to 16-bit rounding level."""
    feats = torch.from_numpy(syn.make_feats(B, T, 80, seed=17))
    mf = from_synthetic(name, 0, precision=prec)
    mu = from_synthetic(name, 0, precision=prec)
    mu.set_option("astp_fused", 0)
    ef, eu = mf.embed(feats.to(DEV)).cpu().numpy(), mu.embed(feats.to(DEV)).cpu().numpy()
    nref = min(B, 4)
    ref = models_torch.forward(name, syn.make_state_dict(name, 0), feats[:nref]).numpy()
    print(f"astp fused vs unfused {name} {prec} B{B} T{T}: rel {rel_l2(ef, eu).max():.2e}; vs oracle fused {rel_l2(ef[:nref], ref).max():.2e} "
          f"unfused {rel_l2(eu[:nref], ref).max():.2e}; launches {mf.last_launches()} vs {mu.last_launches()}")
    assert np.isfinite(ef).all() and rel_l2(ef, eu).max() <= 3e-3
    assert rel_l2(ef[:nref], ref).max() <= TC_TOL[prec]
    assert mf.last_launches() == mu.last_launches() - 1


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["bf16-tc2", "fp16-tc2", "tf32-tc2", "tf32x3-tc2", "bf16-tc3", "fp16-tc3", "tf32-tc3", "tf32x3-tc3"])
@pytest.mark.parametrize("variant", ["bias_relu", "bn", "bn_res_relu"])
def test_lean_epilogue_is_bit_identical_to_generic(mode, variant):
    """The tensor-core kernels carry a small 'lean' epilogue instantiation (bias/ReLU/BN/residual/ReLU) next to the generic
    one; WS_EPI_GENERIC=1 forces the generic one.  Same arithmetic in the same order -> identical bits."""
    prec, path = mode.split("-")
    B, F, T, Cin, Cout = 7, 1, 150, 256, 512
    g = torch.Generator().manual_seed(11)
    x = torch.randn(B, F, T, Cin, generator=g)
    w = torch.randn(Cout, Cin, 1, 3, generator=g) / np.sqrt(3 * Cin)
    bias = 0.1 * torch.randn(Cout, generator=g)
    scale = shift = res = None
    act2 = 0
    if variant != "bias_relu":
        scale, shift = 0.5 + torch.rand(Cout, generator=g), 0.1 * torch.randn(Cout, generator=g)
    if variant == "bn_res_relu":
        res, act2 = torch.randn(B, F, T, Cout, generator=g), 1
    outs = []
    for generic in ("0", "1"):
        os.environ["WS_EPI_GENERIC"] = generic
        os.environ["WS_TC3_MIN_POS"] = "1"
        try:
            outs.append(run_conv(x, w, bias, scale, shift, res, prec, {"tc2": 2, "tc3": 3}[path], 1, 3, (1, 2), (0, 2), (1, 1), 1, act2))
        finally:
            os.environ.pop("WS_EPI_GENERIC", None)
            os.environ.pop("WS_TC3_MIN_POS", None)
    assert torch.equal(outs[0], outs[1])
    ref = ref_conv(x, w, bias, scale, shift, res, DT[prec][1], 1, 3, (1, 2), (0, 2), (1, 1), 1, act2)
    assert (outs[0].double() - ref).abs().max().item() <= {"tf32x3": 2e-5, "tf32": 4e-3, "bf16": 1.2e-2, "fp16": 2e-3}[prec] * max(1.0, ref.abs().max().item())



@pytest.mark.parametrize("path", ["tc2", "tc3"])
@pytest.mark.parametrize("prec,B,T", [("bf16", 5, 150), ("fp16", 3, 200), ("bf16", 2, 128), ("bf16", 7, 333)])
def test_conv_fused_se_column_sums(path, prec, B, T):
    """ws_conv_desc.colsum: the dense 1x1 conv also emits per-64-position column sums of what it stored (the SE squeeze of
    ecapa_tdnn.py:120-121 without a second pass); rebuilt per-utterance means must equal the mean of the output tensor."""
    code, tdt = DT[prec]
    Cin, Cout = 256, 512
    g = torch.Generator().manual_seed(B * 1000 + T)
    x = torch.randn(B, 1, T, Cin, generator=g).to(DEV, tdt)
    w = (torch.randn(Cout, Cin, generator=g) / 16).to(DEV, tdt)
    bias = (0.1 * torch.randn(Cout, generator=g)).to(DEV)
    scale = (0.5 + torch.rand(Cout, generator=g)).to(DEV)
    shift = (0.1 * torch.randn(Cout, generator=g)).to(DEV)
    out = torch.zeros(B, 1, T, Cout, device=DEV, dtype=tdt)
    units = (B * T + 63) // 64
    cs = torch.full((2 * units, Cout), float("nan"), device=DEV)
    d = lib.ConvDesc()
    d.x, d.B, d.F, d.T, d.Cin, d.x_ld = x.data_ptr(), B, 1, T, Cin, Cin
    d.w, d.Cout, d.kf, d.kt = w.data_ptr(), Cout, 1, 1
    d.dil_f = d.dil_t = d.stride_f = d.stride_t = 1
    d.bias, d.act1, d.scale, d.shift = bias.data_ptr(), 1, scale.data_ptr(), shift.data_ptr()
    d.out, d.out_ld, d.dtype, d.use_tc, d.colsum = out.data_ptr(), Cout, code, {"tc2": 2, "tc3": 3}[path], cs.data_ptr()
    os.environ["WS_TC3_MIN_POS"] = "1"
    try:
        lib.check(lib.load().ws_conv(C.byref(d), None), "ws_conv")
    finally:
        os.environ.pop("WS_TC3_MIN_POS", None)
    torch.cuda.synchronize()
    cs = cs.cpu().double().numpy()
    assert np.isfinite(cs).all()
    sums = np.zeros((B, Cout))
    for u in range(units):
        b0 = (64 * u) // T
        sums[b0] += cs[2 * u]
        if b0 + 1 < B:
            sums[b0 + 1] += cs[2 * u + 1]
        else:
            assert (cs[2 * u + 1] == 0).all()
    want = out.double().sum(dim=(1, 2)).cpu().numpy()
    assert np.abs(sums - want).max() <= 1e-4 * max(1.0, np.abs(want).max())
    ref = ref_conv(x.float().cpu(), w.float().cpu()[:, :, None, None], bias.cpu(), scale.cpu(), shift.cpu(), None, tdt, 1, 1, (1, 1),
                   (0, 0), (1, 1), 1, 0)
    assert (out.double().cpu() - ref).abs().max().item() <= {"bf16": 1.2e-2, "fp16": 2e-3}[prec] * max(1.0, ref.abs().max().item())


def test_ecapa_se_colsum_matches_separate_squeeze():
    m = from_synthetic("ECAPA_TDNN_c512", 0, precision="bf16")
    feats = torch.from_numpy(syn.make_feats(6, 200, 80, seed=3)).to(DEV)
    a = m.embed(feats).cpu().numpy()
    m2 = from_synthetic("ECAPA_TDNN_c512", 0, precision="bf16")
    m2.set_option("se_colsum", 0)
    b = m2.embed(feats).cpu().numpy()
    assert rel_l2(a, b).max() < 2e-3


# ------------------------------------------------------------------------------------------ fbank + CMN
@pytest.mark.parametrize("wt", ["hamming", "povey"])
def test_fbank_matches_torchaudio_golden(wt):
    wavs = torch.from_numpy(syn.make_wavs(3, 32000, seed=0)).to(DEV)
    out = frontend.fbank_batch(wavs, window_type=wt).cpu().numpy()
    ref = G_FBANK[f"fbank_{wt}"]
    d = np.abs(out - ref)
    print(f"fbank {wt}: max {d.max():.3e} mean {d.mean():.3e}")
    assert out.shape == ref.shape and d.max() < 2e-3 and d.mean() < 5e-5
    # int16 PCM input is bit-identical to the float path (samples are integers)
    out16 = frontend.fbank_batch(wavs.to(torch.int16), window_type=wt).cpu().numpy()
    assert np.array_equal(out16, out)


def test_fbank_cmn_short_ragged_and_oracle():
    short = syn.make_wavs(1, 16000 + 77, seed=5)
    out = frontend.fbank_batch(torch.from_numpy(short).to(DEV)).cpu().numpy()[0]
    assert out.shape == (98, 80) and np.abs(out - G_FBANK["fbank_hamming_short"]).max() < 2e-3
    assert np.abs(out - fbank_np.fbank(short[0])).max() < 2e-3
    cm = frontend.fbank_batch(torch.from_numpy(syn.make_wavs(3, 32000, seed=0)).to(DEV), cmn=True).cpu().numpy()
    assert np.abs(cm - G_FBANK["cmvn_hamming"]).max() < 2e-3
    assert np.abs(cm.mean(axis=1)).max() < 1e-4
    # edge cases: shorter than one frame -> zero frames; exactly one frame
    assert frontend.fbank_batch(torch.zeros(2, 399, device=DEV)).shape == (2, 0, 80)
    one = frontend.fbank_batch(torch.from_numpy(syn.make_wavs(1, 400, seed=1)).to(DEV)).cpu().numpy()
    assert one.shape == (1, 1, 80) and np.abs(one[0] - fbank_np.fbank(syn.make_wavs(1, 400, seed=1)[0])).max() < 2e-3
    # odd sample counts with B > 1 (rows start at odd offsets: the paired-sample loads must fall back to scalar loads)
    wo = syn.make_wavs(3, 16077, seed=6)
    fo = frontend.fbank_batch(torch.from_numpy(wo).to(DEV)).cpu().numpy()
    for i in range(3):
        assert np.abs(fo[i] - fbank_np.fbank(wo[i])).max() < 2e-3
    # CMN'd features are invariant to the input gain (log-mel gain is additive): property at full size
    w = torch.from_numpy(syn.make_wavs(8, 32000, seed=7)).to(DEV)
    a = frontend.fbank_batch(w, cmn=True)
    b = frontend.fbank_batch(w * 0.5, cmn=True)
    assert (a - b).abs().max().item() < 2e-3


# ------------------------------------------------------------------------------------------ model parity
def parse_case(key):
    name, rest = key.split("__")
    s, b, t = rest.split("_")
    return name, int(s[1:]), int(b[1:]), int(t[1:])


@pytest.mark.parametrize("key", list(G_MODELS.files))
def test_model_fp32_matches_reference_golden(key):
    name, seed, B, T = parse_case(key)
    m = from_synthetic(name, seed, precision="fp32")
    feats = torch.from_numpy(syn.make_feats(B, T, 80, seed=seed + 17 * T)).to(DEV)
    out = m(feats)
    emb = (out[-1] if isinstance(out, tuple) else out).cpu().numpy()
    rel = rel_l2(emb, G_MODELS[key])
    print(f"{key} fp32: rel-L2 max {rel.max():.3e}, launches {m.last_launches()}")
    assert rel.max() <= 1e-4, (key, rel)
    # second call replays the CUDA graph: must be bit-identical
    emb2 = m(feats)
    emb2 = (emb2[-1] if isinstance(emb2, tuple) else emb2).cpu().numpy()
    assert np.array_equal(emb, emb2)


TC_TOL = {"tf32": 1e-2, "bf16": 1e-2, "fp16": 1e-2}   # measured: <= 7.9e-3 / 4.2e-3 / 5.3e-4; the reference itself drifts 4.1e-3 under bf16 autocast


@pytest.mark.parametrize("name,B,T,prec", [("ECAPA_TDNN_c1024", 5, 200, "bf16"), ("ECAPA_TDNN_c512", 3, 198, "fp16"),
                                           ("ECAPA_TDNN_GLOB_c512", 2, 61, "bf16"), ("ECAPA_TDNN_c512", 150, 256, "bf16"),
                                           ("ECAPA_TDNN_c512", 3, 257, "bf16"), ("ECAPA_TDNN_c1024", 2, 385, "fp16"),
                                           ("ECAPA_TDNN_c512", 2, 998, "bf16"), ("ECAPA_TDNN_c1024", 9, 600, "bf16")])
def test_res2_fused_chain_matches_unfused(name, B, T, prec):
    """The fused Res2 chain kernel (7 dilated convs on-chip per utterance) must reproduce the 7-launch path: same
    roundings (sp_i and s_{i+1} are rounded to the activation dtype at the same points), same tap order.  T > 256 runs as
    overlapping 256-row time tiles (halo 32 >= the chain's 7 x dilation receptive field): the stored inner rows are exact."""
    feats = torch.from_numpy(syn.make_feats(B, T, 80, seed=5)).to(DEV)
    mf = from_synthetic(name, 0, precision=prec)
    mu = from_synthetic(name, 0, precision=prec)
    mu.set_option("res2_fused", 0)
    ef, eu = mf.embed(feats).cpu().numpy(), mu.embed(feats).cpu().numpy()
    print(f"res2 fused vs unfused {name} {prec} B{B} T{T}: rel {rel_l2(ef, eu).max():.2e}, launches {mf.last_launches()} vs {mu.last_launches()}")
    assert mf.last_launches() == mu.last_launches() - 18
    assert rel_l2(ef, eu).max() <= 2e-3


@pytest.mark.parametrize("key", list(G_MODELS.files))
def test_model_tf32x3_tensor_cores_meet_fp32_bar(key):
    """3xTF32 on the tensor cores (x_lo*W + x*W_lo + x*W, fp32 accumulation): the tensor-core path itself meets the
    north-star <= 1e-4 bar against the reference goldens."""
    name, seed, B, T = parse_case(key)
    m = from_synthetic(name, seed, precision="tf32x3")
    feats = torch.from_numpy(syn.make_feats(B, T, 80, seed=seed + 17 * T)).to(DEV)
    out = m(feats)
    emb = (out[-1] if isinstance(out, tuple) else out).cpu().numpy()
    rel = rel_l2(emb, G_MODELS[key])
    print(f"{key} tf32x3: rel-L2 max {rel.max():.3e}")
    assert rel.max() <= 1e-4, (key, rel)


@pytest.mark.parametrize("prec", ["tf32", "bf16", "fp16"])
@pytest.mark.parametrize("key", ["ECAPA_TDNN_c512__s0_B4_T198", "ECAPA_TDNN_GLOB_c1024__s1_B2_T200",
                                 "ResNet34__s0_B2_T99", "CAMPPlus__s0_B2_T455", "ResNet50__s0_B2_T99", "ResNet101__s0_B1_T120",
                                 "XVEC__s0_B3_T200"])
def test_model_tensor_core_precisions(key, prec):
    name, seed, B, T = parse_case(key)
    m = from_synthetic(name, seed, precision=prec)
    feats = torch.from_numpy(syn.make_feats(B, T, 80, seed=seed + 17 * T)).to(DEV)
    out = m(feats)
    emb = (out[-1] if isinstance(out, tuple) else out).cpu().numpy()
    rel = rel_l2(emb, G_MODELS[key])
    print(f"{key} {prec}: rel-L2 max {rel.max():.3e}")
    assert np.isfinite(emb).all() and rel.max() <= TC_TOL[prec], (key, prec, rel)


@pytest.mark.parametrize("name,prec,B", [("ECAPA_TDNN_c1024", "bf16", 256), ("ECAPA_TDNN_c512", "tf32x3", 256),
                                         ("ECAPA_TDNN_c512", "bf16", 96), ("ResNet34", "fp16", 64)])
def test_bench_size_batch_matches_oracle(name, prec, B):
    """The benchmarked configurations themselves against the CPU oracle: at >= 132*128 positions the big layers run the
    weight-sharing cluster kernel (ws_tc3_launch), which the small golden cases never reach.  6 utterances spread over the
    batch are compared with oracle.models_torch on the same features (the oracle is pinned by tests/test_oracle_golden.py)."""
    T = 200
    m = from_synthetic(name, 0, precision=prec)
    feats = torch.from_numpy(syn.make_feats(B, T, 80, seed=23))
    emb = m.embed(feats.to(DEV)).cpu().numpy()
    sel = sorted({0, 1, B // 3, B // 2, B - 2, B - 1})
    ref = models_torch.forward(name, syn.make_state_dict(name, 0), feats[sel]).numpy()
    rel = rel_l2(emb[sel], ref)
    tol = 1e-4 if prec in ("fp32", "tf32x3") else TC_TOL[prec]
    print(f"bench-size {name} {prec} B{B}: rel-L2 max {rel.max():.3e} (bar {tol:g}), launches {m.last_launches()}")
    assert np.isfinite(emb).all() and rel.max() <= tol, (name, prec, rel)


def test_ecapa1024_bf16_matches_reference_golden():
    """BASELINE.json configs[1]'s model in its benchmarked precision against the reference golden (non-GLOB c1024)."""
    key = [k for k in G_MODELS.files if k.startswith("ECAPA_TDNN_c1024__")][0]
    name, seed, B, T = parse_case(key)
    m = from_synthetic(name, seed, precision="bf16")
    feats = torch.from_numpy(syn.make_feats(B, T, 80, seed=seed + 17 * T)).to(DEV)
    emb = m.embed(feats).cpu().numpy()
    rel = rel_l2(emb, G_MODELS[key])
    print(f"{key} bf16: rel-L2 max {rel.max():.3e}")
    assert rel.max() <= TC_TOL["bf16"], rel


def test_config1_ecapa512_16utts_wav_to_embedding():
    """BASELINE.json configs[0]: ECAPA-TDNN-512, 16 synthetic 2 s utterances, fbank -> CMN -> forward.
    Parity on identical fbank inputs (<=1e-4) and end-to-end from the waveform (fbank rounding included)."""
    name = "ECAPA_TDNN_c512"
    m = from_synthetic(name, 0, precision="fp32")
    sd = syn.make_state_dict(name, 0)
    wavs = syn.make_wavs(16, 32000, seed=0)
    emb, feats = m.extract_from_wav(torch.from_numpy(wavs).to(DEV), return_feats=True)
    emb, feats = emb.cpu().numpy(), feats.cpu()
    ref_same_feats = models_torch.forward(name, sd, feats).numpy()
    rel = rel_l2(emb, ref_same_feats)
    print(f"config1 identical-fbank rel-L2 max {rel.max():.3e}")
    assert rel.max() <= 1e-4
    of = np.stack([fbank_np.cmn(fbank_np.fbank(w)) for w in wavs])
    ref_e2e = models_torch.forward(name, sd, torch.from_numpy(of)).numpy()
    rel2 = rel_l2(emb, ref_e2e)
    print(f"config1 wav->emb rel-L2 max {rel2.max():.3e}")
    assert rel2.max() <= 1e-3
    # host-buffer entry point == device entry point
    emb_h = m.extract_from_wav(torch.from_numpy(wavs)).numpy()
    assert np.array_equal(emb_h, emb)
    emb_i16 = m.extract_from_wav(torch.from_numpy(wavs).to(torch.int16)).numpy()
    assert np.array_equal(emb_i16, emb)
    # pipelined host API (double-buffered H2D): same bits, batch order preserved, ragged last batch
    w16 = torch.from_numpy(wavs).to(torch.int16)
    chunks = [w16[0:6].pin_memory(), w16[6:12].pin_memory(), w16[12:16].pin_memory(), w16[0:6].pin_memory(), w16[3:5]]
    outs = [o.numpy().copy() for o in m.extract_stream(chunks)]
    assert [o.shape[0] for o in outs] == [6, 6, 4, 6, 2]
    assert np.array_equal(np.concatenate(outs[:3]), emb) and np.array_equal(outs[3], emb[:6]) and np.array_equal(outs[4], emb[3:5])


@pytest.mark.parametrize("name,prec", [("ECAPA_TDNN_c1024", "bf16"), ("ResNet34", "fp16"), ("CAMPPlus", "bf16")])
def test_batch_invariance_at_bench_size(name, prec):
    """Size-independent property at BASELINE sizes: an utterance's embedding does not depend on its batch
    (no cross-utterance leakage through tiles / padding), and the host-buffer ABI equals the device ABI."""
    B, T = (256, 200) if name.startswith("ECAPA") else (64, 200)
    m = from_synthetic(name, 0, precision=prec)
    feats = torch.from_numpy(syn.make_feats(B, T, 80, seed=11)).to(DEV)
    full = m.embed(feats).cpu().numpy()
    sub = m.embed(feats[5:8].contiguous()).cpu().numpy()
    assert np.isfinite(full).all()
    if name.startswith("ECAPA"):
        # default 16-bit ECAPA plan: the SE squeeze is summed inside the conv epilogue per 64-position unit of the FLAT
        # batch, so the fp32 summation order (not the set of summands) depends on the utterance's offset in the batch:
        # differences stay at 16-bit rounding level; any cross-utterance leak would be O(1)
        assert rel_l2(sub, full[5:8]).max() < 1e-3
        m.set_option("se_colsum", 0)   # separate squeeze pass: bitwise batch-independent again
        full0 = m.embed(feats).cpu().numpy()
        sub0 = m.embed(feats[5:8].contiguous()).cpu().numpy()
        assert rel_l2(sub0, full0[5:8]).max() < 1e-6
        assert rel_l2(full0, full).max() < 2e-3
        m.set_option("se_colsum", 1)
    else:
        assert rel_l2(sub, full[5:8]).max() < 1e-6
    host = m.embed(feats.cpu()).numpy()
    assert np.array_equal(host, full)


# ------------------------------------------------------------------------------------------ PLDA
def _tol_ok(s, ref):
    return np.abs(s - ref) <= 1e-5 * np.maximum(1.0, np.abs(ref))


@pytest.mark.parametrize("tag", ["norm", "raw"])
def test_plda_matches_reference_golden(tag):
    nl = tag == "norm"
    p = TwoCovPLDA.from_arrays(**syn.make_plda(256, seed=3, normalize_length=nl))
    enroll, test = syn.make_embeddings(48, 256, seed=3), syn.make_embeddings(40, 256, seed=4)
    e_t, t_t = p.transform_batch(enroll), p.transform_batch(test)
    assert np.abs(e_t.cpu().numpy() - G_PLDA[f"enroll_t_{tag}"]).max() < 1e-10
    assert np.abs(t_t.cpu().numpy() - G_PLDA[f"test_t_{tag}"]).max() < 1e-10
    s1 = p.score_matrix(e_t, t_t, 1, out_dtype=torch.float64).cpu().numpy()
    counts = ((np.arange(48) % 5) + 1).astype(np.int32)
    sn = p.score_matrix(e_t, t_t, counts, out_dtype=torch.float64).cpu().numpy()
    print(f"plda {tag}: max err n1 {np.abs(s1 - G_PLDA[f'scores_n1_{tag}']).max():.2e} nvar {np.abs(sn - G_PLDA[f'scores_nvar_{tag}']).max():.2e}")
    assert _tol_ok(s1, G_PLDA[f"scores_n1_{tag}"]).all() and _tol_ok(sn, G_PLDA[f"scores_nvar_{tag}"]).all()
    s1f = p.score_matrix(e_t, t_t, 1).cpu().numpy()  # fp32 output buffer (the bench configuration)
    assert _tol_ok(s1f.astype(np.float64), G_PLDA[f"scores_n1_{tag}"]).all()
    ei, ti = np.array([0, 5, 47, 13]), np.array([0, 7, 39, 2])
    tr = p.score_trials(e_t, t_t, ei, ti, counts).cpu().numpy()
    assert _tol_ok(tr, G_PLDA[f"scores_nvar_{tag}"][ei, ti]).all()
    one = p.log_likelihood_ratio(G_PLDA[f"enroll_t_{tag}"][5], G_PLDA[f"test_t_{tag}"][7], 1)
    assert abs(one - G_PLDA[f"scores_n1_{tag}"][5, 7]) <= 1e-5 * max(1, abs(one))


def test_plda_4096_block_vs_oracle_and_symmetry():
    """SURVEY §8d config 5 parity block (4096 x 4096) vs the fp64 oracle; n=1 scores are symmetric."""
    pm = syn.make_plda(256, seed=3, normalize_length=True)
    p = TwoCovPLDA.from_arrays(**pm)
    a, b = syn.make_embeddings(4096, 256, seed=21), syn.make_embeddings(4096, 256, seed=22)
    a_t, b_t = p.transform_batch(a), p.transform_batch(b)
    s = p.score_matrix(a_t, b_t, 1).cpu().numpy().astype(np.float64)
    ref = plda_np.llr_matrix(pm, plda_np.prepare_test(pm, a.astype(np.float64))[:512],
                             plda_np.prepare_test(pm, b.astype(np.float64)), 1)
    assert _tol_ok(s[:512], ref).all(), np.abs(s[:512] - ref).max()
    st = p.score_matrix(b_t, a_t, 1).cpu().numpy().astype(np.float64)
    assert np.abs(s - st.T).max() < 1e-5
    # ragged sizes (not multiples of the 128x64 tile) and empty inputs
    s2 = p.score_matrix(a_t[:130], b_t[:67], 3, out_dtype=torch.float64).cpu().numpy()
    ref2 = plda_np.llr_matrix(pm, a_t[:130].cpu().numpy(), b_t[:67].cpu().numpy(), 3)
    assert _tol_ok(s2, ref2).all()
    assert p.score_matrix(a_t[:0], b_t[:5], 1).shape == (0, 5)


# ------------------------------------------------------------------------------------------ config 4 + drop-in seams
def test_config4_campplus_variable_length_bucketed():
    """BASELINE.json configs[3]: CAM++, durations U{1..10} s, bucketed by exact length; parity per utterance against the
    oracle run at batch 1 with that utterance's own T (the reference has no padding/masking)."""
    name = "CAMPPlus"
    rng = np.random.default_rng(2)
    durs = rng.integers(1, 11, size=12)
    Ts = [1 + (int(d) * 16000 - 400) // 160 for d in durs]
    feats = [torch.from_numpy(syn.make_feats(1, T, 80, seed=100 + i)[0]) for i, T in enumerate(Ts)]
    sd = syn.make_state_dict(name, 0)
    ref = np.stack([models_torch.forward(name, sd, f[None]).numpy()[0] for f in feats])
    m32 = from_synthetic(name, 0, precision="fp32")
    e32 = m32.embed_list(feats, device=DEV).cpu().numpy()
    assert rel_l2(e32, ref).max() <= 1e-4, rel_l2(e32, ref)
    mb = from_synthetic(name, 0, precision="bf16")
    eb = mb.embed_list(feats, device=DEV).cpu().numpy()
    print(f"config4 CAM++ variable length: fp32 {rel_l2(e32, ref).max():.2e}, bf16 {rel_l2(eb, ref).max():.2e}, T={sorted(set(Ts))}")
    assert rel_l2(eb, ref).max() <= 3e-2


def _write_wav(path, pcm_i16):
    import wave
    with wave.open(str(path), "wb") as w:
        w.setnchannels(1); w.setsampwidth(2); w.setframerate(16000)
        w.writeframes(np.asarray(pcm_i16, dtype="<i2").tobytes())


def test_resample_kernel_matches_torchaudio_goldens_and_feeds_the_extractors(tmp_path):
    """ws_resample (device sinc resampler) against torchaudio.transforms.Resample outputs (goldens) for int16 and float input;
    then the two call sites of the reference: Speaker.extract_embedding on an 8 kHz file (cli/speaker.py:157-159) and
    extract() on a raw list with 8 kHz audio (processor.py:242-262) equal resample -> 16 kHz extraction."""
    import json
    import wave
    import yaml
    from oracle import resample_np
    from wespeaker_b200 import frontend, kaldi_io
    from wespeaker_b200.extract import extract
    from wespeaker_b200.speaker import Speaker
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "resample.npz"))
    for tag in ("8k_16k", "44k1_16k", "48k_16k", "22k05_16k", "16k_8k"):
        o, n = (int(v) for v in g[f"{tag}_rates"])
        x, y = g[f"{tag}_x"], g[f"{tag}_y"]
        for dt in (torch.float32, torch.int16):
            r = frontend.resample(torch.from_numpy(x).to(dt).to(DEV), o, n).cpu().numpy()
            assert r.shape == y.shape
            err = np.abs(r - y).max() / np.abs(y).max()
            assert err <= 1e-5, (tag, dt, err)
        one = frontend.resample(torch.from_numpy(x[0]).to(DEV), o, n)
        assert one.dim() == 1 and one.shape[0] == y.shape[1]
    name = "ECAPA_TDNN_c512"
    sd_np = syn.make_state_dict(name, 0)
    mdir = tmp_path / "model"
    mdir.mkdir()
    torch.save({k: torch.from_numpy(np.asarray(v)) for k, v in sd_np.items()}, mdir / "avg_model.pt")
    cfg = {"model": name, "model_args": dict(syn.DEFAULT_MODEL_ARGS[name]),
           "dataset_args": {"resample_rate": 16000, "fbank_args": {"num_mel_bins": 80}}}
    (mdir / "config.yaml").write_text(yaml.safe_dump(cfg))
    w8 = syn.make_wavs(2, 12000, seed=8).astype(np.int16)           # 1.5 s at 8 kHz
    lines = []
    for i in range(2):
        with wave.open(str(tmp_path / f"n{i}.wav"), "wb") as w:
            w.setnchannels(1); w.setsampwidth(2); w.setframerate(8000)
            w.writeframes(w8[i].astype("<i2").tobytes())
        lines.append(json.dumps({"key": f"nb{i}", "wav": str(tmp_path / f"n{i}.wav"), "spk": "s"}))
    (tmp_path / "raw8k.list").write_text("\n".join(lines) + "\n")
    ark = tmp_path / "emb8k" / "xvector.ark"
    assert extract(str(mdir / "config.yaml"), model_path=str(mdir / "avg_model.pt"), data_type="raw", data_list=str(tmp_path / "raw8k.list"),
                   embed_ark=str(ark), batch_size=1, precision="fp32") == 2
    got = kaldi_io.read_vec_scp_file(str(ark)[:-3] + "scp")
    spk = Speaker(str(mdir), precision="fp32")
    for i in range(2):
        up = resample_np.resample(w8[i:i + 1].astype(np.float32), 8000, 16000)[0]
        ref = models_torch.forward(name, sd_np, torch.from_numpy(fbank_np.cmn(fbank_np.fbank(up)))[None]).numpy()[0]
        assert rel_l2(got[f"nb{i}"], ref) <= 1e-3, rel_l2(got[f"nb{i}"], ref)
        e = spk.extract_embedding(str(tmp_path / f"n{i}.wav")).numpy()
        assert rel_l2(e, got[f"nb{i}"]) <= 1e-5


def test_extract_dropin_and_speaker_api(tmp_path):
    """Seams B2/B3: extract(config, **kwargs) writes Kaldi ark/scp from a raw data list; Speaker.extract_embedding*
    returns the same vectors; both equal the oracle pipeline (fbank -> CMN -> forward) to fp32 accuracy."""
    import json
    import yaml
    from wespeaker_b200 import kaldi_io
    from wespeaker_b200.extract import extract
    from wespeaker_b200.speaker import Speaker
    name = "ECAPA_TDNN_GLOB_c512"
    sd_np = syn.make_state_dict(name, 0)
    mdir = tmp_path / "model"
    mdir.mkdir()
    torch.save({k: torch.from_numpy(np.asarray(v)) for k, v in sd_np.items()}, mdir / "avg_model.pt")
    cfg = {"model": name, "model_args": dict(syn.DEFAULT_MODEL_ARGS[name]),
           "dataset_args": {"resample_rate": 16000, "fbank_args": {"num_mel_bins": 80, "dither": 1.0}}}
    (mdir / "config.yaml").write_text(yaml.safe_dump(cfg))
    wavs = np.concatenate([syn.make_wavs(3, 32000, seed=3), syn.make_wavs(3, 32000, seed=4)])
    lens = [32000, 32000, 24000, 32000, 24000, 17000]
    lines = []
    for i, n in enumerate(lens):
        _write_wav(tmp_path / f"u{i}.wav", wavs[i, :n].astype(np.int16))
        lines.append(json.dumps({"key": f"utt{i}", "wav": str(tmp_path / f"u{i}.wav"), "spk": "s"}))
    (tmp_path / "raw.list").write_text("\n".join(lines) + "\n")
    ark = tmp_path / "emb" / "xvector.ark"
    # batch_size 1 = whole utterances (extract.py:93 whole_utt), reader pool of 3 threads, pipelined through extract_stream
    n = extract(str(mdir / "config.yaml"), model_path=str(mdir / "avg_model.pt"), data_type="raw",
                data_list=str(tmp_path / "raw.list"), embed_ark=str(ark), batch_size=1, num_workers=3, precision="fp32")
    assert n == 6
    got = kaldi_io.read_vec_scp_file(str(ark)[:-3] + "scp")
    assert sorted(got) == [f"utt{i}" for i in range(6)]
    spk = Speaker(str(mdir), precision="fp32")
    for i, nsamp in enumerate(lens):
        w = wavs[i, :nsamp]
        ref = models_torch.forward(name, sd_np, torch.from_numpy(fbank_np.cmn(fbank_np.fbank(w)))[None]).numpy()[0]
        assert rel_l2(got[f"utt{i}"], ref) <= 1e-3, (i, rel_l2(got[f"utt{i}"], ref))
        e = spk.extract_embedding(str(tmp_path / f"u{i}.wav")).numpy()
        assert rel_l2(e, got[f"utt{i}"]) <= 1e-6
    fb = spk.compute_features(torch.from_numpy(wavs[:1]), cmn=True)[0].cpu().numpy()
    e_feats = spk.extract_embedding_from_feats([fb], batch_size=4, subseg_cmn=True)
    assert rel_l2(e_feats[0], got["utt0"]) <= 1e-5

    # batch_size > 1 = one fixed-length chunk of num_frms frames per utterance (dataset.py:236-242, processor.py:315-347):
    # random start (seeded here), short utterances tiled.  Same chunks rebuilt with the same generator for the oracle.
    import random as _random
    from wespeaker_b200.extract import get_random_chunk
    cfg2 = dict(cfg, dataset_args=dict(cfg["dataset_args"], num_frms=150))
    (mdir / "config2.yaml").write_text(yaml.safe_dump(cfg2))
    ark2 = tmp_path / "emb2" / "xvector.ark"
    n = extract(str(mdir / "config2.yaml"), model_path=str(mdir / "avg_model.pt"), data_type="raw", data_list=str(tmp_path / "raw.list"),
                embed_ark=str(ark2), batch_size=4, num_workers=2, precision="fp32", seed=7)
    got2 = kaldi_io.read_vec_scp_file(str(ark2)[:-3] + "scp")
    assert n == 6 and len(got2) == 6
    rng, clen = _random.Random(7), ((150 - 1) * 10 + 25) * 16
    for i, nsamp in enumerate(lens):
        chunk = get_random_chunk(wavs[i, :nsamp].astype(np.int16), clen, rng).astype(np.float32)
        assert len(chunk) == clen
        ref = models_torch.forward(name, sd_np, torch.from_numpy(fbank_np.cmn(fbank_np.fbank(chunk)))[None]).numpy()[0]
        assert rel_l2(got2[f"utt{i}"], ref) <= 1e-3, (i, rel_l2(got2[f"utt{i}"], ref))

    # shard list: tar members <key>.wav / <key>.spk grouped by prefix (processor.py:68-109); vad segments in a raw list
    import tarfile
    tar_path = tmp_path / "shard_000.tar"
    with tarfile.open(tar_path, "w") as tf:
        for i in range(3):
            (tmp_path / f"utt{i}.spk").write_text("s\n")
            tf.add(tmp_path / f"utt{i}.spk", arcname=f"utt{i}.spk")
            tf.add(tmp_path / f"u{i}.wav", arcname=f"utt{i}.wav")
    (tmp_path / "shards.list").write_text(str(tar_path) + "\n")
    ark3 = tmp_path / "emb3" / "xvector.ark"
    assert extract(str(mdir / "config.yaml"), model_path=str(mdir / "avg_model.pt"), data_type="shard", data_list=str(tmp_path / "shards.list"),
                   embed_ark=str(ark3), batch_size=1, precision="fp32") == 3
    got3 = kaldi_io.read_vec_scp_file(str(ark3)[:-3] + "scp")
    for i in range(3):
        assert rel_l2(got3[f"utt{i}"], got[f"utt{i}"]) <= 1e-6
    (tmp_path / "vad.list").write_text(json.dumps({"key": "v0", "wav": str(tmp_path / "u0.wav"), "spk": "s", "vad": [[0.1, 0.9], [1.2, 1.9]]}) + "\n")
    ark4 = tmp_path / "emb4" / "xvector.ark"
    assert extract(str(mdir / "config.yaml"), model_path=str(mdir / "avg_model.pt"), data_type="raw", data_list=str(tmp_path / "vad.list"),
                   embed_ark=str(ark4), batch_size=1, precision="fp32") == 1
    wv = np.concatenate([wavs[0, 1600:14400], wavs[0, 19200:30400]]).astype(np.int16).astype(np.float32)
    ref = models_torch.forward(name, sd_np, torch.from_numpy(fbank_np.cmn(fbank_np.fbank(wv)))[None]).numpy()[0]
    assert rel_l2(kaldi_io.read_vec_scp_file(str(ark4)[:-3] + "scp")["v0"], ref) <= 1e-3

    # feat list: Kaldi feature matrices by ark:offset (processor.py:169-196), CMN on the device, whole and chunked
    flines = []
    with kaldi_io.MatrixWriter(str(tmp_path / "feats.ark"), str(tmp_path / "feats.scp")) as mw:
        for i, nsamp in enumerate(lens[:4]):
            loc = mw(f"utt{i}", fbank_np.fbank(wavs[i, :nsamp]))
            flines.append(json.dumps({"key": f"utt{i}", "feat": loc, "spk": "s"}))
    (tmp_path / "feat.list").write_text("\n".join(flines) + "\n")
    ark5 = tmp_path / "emb5" / "xvector.ark"
    assert extract(str(mdir / "config.yaml"), model_path=str(mdir / "avg_model.pt"), data_type="feat", data_list=str(tmp_path / "feat.list"),
                   embed_ark=str(ark5), batch_size=1, precision="fp32") == 4
    got5 = kaldi_io.read_vec_scp_file(str(ark5)[:-3] + "scp")
    for i in range(4):
        assert rel_l2(got5[f"utt{i}"], got[f"utt{i}"]) <= 1e-3     # oracle fbank vs device fbank in front of the same model


@pytest.mark.parametrize("name,prec,tol", [("ECAPA_TDNN_c512", "fp32", 1e-5), ("ECAPA_TDNN_GLOB_c512", "bf16", 4e-3),
                                           ("ECAPA_TDNN_c1024", "bf16", 4e-3), ("ECAPA_TDNN_c512", "tf32x3", 1e-4),
                                           ("ResNet34", "fp32", 1e-5), ("ResNet34", "fp16", 2e-3), ("ResNet50", "fp16", 2e-3),
                                           ("CAMPPlus", "bf16", 4e-3), ("CAMPPlus", "fp16", 2e-3)])
def test_length_masked_batch_equals_unpadded_utterances(name, prec, tol):
    """ws_engine_forward_masked: utterances of different lengths padded to a common T in ONE batch must give what each gives
    alone (the reference has no masking: campplus.py:117-135, pooling_layers.py:78-85,119-144 statistics over the true
    frames, conv zero padding at the true end).  The padding rows are filled with large garbage to prove they are ignored;
    also checked against the oracle run per utterance."""
    lens = [200, 137, 163, 101, 256, 64] if name.startswith("ECAPA") else [200, 137, 163, 101, 301, 64]
    Tmax = max(lens)
    g = torch.Generator().manual_seed(5)
    feats = [torch.from_numpy(syn.make_feats(1, n, 80, seed=40 + i))[0] for i, n in enumerate(lens)]
    x = 50.0 * torch.randn(len(lens), Tmax, 80, generator=g)          # garbage everywhere ...
    for i, f in enumerate(feats):
        x[i, : lens[i]] = f                                            # ... except the valid frames
    m = from_synthetic(name, 0, precision=prec)
    got = m.embed_padded(x.to(DEV), lens).cpu().numpy()
    sd = syn.make_state_dict(name, 0)
    worst_self, worst_ref = 0.0, 0.0
    for i, f in enumerate(feats):
        alone = m.embed(f[None].to(DEV)).cpu().numpy()[0]
        ref = models_torch.forward(name, sd, f[None]).numpy()[0]
        worst_self = max(worst_self, float(rel_l2(got[i], alone)))
        worst_ref = max(worst_ref, float(rel_l2(got[i], ref)))
    print(f"masked batch {name} {prec}: vs alone {worst_self:.2e}, vs oracle {worst_ref:.2e}")
    assert np.isfinite(got).all() and worst_self <= tol
    assert worst_ref <= (1e-4 if prec in ("fp32", "tf32x3") else TC_TOL[prec])
    # the list API built on it: any mix of lengths through a few padded plans
    got2 = m.embed_list_padded(feats, max_batch=4, max_pad=0.3, device=DEV).cpu().numpy()
    assert rel_l2(got2, got).max() <= tol


def test_length_masked_wav_extraction():
    """ws_engine_extract_wav_masked: padded waveforms + sample counts -> fbank, CMN over each utterance's own frames, masked
    forward; equals per-utterance extraction."""
    name = "ECAPA_TDNN_c512"
    m = from_synthetic(name, 0, precision="fp32")
    ns = [32000, 24000, 17000, 40000]
    wavs = syn.make_wavs(4, 40000, seed=21)
    pad = wavs.copy()
    for i, n in enumerate(ns):
        pad[i, n:] = 9999.0                                           # garbage behind the end
    got = m.extract_from_wav_padded(torch.from_numpy(pad).to(DEV), ns).cpu().numpy()
    for i, n in enumerate(ns):
        alone = m.extract_from_wav(torch.from_numpy(wavs[i:i + 1, :n].copy()).to(DEV)).cpu().numpy()[0]
        assert rel_l2(got[i], alone) <= 1e-5, (i, rel_l2(got[i], alone))


@pytest.mark.parametrize("name,prec,tol", [("ECAPA_TDNN_c512", "fp32", 1e-5), ("CAMPPlus", "bf16", 4e-3), ("ResNet34", "fp16", 2e-3)])
def test_ragged_wav_list_any_lengths(name, prec, tol):
    """ws_engine_extract_wav_ragged_async: concatenated PCM + offsets, arbitrary sample counts, a bounded set of masked plans;
    every utterance equals its own unpadded extraction (odd offsets exercise the unaligned sample loads)."""
    m = from_synthetic(name, 0, precision=prec)
    rng = np.random.default_rng(9)
    ns = [int(v) for v in rng.integers(6000, 52000, 21)] + [1680, 1999, 16001] + ([400, 560] if name.startswith("ECAPA") else [])
    pool = syn.make_wavs(4, 52000, seed=33)
    for dt in (torch.int16, torch.float32):
        wavs = [torch.from_numpy(pool[i % 4, :n].copy()).to(dt).to(DEV) for i, n in enumerate(ns)]
        got = m.extract_from_wav_list_ragged(wavs, max_batch=8, device=DEV).cpu().numpy()
        assert got.shape == (len(ns), m.embed_dim) and np.isfinite(got).all()
        worst = 0.0
        for i, w in enumerate(wavs):
            alone = m.extract_from_wav(w[None]).cpu().numpy()[0]
            worst = max(worst, float(rel_l2(got[i], alone)))
        print(f"ragged {name} {prec} {dt}: worst vs alone {worst:.2e}")
        assert worst <= tol
    assert m.frame_grid(200) >= 200 and m.frame_grid(17) == 24
    with pytest.raises(ValueError):
        m.extract_from_wav_list_ragged([torch.zeros(399)], device=DEV)


def test_plan_cache_eviction_many_shapes():
    """More distinct (B,T) shapes than the plan cache holds (64): plans are evicted LRU and rebuilt transparently."""
    name = "ECAPA_TDNN_c512"
    m = from_synthetic(name, 0, precision="bf16")
    sd = syn.make_state_dict(name, 0)
    x0 = torch.from_numpy(syn.make_feats(2, 50, 80, seed=1)).to(DEV)
    first = m.embed(x0).cpu().numpy()
    for T in range(51, 51 + 70):
        m.embed(torch.zeros(1, T, 80, device=DEV))
    again = m.embed(x0).cpu().numpy()      # (2,50) was evicted: rebuilt plan must give the same bits
    assert np.array_equal(first, again)
    ref = models_torch.forward(name, sd, x0.cpu()).numpy()
    assert rel_l2(again, ref).max() <= 3e-2
