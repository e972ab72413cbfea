"""The 128 x 256 tile of the persistent conv-GEMM (16-bit activations, lean epilogue, no epilogue-input tile) against the
128 x 128 tile it replaces: same k order, fp32 accumulation per k16 step and epilogue arithmetic, so the outputs, the SE
column sums and whole-model embeddings are bit-identical.  WS_TC2_MAX_BN=128 (read when a conv's plan is built) selects
the narrow tile for the A side.

The operator shapes are large enough that the wide tile is taken under the shape rule of build_tc2 whatever the device's
resident-cluster count: with x = (256-wide tiles) / (resident clusters) >= 5 the rule 20 r256 <= 11 r128 always holds."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from wespeaker_b200 import lib, synthetic as syn  # noqa: E402
from wespeaker_b200.models import from_synthetic  # noqa: E402

DEV = "cuda:0"
DT = {"bf16": (1, torch.bfloat16), "fp16": (2, torch.float16)}
# 218 x 200 = 43 600 positions: 341 position tiles (the last one partial; an odd count leaves the last cluster of 2 or 4 a
# missing tail tile); K = 1000 ends in a ragged 40-channel k-block; 200 frames per utterance for the column sums
B, T, K, N = 218, 200, 1000, 512

# epilogue variants: (name, act1, BN affine, residual + act2, column sums)
EPIS = [("bias_relu", 1, False, False, False), ("bias_relu_bn", 1, True, False, False), ("bias_tanh", 2, False, False, False),
        ("bias_relu_bn_colsum", 1, True, False, True), ("residual_relu", 1, False, True, False)]


def _operands(prec, seed):
    code, tdt = DT[prec]
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, 1, T, K, generator=g).to(DEV, tdt)
    w = (torch.randn(N, K, generator=g) / K ** 0.5).to(DEV, tdt)
    bias = (0.1 * torch.randn(N, generator=g)).to(DEV)
    scale = (0.5 + torch.rand(N, generator=g)).to(DEV)
    shift = (0.1 * torch.randn(N, generator=g)).to(DEV)
    res = torch.randn(B, 1, T, N, generator=g).to(DEV, tdt)
    return x, w, bias, scale, shift, res


def _run(ops, prec, use_tc, epi, max_bn):
    """one ws_conv launch whose plan is built with WS_TC2_MAX_BN=max_bn (None: the default tile choice)"""
    code, tdt = DT[prec]
    x, w, bias, scale, shift, res = ops
    _, act1, bn_aff, resid, colsum = epi
    out = torch.full((B, 1, T, N), float("nan"), device=DEV, dtype=tdt)
    cs = torch.full((2 * ((B * T + 63) // 64), N), float("nan"), device=DEV)
    d = lib.ConvDesc()
    d.x, d.B, d.F, d.T, d.Cin, d.x_ld = x.data_ptr(), B, 1, T, K, K
    d.w, d.Cout, d.kf, d.kt = w.data_ptr(), N, 1, 1
    d.dil_f = d.dil_t = d.stride_f = d.stride_t = 1
    d.bias, d.act1 = bias.data_ptr(), act1
    if bn_aff:
        d.scale, d.shift = scale.data_ptr(), shift.data_ptr()
    if resid:
        d.res, d.res_ld, d.act2 = res.data_ptr(), N, 1
    if colsum:
        d.colsum = cs.data_ptr()
    d.out, d.out_ld, d.dtype, d.use_tc = out.data_ptr(), N, code, use_tc
    old = os.environ.pop("WS_TC2_MAX_BN", None)
    if max_bn is not None:
        os.environ["WS_TC2_MAX_BN"] = str(max_bn)
    try:
        lib.check(lib.load().ws_conv(C.byref(d), None), "ws_conv")
    finally:
        os.environ.pop("WS_TC2_MAX_BN", None)
        if old is not None:
            os.environ["WS_TC2_MAX_BN"] = old
    torch.cuda.synchronize()
    return out, (cs if colsum else None)


def _check_wide_vs_narrow(prec, use_tc, epi):
    ops = _operands(prec, 7 + use_tc)
    wide, cs_w = _run(ops, prec, use_tc, epi, None)
    narrow, cs_n = _run(ops, prec, use_tc, epi, 128)
    assert torch.equal(wide, narrow), (prec, use_tc, epi[0])
    # the narrow path is itself checked against fp64 elsewhere; a loose fp32 reference keeps both from agreeing on garbage
    x, w, bias, scale, shift, res = ops
    _, act1, bn_aff, resid, _ = epi
    y = x.float().reshape(-1, K) @ w.float().t() + bias
    y = torch.relu(y) if act1 == 1 else torch.tanh(y)
    if bn_aff:
        y = y * scale + shift
    if resid:
        y = torch.relu(y + res.float().reshape(-1, N))
    tol = {"bf16": 1.2e-2, "fp16": 2e-3}[prec] * max(1.0, y.abs().max().item())
    assert (wide.float().reshape(-1, N) - y).abs().max().item() <= tol
    if cs_w is not None:
        assert torch.equal(cs_w, cs_n)
        # per-utterance sums rebuilt from the per-64-position units equal the sums of the stored output
        cs = cs_w.cpu().double().numpy()
        sums = np.zeros((B, N))
        for u in range(cs.shape[0] // 2):
            b0 = (64 * u) // T
            sums[b0] += cs[2 * u]
            if b0 + 1 < B:
                sums[b0 + 1] += cs[2 * u + 1]
        want = wide.double().sum(dim=(1, 2)).cpu().numpy()
        assert np.abs(sums - want).max() <= 1e-4 * max(1.0, np.abs(want).max())


@pytest.mark.gpu
@pytest.mark.parametrize("epi", EPIS, ids=[e[0] for e in EPIS])
@pytest.mark.parametrize("prec", ["bf16", "fp16"])
@pytest.mark.parametrize("path", ["cl1", "cl2"])
def test_wide_tile_matches_narrow_tile(path, prec, epi):
    # cl1: the single-CTA kernel (use_tc=2); cl2: clusters of two sharing the weight tile (use_tc=3 at these sizes)
    _check_wide_vs_narrow(prec, 2 if path == "cl1" else 3, epi)


@pytest.mark.gpu
def test_wide_tile_matches_narrow_tile_cluster4():
    """Clusters of four (WS_TC3_CL=4, read whenever a conv op is built) for every precision and epilogue."""
    os.environ["WS_TC3_CL"] = "4"
    try:
        for prec in DT:
            for epi in EPIS:
                _check_wide_vs_narrow(prec, 3, epi)
    finally:
        os.environ.pop("WS_TC3_CL", None)


@pytest.mark.gpu
def test_ecapa1024_wide_tile_embeddings_match_narrow():
    """ECAPA-TDNN-1024 bf16 at the headline size: embeddings with the wide tile equal those with WS_TC2_MAX_BN=128, and
    the CUDA-graph replay is bit-identical."""
    feats = torch.from_numpy(syn.make_feats(256, 200, 80, seed=5)).to(DEV)
    os.environ["WS_TC2_MAX_BN"] = "128"
    try:
        m_n = from_synthetic("ECAPA_TDNN_c1024", 0, precision="bf16")
        e_n = m_n.embed(feats).cpu()
    finally:
        os.environ.pop("WS_TC2_MAX_BN", None)
    del m_n
    m = from_synthetic("ECAPA_TDNN_c1024", 0, precision="bf16")
    e1 = m.embed(feats).cpu()
    e2 = m.embed(feats).cpu()
    assert torch.isfinite(e1).all()
    assert torch.equal(e1, e2)
    assert torch.equal(e1, e_n)


def test_ecapa1024_plan_uses_wide_tile_on_the_dense_1x1_convs():
    """Plan-check engine (no device): at B=256, T=200 the seven dense 1x1 convs (three se_res2block.0, three
    se_res2block.2, the 3072 -> 1536 conv) and layer1's k=5 conv (80 -> 1024, K = 400) take 256-wide tiles;
    WS_TC2_MAX_BN=128 gives back the narrow plan, and no other op changes."""
    m = from_synthetic("ECAPA_TDNN_c1024", precision="bf16")
    wide = m.plan_check(256, 200)
    os.environ["WS_TC2_MAX_BN"] = "128"
    try:
        narrow = m.plan_check(256, 200)
    finally:
        os.environ.pop("WS_TC2_MAX_BN", None)
    assert len(wide) == len(narrow)
    changed = [(a, b) for (a, _), (b, _) in zip(wide, narrow) if a != b]
    assert len(changed) == 8, changed
    for a, b in changed:
        assert a.startswith("conv_tc3") and " bn=256 " in a and " bn=128 " in b, (a, b)
        assert a.split(" pos=")[1] == b.split(" pos=")[1]
    shapes = sorted(a.split(" pos=")[1] for a, _ in changed)
    assert shapes == ["51200 K=1024 N=1024"] * 6 + ["51200 K=3072 N=1536", "51200 K=400 N=1024"], shapes
    assert [f for _, f in wide] == [f for _, f in narrow]
