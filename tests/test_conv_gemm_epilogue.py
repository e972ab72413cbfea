"""The one-pass epilogue of the 128 x 256 conv-GEMM tile against the 128 x 128 tile (WS_TC2_MAX_BN=128), bit for bit, on
the cases that stress its hand-offs: the consumers write the staged tile from their accumulator fragments, a helper warp
stages the next tile's per-channel parameters into one of two buffers, and the store / column-sum warps hand the
staging buffer back.

- K = 64 (one k-block per tile): epilogues run back to back, so every tile waits on the staging and parameter hand-offs.
- N = 1536 (a CTA's channel tile stays the same from tile to tile) and N = 1024 (it changes on every tile).
- SE column sums at T = 128 (utterance boundaries on 64-row units) and T = 200 (units split at the boundary).
- fp16 with tanh; clusters of 1, 2 and 4 (WS_TC3_CL=4).

Positions are B x T >= 40 000, so every shape takes the wide tile under build_tc2's shape rule (256-wide tiles per
resident cluster >= 5) and clusters of four are allowed (>= 2 x 132 x 128 positions)."""
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

# (name, prec, B, T, K, N, act1 (1 relu, 2 tanh), BN affine, column sums)
CASES = [
    ("k64_n1024_t200_relu_bn_colsum", "bf16", 200, 200, 64, 1024, 1, True, True),
    ("k64_n1536_t128_relu_bn_colsum", "bf16", 320, 128, 64, 1536, 1, True, True),
    ("k64_n1024_t128_tanh_bn_colsum", "fp16", 320, 128, 64, 1024, 2, True, True),
    ("k64_n1536_t200_tanh", "fp16", 200, 200, 64, 1536, 2, False, False),
    ("k192_n1024_t200_relu", "bf16", 200, 200, 192, 1024, 1, False, False),
]


def _run(case, ops, use_tc, max_bn):
    """one ws_conv launch whose plan is built with WS_TC2_MAX_BN=max_bn (None: the default tile choice)"""
    _, prec, B, T, K, N, act1, bn_aff, colsum = case
    code, tdt = DT[prec]
    x, w, bias, scale, shift = ops
    out = torch.full((B, 1, T, N), float("nan"), device=DEV, dtype=tdt)
    cs = torch.full((2 * ((B * T + 63) // 64), N), float("nan"), device=DEV)
    d = lib.ConvDesc()
    d.x, d.B, d.F, d.T, d.Cin, d.x_ld = x.data_ptr(), B, 1, T, K, K
    d.w, d.Cout, d.kf, d.kt = w.data_ptr(), N, 1, 1
    d.dil_f = d.dil_t = d.stride_f = d.stride_t = 1
    d.bias, d.act1 = bias.data_ptr(), act1
    if bn_aff:
        d.scale, d.shift = scale.data_ptr(), shift.data_ptr()
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


def _check(case, use_tc):
    name, prec, B, T, K, N, act1, bn_aff, colsum = case
    _, tdt = DT[prec]
    g = torch.Generator().manual_seed(K + N + T)
    x = torch.randn(B, 1, T, K, generator=g).to(DEV, tdt)
    w = (torch.randn(N, K, generator=g) / K ** 0.5).to(DEV, tdt)
    bias = (0.1 * torch.randn(N, generator=g)).to(DEV)
    scale = (0.5 + torch.rand(N, generator=g)).to(DEV)
    shift = (0.1 * torch.randn(N, generator=g)).to(DEV)
    ops = (x, w, bias, scale, shift)
    wide, cs_w = _run(case, ops, use_tc, None)
    narrow, cs_n = _run(case, ops, use_tc, 128)
    assert torch.equal(wide, narrow), (name, use_tc)
    # a loose fp32 reference keeps both tiles from agreeing on garbage
    y = x.float().reshape(-1, K) @ w.float().t() + bias
    y = torch.relu(y) if act1 == 1 else torch.tanh(y)
    if bn_aff:
        y = y * scale + shift
    tol = {"bf16": 1.2e-2, "fp16": 2e-3}[prec] * max(1.0, y.abs().max().item())
    assert (wide.float().reshape(-1, N) - y).abs().max().item() <= tol, name
    if colsum:
        assert torch.equal(cs_w, cs_n), (name, use_tc)
        # per-utterance sums rebuilt from the per-64-position units equal the sums of the stored output
        cs = cs_w.cpu().double().numpy()
        sums = np.zeros((B, N))
        for u in range(cs.shape[0] // 2):
            b0 = (64 * u) // T
            sums[b0] += cs[2 * u]
            if b0 + 1 < B:
                sums[b0 + 1] += cs[2 * u + 1]
        want = wide.double().sum(dim=(1, 2)).cpu().numpy()
        assert np.abs(sums - want).max() <= 1e-4 * max(1.0, np.abs(want).max()), name


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
@pytest.mark.parametrize("path", ["cl1", "cl2"])
def test_wide_epilogue_matches_narrow_tile(path, case):
    # cl1: the single-CTA kernel (use_tc=2); cl2: clusters of two sharing the weight tile (use_tc=3)
    _check(case, 2 if path == "cl1" else 3)


@pytest.mark.gpu
def test_wide_epilogue_matches_narrow_tile_cluster4():
    """Clusters of four (WS_TC3_CL=4, read whenever a conv op is built) on every case."""
    os.environ["WS_TC3_CL"] = "4"
    try:
        for c in CASES:
            _check(c, 3)
    finally:
        os.environ.pop("WS_TC3_CL", None)


@pytest.mark.gpu
def test_ecapa512_wide_tile_embeddings_match_narrow():
    """ECAPA-TDNN-512 bf16 at 256 x 200 (K = 512 wide convs, where the per-tile epilogue weighs most): embeddings with
    the wide tile equal those with WS_TC2_MAX_BN=128, and the CUDA-graph replay is bit-identical."""
    feats = torch.from_numpy(syn.make_feats(256, 200, 80, seed=6)).to(DEV)
    os.environ["WS_TC2_MAX_BN"] = "128"
    try:
        m_n = from_synthetic("ECAPA_TDNN_c512", 0, precision="bf16")
        e_n = m_n.embed(feats).cpu()
    finally:
        os.environ.pop("WS_TC2_MAX_BN", None)
    del m_n
    m = from_synthetic("ECAPA_TDNN_c512", 0, precision="bf16")
    e1 = m.embed(feats).cpu()
    e2 = m.embed(feats).cpu()
    assert torch.isfinite(e1).all()
    assert torch.equal(e1, e2)
    assert torch.equal(e1, e_n)


def test_ecapa512_plan_uses_wide_tile():
    """Plan-check engine (no device): ECAPA-TDNN-512 bf16 at B=256, T=200 runs 256-wide tiles, which the narrow cap
    gives back, so the model test above compares the two tiles."""
    m = from_synthetic("ECAPA_TDNN_c512", precision="bf16")
    wide = m.plan_check(256, 200)
    os.environ["WS_TC2_MAX_BN"] = "128"
    try:
        narrow = m.plan_check(256, 200)
    finally:
        os.environ.pop("WS_TC2_MAX_BN", None)
    assert any(" bn=256 " in a for a, _ in wide)
    assert not any(" bn=256 " in a for a, _ in narrow)
