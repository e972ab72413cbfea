"""A kernel that uses more than 48 KB of dynamic shared memory is opted in to it where it is launched, once per device.
Each case runs in a fresh process, so that nothing has opted anything in before and the first library call of the
process is the one under test.  Each result is checked against the reference and bar of the case's existing test; the
model cases run their first embed with and without CUDA-graph capture."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from wespeaker_b200 import synthetic as syn  # noqa: E402
from wespeaker_b200.models import from_synthetic  # noqa: E402

MODELS = [("ECAPA_TDNN_c512__s0_B4_T198", "bf16"), ("ResNet34__s0_B2_T99", "fp16"), ("CAMPPlus__s0_B2_T455", "bf16"),
          ("Gemini_DF_ResNet60__s0_B2_T200_e256_w0", "fp16")]


def _conv_tc2():
    import test_conv_gemm_wide_tile as w
    w._check_wide_vs_narrow("bf16", 2, w.EPIS[0])   # the 128 x 256 tile first, then the 128 x 128 one


def _conv_tc3():
    import test_gpu_parity as g
    g.test_conv_operator(g.CONV_CASES[0], "bf16-tc3")   # sets WS_TC3_MIN_POS=1


def _conv3x3():
    import test_gpu_parity as g
    g.test_conv3x3_halo_kernel(g.C3_CASES[0], "fp16", "relu")


def _dwconv():
    import test_gemini_dfresnet as g
    g.test_gpu_dwconv_kernel_against_fp64(torch.float32, 2, 10, 64, 128, None)   # 10 x 32 fp32 tiles: 51 KB


def _plda_dmma():
    from oracle import plda_np
    from wespeaker_b200.plda import TwoCovPLDA
    pm = syn.make_plda(256, seed=3)
    p = TwoCovPLDA.from_arrays(**pm)
    # transformed on the host, so that the scoring GEMM is the first kernel launched
    e_t = plda_np.prepare_test(pm, syn.make_embeddings(130, 256, seed=1))
    t_t = plda_np.prepare_test(pm, syn.make_embeddings(67, 256, seed=2))
    ref = plda_np.llr_matrix(pm, e_t, t_t, 3)
    for dt in (torch.float64, torch.float32):
        s = p.score_matrix(e_t, t_t, 3, out_dtype=dt).cpu().numpy().astype(np.float64)
        assert (np.abs(s - ref) <= 1e-5 * np.maximum(1.0, np.abs(ref))).all(), (dt, np.abs(s - ref).max())


def _first_embed(key, prec, graph):
    if key.startswith("Gemini"):
        import test_gemini_dfresnet as g
        name, seed, B, T, args = g.parse_case(key)
        golden = g.G[key]
    else:
        import test_gpu_parity as g
        name, seed, B, T = g.parse_case(key)
        args, golden = {}, g.G_MODELS[key]
    m = from_synthetic(name, seed, precision=prec, **args)
    m.set_option("cuda_graph", graph)
    emb = m.embed(torch.from_numpy(syn.make_feats(B, T, 80, seed=seed + 17 * T)).to("cuda:0")).cpu().numpy()
    rel = g.rel_l2(emb, golden)
    print(f"{key} {prec} cuda_graph={graph}: rel-L2 max {rel.max():.3e}")
    assert np.isfinite(emb).all() and rel.max() <= 1e-2, rel


def _second_device_first():
    """the per-device opt-in: an engine on cuda:1 first, then one on cuda:0"""
    feats = torch.from_numpy(syn.make_feats(4, 198, 80, seed=5))
    e1 = from_synthetic("ECAPA_TDNN_c512", 0, precision="bf16").embed(feats.to("cuda:1")).cpu()
    e0 = from_synthetic("ECAPA_TDNN_c512", 0, precision="bf16").embed(feats.to("cuda:0")).cpu()
    assert torch.isfinite(e0).all() and torch.equal(e0, e1)


# case -> (function, environment)
CASES = {"conv_tc2": (_conv_tc2, {}), "conv_tc3_cl2": (_conv_tc3, {}), "conv_tc3_cl4": (_conv_tc3, {"WS_TC3_CL": "4"}),
         "conv3x3": (_conv3x3, {}), "dwconv": (_dwconv, {}), "plda_dmma": (_plda_dmma, {}),
         "second_device_first": (_second_device_first, {})}
for _key, _prec in MODELS:
    for _graph in (1, 0):
        CASES[f"embed_{_key.split('__')[0]}_{_prec}_graph{_graph}"] = (
            lambda k=_key, p=_prec, g=_graph: _first_embed(k, p, g), {})


def run(case):
    CASES[case][0]()


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_first_launch_in_a_fresh_process(case):
    if case == "second_device_first" and torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    env = {k: v for k, v in os.environ.items() if not k.startswith("WS_")}
    env.update(CASES[case][1])
    r = subprocess.run([sys.executable, "-c", f"import test_kernel_opt_in as t; t.run({case!r})"], cwd=HERE, env=env,
                       capture_output=True, text=True, timeout=900)
    print(r.stdout)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
