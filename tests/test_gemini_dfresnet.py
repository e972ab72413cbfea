"""Gemini DF-ResNet60 / 114 / 183 / 237 (`wespeaker/models/gemini_dfresnet.py`): a plain-torch restatement pinned on goldens
from the real reference module (tests/golden/make_golden_gemini.py), the plan builder checked without a device (the traced
plan re-evaluated on the host, including the depthwise 3x3 op), the model surface, and - on the GPU - the depthwise kernel
against fp64 and the engine against the goldens per precision."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import plan_interp  # noqa: E402  (tests/ is on sys.path under pytest's rootdir conftest)
from oracle.models_torch import _bn, _t, tstp
from wespeaker_b200 import synthetic as syn
from wespeaker_b200.models import from_synthetic, get_speaker_model

HERE = os.path.dirname(os.path.abspath(__file__))
with np.load(os.path.join(HERE, "golden", "models_gemini.npz")) as _z:
    G = {k: _z[k] for k in _z.files}
NAMES = tuple(syn.GEMINI_NAMES)
STRIDE_T = (1, 2, 1, 1)   # gemini_dfresnet.py:74-75; the frequency stride is 2 in all four downsample convs


# ------------------------------------------------------------------------------------------ oracle (torch, CPU)
def _inverted_bottleneck(x, sd, p):
    """`gemini_dfresnet.py:30-48`: 1x1 expand, depthwise 3x3, 1x1 project, each with BN; + x, ReLU."""
    out = F.relu(_bn(F.conv2d(x, _t(sd, p + ".conv1.weight", x)), sd, p + ".bn1"))
    w2 = _t(sd, p + ".conv2.weight", x)
    out = F.relu(_bn(F.conv2d(out, w2, padding=1, groups=w2.shape[0]), sd, p + ".bn2"))
    out = _bn(F.conv2d(out, _t(sd, p + ".conv3.weight", x)), sd, p + ".bn3")
    return F.relu(out + x)


def gemini_forward(sd, feats, depths, two_emb_layer=False):
    """`gemini_dfresnet.py:103-136`: feats (B, T, F) -> embed_a, or embed_b with two_emb_layer (the forward's last output)."""
    sd = {k: torch.as_tensor(np.asarray(v)) for k, v in sd.items()}
    with torch.no_grad():
        x = torch.as_tensor(feats).permute(0, 2, 1).unsqueeze(1)
        out = F.relu(_bn(F.conv2d(x, _t(sd, "downsample_layers.0.0.weight", x), padding=1), sd, "downsample_layers.0.1"))
        for i in range(4):
            p = f"downsample_layers.{i + 1}"
            out = _bn(F.conv2d(out, _t(sd, p + ".0.weight", x), stride=(2, STRIDE_T[i]), padding=1), sd, p + ".1")
            for j in range(depths[i]):
                out = _inverted_bottleneck(out, sd, f"stages.{i}.{j}")
        emb = F.linear(tstp(out), _t(sd, "seg_1.weight", x), _t(sd, "seg_1.bias", x))
        if two_emb_layer:
            emb = F.linear(_bn(F.relu(emb), sd, "seg_bn_1", affine=False), _t(sd, "seg_2.weight", x), _t(sd, "seg_2.bias", x))
        return emb


def forward(name, sd, feats, args=None):
    return gemini_forward(sd, feats, syn.GEMINI_NAMES[name], bool((args or {}).get("two_emb_layer", False)))


def parse_case(key):
    name, rest = key.split("__")
    s, b, t, e, w = rest.split("_")
    return name, int(s[1:]), int(b[1:]), int(t[1:]), dict(embed_dim=int(e[1:]), two_emb_layer=bool(int(w[1:])))


def case_inputs(key):
    name, seed, B, T, args = parse_case(key)
    return name, args, syn.make_state_dict(name, seed, **args), syn.make_feats(B, T, 80, seed=seed + 17 * T)


def rel_l2(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.linalg.norm(a - b, axis=-1) / np.linalg.norm(b, axis=-1)


@pytest.mark.parametrize("key", sorted(G))
def test_oracle_matches_reference(key):
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    name, args, sd, feats = case_inputs(key)
    emb = forward(name, sd, feats, args).numpy()
    assert rel_l2(emb, G[key]).max() <= 1e-5, key


def test_param_counts_and_keys():
    # parameters and state_dict keys as the reference modules report them (feat_dim 80, embed_dim 256)
    for name, params, keys in (("Gemini_DF_ResNet60", 4.048, 356), ("Gemini_DF_ResNet114", 6.532, 680),
                               ("Gemini_DF_ResNet183", 9.196, 1094), ("Gemini_DF_ResNet237", 11.680, 1418)):
        spec = syn.state_dict_spec(name, **syn.DEFAULT_MODEL_ARGS[name])
        n = sum(int(np.prod(s)) for k, s in spec.items() if not k.endswith(("running_mean", "running_var", "num_batches_tracked")))
        assert abs(n / 1e6 - params) < 0.001 and len(spec) == keys, (name, n, len(spec))
        assert len(syn.state_dict_spec(name, **dict(syn.DEFAULT_MODEL_ARGS[name], two_emb_layer=True))) == keys + 5


# ------------------------------------------------------------------------------------------ plan builder, no device
@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("prec", ["fp32", "tf32x3", "tf32", "bf16", "fp16"])
def test_plan_check(name, prec):
    ops = from_synthetic(name, precision=prec).plan_check(2, 200)
    labels = [n for n, _ in ops]
    assert labels.count("dwconv3x3") == sum(syn.GEMINI_NAMES[name])
    assert labels[0] == "stem" and labels[-1] == "linear_rows" and labels.count("tstats") == 1


def test_rejects_other_pooling_and_feat_dims():
    from wespeaker_b200 import lib
    with pytest.raises(AssertionError, match="TSTP"):
        get_speaker_model("Gemini_DF_ResNet114")(feat_dim=80, embed_dim=256, pooling_func="ASTP")
    # feat_dim 88 leaves 6 frequency rows after four stride-2 convs; the reference sizes seg_1 for int(88 / 16) = 5
    with pytest.raises(lib.B200Error, match="stats_dim"):
        from_synthetic("Gemini_DF_ResNet60", precision="fp16", feat_dim=88).plan_check(1, 100)
    m = from_synthetic("Gemini_DF_ResNet60", precision="fp16", feat_dim=64, embed_dim=192)
    assert m.feat_dim == 64 and len(m.plan_check(1, 100)) > 0


@pytest.fixture
def interp():
    """the depthwise 3x3 contract lives in plan_interp"""
    return plan_interp


@pytest.mark.parametrize("name,prec,B,T,lens,args", [
    ("Gemini_DF_ResNet60", "fp32", 2, 40, None, {}),
    ("Gemini_DF_ResNet60", "tf32x3", 1, 37, None, {}),
    ("Gemini_DF_ResNet60", "bf16", 1, 48, None, {}),
    ("Gemini_DF_ResNet60", "fp16", 3, 45, [45, 17, 3], {}),   # TSTP needs 2 frames behind the time stride
    ("Gemini_DF_ResNet114", "fp16", 1, 33, None, dict(embed_dim=192, two_emb_layer=True)),
])
def test_plan_arithmetic_matches_oracle_on_the_host(interp, name, prec, B, T, lens, args, tmp_path):
    """The Gemini launch plan (folded BNs, the depthwise op, the strided downsample convs on the halo-resident kernel or the
    conv-GEMM, the identity residual in the project conv's epilogue, TSTP at stride level 1) re-evaluated on the host equals
    the oracle - for the fp32 (FFMA), 3xTF32 and 16-bit plans, and for a length-masked plan whose padding holds large
    garbage.  No device, nothing computed by the library."""
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    m = from_synthetic(name, precision=prec, **args)
    path = str(tmp_path / "plan.bin")
    m.plan_trace(path, B, T, masked=lens is not None)
    feats = syn.make_feats(B, T, 80, seed=5)
    if lens is not None:
        g = np.random.default_rng(1)
        for b in range(B):
            feats[b, lens[b]:] = 50.0 * g.standard_normal((T - lens[b], 80))
    emb, meta = interp.run_plan(path, feats, n_frames=lens)
    kinds = [op["trace"]["kind"] for op in meta["ops"]]
    assert kinds.count("dwconv3x3") == sum(syn.GEMINI_NAMES[name]) and "stem" in kinds
    assert ("conv3x3" in kinds) == (prec in ("bf16", "fp16"))
    sd = syn.make_state_dict(name, 0, **args)
    for b in range(B):
        n = T if lens is None else lens[b]
        ref = forward(name, sd, feats[b:b + 1, :n], args).numpy()[0]
        assert rel_l2(emb[b], ref) <= 2e-5, (prec, b, rel_l2(emb[b], ref))


# ------------------------------------------------------------------------------------------ model surface
def test_reference_constructor_and_config_yaml(tmp_path):
    """`get_speaker_model(name)(**model_args)` with the recipe's arguments, and a model directory whose config.yaml uses them
    loads through speaker.load_model_pt (cli/speaker.py:306-335)."""
    m = get_speaker_model("Gemini_DF_ResNet114")(feat_dim=80, embed_dim=256, pooling_func="TSTP", two_emb_layer=False)
    assert m.feat_dim == 80 and m.embed_dim == 256 and len(m.state_dict()) == 680
    import yaml
    from wespeaker_b200.speaker import load_model_pt
    args = dict(feat_dim=80, embed_dim=192, pooling_func="TSTP", two_emb_layer=True)
    with open(tmp_path / "config.yaml", "w") as f:
        yaml.safe_dump(dict(model="Gemini_DF_ResNet60", model_args=args, dataset_args=dict(frontend="fbank")), f)
    sd = syn.make_state_dict("Gemini_DF_ResNet60", 3, **args)
    torch.save({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}, tmp_path / "avg_model.pt")
    model = load_model_pt(str(tmp_path), precision="fp16")
    assert model.model_name == "Gemini_DF_ResNet60" and model.feat_dim == 80 and model.embed_dim == 192
    assert np.array_equal(model.state_dict()["seg_2.weight"].numpy(), sd["seg_2.weight"])
    assert len(model.plan_check(1, 100)) > 0


# ------------------------------------------------------------------------------------------ GPU
DEV = "cuda:0"
# the default bars hold for all four models, the 77-block Gemini237 included (H100: fp32 6.6e-7, tf32x3 5.8e-5, fp16 5.6e-4,
# bf16 3.8e-3)


def _embed(name, seed, prec, feats, args):
    m = from_synthetic(name, seed, precision=prec, **args)
    out = m(torch.from_numpy(feats).to(DEV))
    assert isinstance(out, tuple) and len(out) == 2   # gemini_dfresnet.py:130-136
    return out[-1].cpu().numpy(), m


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["fp32", "tf32x3"])
@pytest.mark.parametrize("key", sorted(G))
def test_gpu_gemini_fp32_class_paths_match_reference_golden(key, prec):
    name, seed, B, T, args = parse_case(key)
    _, _, _, feats = case_inputs(key)
    emb, m = _embed(name, seed, prec, feats, args)
    rel = rel_l2(emb, G[key])
    print(f"{key} {prec}: rel-L2 max {rel.max():.3e}, launches {m.last_launches()}")
    assert np.isfinite(emb).all() and rel.max() <= 1e-4, (key, prec, rel)
    emb2 = m(torch.from_numpy(feats).to(DEV))[-1].cpu().numpy()      # CUDA-graph replay: bit-identical
    assert np.array_equal(emb, emb2)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["fp16", "bf16"])
@pytest.mark.parametrize("key", sorted(G))
def test_gpu_gemini_16bit_paths_match_reference_golden(key, prec):
    name, seed, B, T, args = parse_case(key)
    _, _, _, feats = case_inputs(key)
    emb, m = _embed(name, seed, prec, feats, args)
    rel = rel_l2(emb, G[key])
    print(f"{key} {prec}: rel-L2 max {rel.max():.3e}, launches {m.last_launches()}")
    assert np.isfinite(emb).all() and rel.max() <= 1e-2, (key, prec, rel)
    emb2 = m(torch.from_numpy(feats).to(DEV))[-1].cpu().numpy()
    assert np.array_equal(emb, emb2)


def _dwconv_operands(dtype, B, Fm, T, C, lens, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.relu(torch.randn(B, Fm, T, C, generator=g) + 0.3) * (0.5 + torch.rand(C, generator=g))
    for b in range(B):
        x[b, :, (lens[b] if lens is not None else T):] = 1e3   # what the expand conv leaves behind an utterance's end
    w = torch.randn(C, 3, 3, generator=g) / 3.0
    shift = 0.3 * torch.randn(C, generator=g)
    return x.to(dtype), w, shift


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("B,Fm,T,C,lens", [
    (2, 40, 200, 128, None),            # stage 1 (dim 32)
    (3, 20, 37, 256, [37, 1, 20]),      # stage 2: a 1-frame utterance, garbage behind the frame counts
    (3, 10, 25, 512, [25, 13, 7]),      # stage 3
    (2, 5, 100, 1024, [100, 64]),       # stage 4
])
def test_gpu_dwconv_kernel_against_fp64(dtype, B, Fm, T, C, lens):
    """ws_dwconv against fp64 on the rounded operands: error within one rounding of the output dtype relative to
    sum |w x| + |shift|; the 3xTF32 low part is exact; rows behind an utterance's end are zeros."""
    import ctypes as C_
    from wespeaker_b200 import lib
    code = {torch.float32: 0, torch.bfloat16: 1, torch.float16: 2}[dtype]
    x, w, shift = _dwconv_operands(dtype, B, Fm, T, C, lens, seed=C + T)
    xd, wd, sd = x.to(DEV).contiguous(), w.to(DEV).contiguous(), shift.to(DEV).contiguous()
    out = torch.full((B, Fm, T, C), 7.0, dtype=dtype, device=DEV)
    out_lo = torch.full((B, Fm, T, C), 7.0, device=DEV) if dtype == torch.float32 else None
    lens_d = torch.tensor(lens, dtype=torch.int32, device=DEV) if lens is not None else None
    d = lib.DwConvDesc()
    d.x, d.x_ld, d.B, d.F, d.T, d.C = xd.data_ptr(), C, B, Fm, T, C
    d.lens = lens_d.data_ptr() if lens_d is not None else None
    d.w, d.shift, d.out, d.out_ld = wd.data_ptr(), sd.data_ptr(), out.data_ptr(), C
    d.out_lo = out_lo.data_ptr() if out_lo is not None else None
    d.dtype = code
    lib.check(lib.load().ws_dwconv(C_.byref(d), None), "ws_dwconv")
    torch.cuda.synchronize()
    o = out.double().cpu()
    if out_lo is not None:
        hi = out.cpu()
        assert torch.equal(out_lo.cpu(), hi - (hi.view(torch.int32) & -8192).view(torch.float32))
    x64 = x.double()
    Tb = lens if lens is not None else [T] * B
    valid = (torch.arange(T)[None, :] < torch.tensor(Tb)[:, None])[:, None, :, None]
    x64 = x64 * valid
    xp = F.pad(x64.permute(0, 3, 1, 2), (1, 1, 1, 1))                  # (B, C, F + 2, T + 2)
    acc = torch.zeros(B, C, Fm, T, dtype=torch.float64)
    mag = torch.zeros(B, C, Fm, T, dtype=torch.float64)
    for jf in range(3):
        for jt in range(3):
            term = xp[:, :, jf:jf + Fm, jt:jt + T] * w.double()[None, :, jf, jt, None, None]
            acc += term
            mag += term.abs()
    ref = (torch.relu(acc + shift.double()[None, :, None, None]).permute(0, 2, 3, 1)) * valid
    mag = mag.permute(0, 2, 3, 1) + shift.double().abs()
    # one rounding of the output dtype (unit roundoff u; fp32: 0) plus the fp32 sum of 10 terms (< 2e-6)
    u = {torch.float32: 0.0, torch.bfloat16: 2 ** -8, torch.float16: 2 ** -11}[dtype]
    err = ((o - ref).abs() / (mag + 1e-30)).max().item()
    print(f"dwconv {dtype} B{B} F{Fm} T{T} C{C} lens {lens}: max error / (sum |w x| + |shift|) {err:.2e}")
    assert err <= u + 2e-6, err
    for b in range(B):   # rows behind an utterance's end are zeros
        assert torch.all(o[b, :, Tb[b]:] == 0)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["fp16", "tf32x3"])
def test_gpu_length_masked_batch_equals_unpadded_utterances(prec):
    """ws_engine_forward_masked: utterances of different lengths padded with large garbage into ONE batch give what each gives
    alone, bit for bit - the depthwise op reads rows behind an utterance's end as zeros, the stage outputs are zeroed there
    before a downsample conv reads them, TSTP runs over each utterance's frames - and match the oracle per utterance."""
    name = "Gemini_DF_ResNet114"
    lens = [200, 137, 163, 101, 301, 64]
    g = torch.Generator().manual_seed(5)
    feats = [torch.from_numpy(syn.make_feats(1, n, 80, seed=40 + i))[0] for i, n in enumerate(lens)]
    x = 50.0 * torch.randn(len(lens), max(lens), 80, generator=g)
    for i, f in enumerate(feats):
        x[i, : lens[i]] = f
    m = from_synthetic(name, 0, precision=prec)
    got = m.embed_padded(x.to(DEV), lens).cpu().numpy()
    sd = syn.make_state_dict(name, 0)
    worst_self, worst_ref, exact = 0.0, 0.0, 0
    for i, f in enumerate(feats):
        alone = m.embed(f[None].to(DEV)).cpu().numpy()[0]
        ref = forward(name, sd, f[None]).numpy()[0]
        exact += int(np.array_equal(got[i], alone))
        worst_self = max(worst_self, float(rel_l2(got[i], alone)))
        worst_ref = max(worst_ref, float(rel_l2(got[i], ref)))
    print(f"masked batch {name} {prec}: vs alone {worst_self:.2e} ({exact}/{len(lens)} bit-identical), vs oracle {worst_ref:.2e}")
    assert np.isfinite(got).all() and exact == len(lens), worst_self
    assert worst_ref <= (1e-4 if prec == "tf32x3" else 1e-2)


@pytest.mark.gpu
def test_gpu_batch_of_64_fp16_matches_oracle():
    name = "Gemini_DF_ResNet114"
    feats = syn.make_feats(64, 200, 80, seed=31)
    emb, m = _embed(name, 0, "fp16", feats, {})
    sel = [0, 21, 63]
    ref = forward(name, syn.make_state_dict(name, 0), feats[sel]).numpy()
    rel = rel_l2(emb[sel], ref)
    print(f"{name} fp16 B64 T200: rel-L2 vs oracle {rel.max():.3e}, launches {m.last_launches()}")
    assert np.isfinite(emb).all() and rel.max() <= 1e-2


@pytest.mark.gpu
def test_gpu_ragged_wav_extraction():
    """extract_from_wav_list_ragged (length-masked buckets over concatenated PCM) equals per-utterance extraction."""
    m = from_synthetic("Gemini_DF_ResNet114", 0, precision="fp16")
    ns = [16000, 23456, 40000, 8000, 31234]
    wavs = [torch.from_numpy(syn.make_wavs(1, n, seed=60 + i))[0] for i, n in enumerate(ns)]
    got = m.extract_from_wav_list_ragged(wavs).cpu().numpy()
    alone = np.stack([m.extract_from_wav(w[None].to(DEV)).cpu().numpy()[0] for w in wavs])
    rel = rel_l2(got, alone)
    print(f"ragged Gemini114 fp16: rel-L2 vs per-utterance extraction {rel.max():.2e}")
    assert got.shape == (len(ns), 256) and np.isfinite(got).all() and rel.max() <= 1e-5
