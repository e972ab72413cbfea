"""8 kHz and any-bin-count fbank (the SRE recipes' front end: `examples/sre/v2|v3/conf/resnet.yaml`, `resample_rate: 8000`
with 40 / 64 bins, and the CLI's `set_resample_rate(8000)` with 80 bins).  Goldens: tests/golden/make_golden_fbank_rates.py
(torchaudio kaldi.fbank / Resample, the reference's ResNet34 and its compiled SpeakerEngine::ExtractFeature).

CPU tests pin the oracle and the refusals; GPU tests hold the kernel to the bars of test_fbank_matches_torchaudio_golden."""
import ctypes as C
import os
import sys

import numpy as np
import pytest
import torch
import yaml

from oracle import fbank_np, models_torch, resample_np
from wespeaker_b200 import extract, frontend, lib, synthetic as syn
from wespeaker_b200.models import from_synthetic
from wespeaker_b200.speaker_engine import SpeakerEngine, chunk_frame_index

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_fbank_rates as mg  # noqa: E402  (the seeded inputs of the goldens)

G = np.load(os.path.join(HERE, "golden", "fbank_rates.npz"))
CASES = [(r, b, w) for r in mg.RATES for b in mg.BINS for w in mg.WINDOWS]
# the sre/v2 and sre/v3 dataset_args (examples/sre/v2|v3/conf/resnet.yaml)
SRE_V2 = {"resample_rate": 8000, "fbank_args": {"num_mel_bins": 40, "frame_shift": 10, "frame_length": 25, "dither": 1.0}}
SRE_V3 = {"resample_rate": 8000, "fbank_args": {"num_mel_bins": 64, "frame_shift": 10, "frame_length": 25, "dither": 1.0}}


def rel_l2(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.linalg.norm(a - b, axis=-1) / np.linalg.norm(b, axis=-1)


# ------------------------------------------------------------------------------------------ CPU: oracle and refusals
@pytest.mark.parametrize("rate,bins,wt", CASES)
def test_fbank_oracle_matches_torchaudio_at_rate(rate, bins, wt):
    ref = G[f"fbank_{rate}_{bins}_{wt}"]
    for w, r in zip(mg.wavs_for(rate, wt), ref):
        out = fbank_np.fbank(w, num_mel_bins=bins, sample_frequency=rate, window_type=wt)
        assert out.shape == r.shape
        assert np.abs(out - r).max() < 2e-3 and np.abs(out - r).mean() < 2e-5


def test_fbank_oracle_short_resampled_and_geometry():
    short, one = mg.short_wavs()
    assert np.abs(fbank_np.fbank(short, 64, sample_frequency=8000) - G["fbank_8000_64_short"]).max() < 2e-3
    assert np.abs(fbank_np.fbank(one, 40, sample_frequency=8000) - G["fbank_8000_40_one"]).max() < 2e-3
    assert fbank_np.fbank(one[:199], 40, sample_frequency=8000).shape == (0, 40)
    _, w16k = mg.model_wavs()
    r = resample_np.resample(w16k[None], 16000, 8000)[0]
    assert np.abs(r - G["resampled_16000_8000"]).max() < 1e-2 * max(1.0, np.abs(G["resampled_16000_8000"]).max() / 3e3)
    assert np.abs(fbank_np.fbank(G["resampled_16000_8000"], 64, sample_frequency=8000) - G["fbank_resampled_8000_64"]).max() < 2e-3
    assert frontend.frame_geometry(8000) == (200, 80) and frontend.frame_geometry(16000) == (400, 160)


@pytest.mark.parametrize("bins", [40, 64])
def test_resnet34_oracle_matches_reference_at_feat_dim(bins):
    sd = syn.make_state_dict("ResNet34", 0, feat_dim=bins)
    out = models_torch.forward("ResNet34", sd, torch.from_numpy(G[f"resnet34_fd{bins}_feats"])).numpy()
    assert rel_l2(out, G[f"resnet34_fd{bins}_emb"]).max() < 1e-5


def test_speaker_engine_oracle_at_8k_64_pinned_on_compiled_reference():
    """fbank_np at 8 kHz / 64 bins against the reference's native fbank (SpeakerEngine::ExtractFeature, 2 s chunks at 8 kHz
    = 198 frames, ApplyMean per chunk), through the chunk index of speaker_engine.py."""
    pcm = mg.engine_pcm().astype(np.float32)
    full = fbank_np.fbank(pcm, 64, sample_frequency=8000, window_type="hamming")
    want = G["engine_8000_64_chunks_cmn"]
    eng = SpeakerEngine(model=None, feat_dim=64, sample_rate=8000, samples_per_chunk=16000, fbank_fn=lambda w: None)
    assert eng.num_chunk_frames() == want.shape[1] == 198
    chunks = full[chunk_frame_index(full.shape[0], 198)]
    got = chunks - chunks.mean(axis=1, keepdims=True)
    assert got.shape == want.shape
    d = np.abs(got - want)
    assert d.max() < 5e-3 and d.mean() < 5e-5


@pytest.mark.parametrize("bins", [40, 64])
@pytest.mark.parametrize("frames", [200, 1000])
def test_plan_check_resnet34_at_sre_feat_dims(bins, frames):
    m = from_synthetic("ResNet34", 0, precision="fp16", feat_dim=bins)
    ops = m.plan_check(batch=64, frames=frames)
    assert len(ops) > 10


def test_extract_frontend_args_accepts_sre_configs():
    assert extract.frontend_args(SRE_V2, 40) == (8000, 40)
    assert extract.frontend_args(SRE_V3, 64) == (8000, 64)
    assert extract.frontend_args({}, 80) == (16000, 80)
    assert extract.frontend_args({"resample_rate": 8000}, 64) == (8000, 64)


@pytest.mark.parametrize("dataset_args,err,match", [
    (dict(SRE_V3, resample_rate=11025), NotImplementedError, "11025"),
    (dict(SRE_V3, fbank_args={"num_mel_bins": 100}), ValueError, "num_mel_bins = 100 does not match the model's feat_dim = 64"),
    (dict(SRE_V3, fbank_args={"num_mel_bins": 64, "frame_length": 20}), NotImplementedError, "frame_length"),
])
def test_extract_refuses_unsupported_frontend(dataset_args, err, match, tmp_path):
    cfg = {"model": "ResNet34", "model_args": dict(syn.DEFAULT_MODEL_ARGS["ResNet34"], feat_dim=64),
           "model_path": str(tmp_path / "missing.pt"), "embed_ark": str(tmp_path / "x.ark"),
           "data_list": str(tmp_path / "missing.list"), "dataset_args": dataset_args}
    path = tmp_path / "config.yaml"
    path.write_text(yaml.safe_dump(cfg))
    with pytest.raises(err, match=match):
        extract.extract(str(path))


def test_c_abi_refuses_bad_rates_and_bins():
    L = lib.load()
    assert L.ws_fbank_num_frames_at(16000, 8000) == 198 and L.ws_fbank_num_frames_at(199, 8000) == 0
    assert L.ws_fbank_num_frames_at(200, 8000) == 1 and L.ws_fbank_num_frames_at(32000, 16000) == L.ws_fbank_num_frames(32000)
    assert L.ws_fbank_num_frames_at(16000, 11025) == -1
    # refused before any device is touched: the pointers are never dereferenced
    fake = C.c_void_p(16)

    def fbank_at(rate, bins, n=16000):
        return L.ws_fbank_at(fake, 0, n, n, 1, b"hamming", rate, bins, 1, fake, None)
    for rate, bins, n, msg in ((11025, 64, 16000, b"sample rate"), (8000, 3, 16000, b"num_mel_bins"),
                               (8000, 129, 16000, b"num_mel_bins"), (8000, 64, 199, b"shorter than one")):
        assert fbank_at(rate, bins, n) != 0
        assert msg in L.ws_last_error()
    assert L.ws_fbank_ragged_at(fake, 0, 100, fake, fake, 1, 1, b"hamming", 22050, 64, fake, None) != 0
    assert b"sample rate" in L.ws_last_error()
    assert L.ws_fbank_ragged_at(fake, 0, 100, fake, fake, 1, 1, b"hamming", 8000, 200, fake, None) != 0
    # the engine option: only 8000 / 16000
    h = lib.c_engine_p()
    lib.check(L.ws_engine_create_plan_check(b"ResNet34", b"fp16", 64, 256, C.byref(h)), "create")
    try:
        assert L.ws_engine_set_option(h, b"sample_rate", 8000) == 0
        assert L.ws_engine_set_option(h, b"sample_rate", 11025) != 0 and b"sample_rate" in L.ws_last_error()
    finally:
        L.ws_engine_destroy(h)
    with pytest.raises(NotImplementedError):
        frontend.check_rate_bins(44100)
    with pytest.raises(NotImplementedError):
        SpeakerEngine(model=None, feat_dim=200, sample_rate=8000)


# ------------------------------------------------------------------------------------------ GPU
DEV = "cuda:0"


@pytest.mark.gpu
@pytest.mark.parametrize("rate,bins,wt", CASES)
def test_fbank_kernel_matches_torchaudio_at_rate(rate, bins, wt):
    wavs = torch.from_numpy(mg.wavs_for(rate, wt)).to(DEV)
    out = frontend.fbank_batch(wavs, window_type=wt, sample_rate=rate, num_mel_bins=bins).cpu().numpy()
    ref = G[f"fbank_{rate}_{bins}_{wt}"]
    d = np.abs(out - ref)
    print(f"fbank {rate} Hz {bins} bins {wt}: max {d.max():.3e} mean {d.mean():.3e}")
    assert out.shape == ref.shape and d.max() < 2e-3 and d.mean() < 5e-5
    out16 = frontend.fbank_batch(wavs.to(torch.int16), window_type=wt, sample_rate=rate, num_mel_bins=bins).cpu().numpy()
    assert np.array_equal(out16, out)


@pytest.mark.gpu
def test_fbank_kernel_short_one_frame_and_resampled():
    short, one = mg.short_wavs()
    out = frontend.fbank(torch.from_numpy(short).to(DEV), num_mel_bins=64, sample_frequency=8000, window_type="hamming")
    assert out.shape == (98, 64) and np.abs(out.cpu().numpy() - G["fbank_8000_64_short"]).max() < 2e-3
    o1 = frontend.fbank_batch(torch.from_numpy(one[None]).to(DEV), sample_rate=8000, num_mel_bins=40).cpu().numpy()
    assert o1.shape == (1, 1, 40) and np.abs(o1[0] - G["fbank_8000_40_one"]).max() < 2e-3
    assert frontend.fbank_batch(torch.zeros(2, 199, device=DEV), sample_rate=8000, num_mel_bins=40).shape == (2, 0, 40)
    _, w16k = mg.model_wavs()
    r = frontend.resample(torch.from_numpy(w16k).to(DEV), 16000, 8000)
    fr = frontend.fbank_batch(r[None], sample_rate=8000, num_mel_bins=64).cpu().numpy()[0]
    assert np.abs(fr - G["fbank_resampled_8000_64"]).max() < 2e-2 and np.abs(fr - G["fbank_resampled_8000_64"]).mean() < 5e-4
    # odd sample counts with B > 1 (rows start at odd offsets: paired-sample loads fall back to scalar loads)
    wo = syn.make_wavs(3, 8077, seed=6)
    fo = frontend.fbank_batch(torch.from_numpy(wo).to(DEV), sample_rate=8000, num_mel_bins=64).cpu().numpy()
    for i in range(3):
        assert np.abs(fo[i] - fbank_np.fbank(wo[i], 64, sample_frequency=8000)).max() < 2e-3


@pytest.mark.gpu
def test_ragged_fbank_at_8k_equals_each_row_alone():
    L = lib.load()
    ns = [8000, 1234, 200, 16077, 999]
    wavs = [syn.make_wavs(1, n, seed=30 + i)[0] for i, n in enumerate(ns)]
    flat = torch.from_numpy(np.concatenate(wavs)).to(DEV)
    offs = torch.from_numpy(np.concatenate([[0], np.cumsum(ns)[:-1]]).astype(np.int64)).to(DEV)
    nf = [frontend.num_frames(n, 8000) for n in ns]
    nfd = torch.tensor(nf, dtype=torch.int32, device=DEV)
    T = max(nf)
    out = torch.full((len(ns), T, 64), -7.0, device=DEV)
    lib.check(L.ws_fbank_ragged_at(flat.data_ptr(), 0, flat.numel(), offs.data_ptr(), nfd.data_ptr(), T, len(ns), b"hamming",
                                   8000, 64, out.data_ptr(), lib.cur_stream_ptr(0)), "ws_fbank_ragged_at")
    out = out.cpu().numpy()
    for i, w in enumerate(wavs):
        alone = frontend.fbank_batch(torch.from_numpy(w[None]).to(DEV), sample_rate=8000, num_mel_bins=64).cpu().numpy()[0]
        assert np.array_equal(out[i, :nf[i]], alone)
        assert (out[i, nf[i]:] == -7.0).all()          # rows behind the end are not written


@pytest.mark.gpu
def test_16k_80_new_entry_points_equal_old_bit_for_bit():
    L = lib.load()
    w = torch.from_numpy(syn.make_wavs(4, 32077, seed=9)).to(DEV)
    st = lib.cur_stream_ptr(0)
    T = frontend.num_frames(w.shape[1])
    for wt in mg.WINDOWS:
        for cmn in (0, 1):
            a = torch.empty((4, T, 80), device=DEV)
            b = torch.empty_like(a)
            lib.check(L.ws_fbank(w.data_ptr(), 0, w.shape[1], w.shape[1], 4, wt.encode(), cmn, a.data_ptr(), st), "ws_fbank")
            lib.check(L.ws_fbank_at(w.data_ptr(), 0, w.shape[1], w.shape[1], 4, wt.encode(), 16000, 80, cmn, b.data_ptr(), st),
                      "ws_fbank_at")
            assert torch.equal(a, b)
    flat = w.reshape(-1)
    offs = torch.tensor([0, 32077, 64154 + 3], dtype=torch.int64, device=DEV)
    nfd = torch.tensor([199, 150, 12], dtype=torch.int32, device=DEV)
    a = torch.zeros((3, 199, 80), device=DEV)
    b = torch.zeros_like(a)
    lib.check(L.ws_fbank_ragged(flat.data_ptr(), 0, flat.numel(), offs.data_ptr(), nfd.data_ptr(), 199, 3, b"hamming", a.data_ptr(),
                                st), "ws_fbank_ragged")
    lib.check(L.ws_fbank_ragged_at(flat.data_ptr(), 0, flat.numel(), offs.data_ptr(), nfd.data_ptr(), 199, 3, b"hamming", 16000,
                                   80, b.data_ptr(), st), "ws_fbank_ragged_at")
    assert torch.equal(a, b)
    m = from_synthetic("ResNet34", 0, precision="fp16")
    e_default, f_default = m.extract_from_wav(w, return_feats=True)
    e_16k, f_16k = m.extract_from_wav(w, return_feats=True, sample_rate=16000)
    assert torch.equal(f_default, f_16k) and torch.equal(e_default, e_16k)


BARS = {"fp32": 1e-4, "tf32x3": 1e-4, "bf16": 1e-2, "fp16": 1e-2}


@pytest.mark.gpu
@pytest.mark.parametrize("bins", [40, 64])
@pytest.mark.parametrize("prec", ["fp32", "tf32x3", "bf16", "fp16"])
def test_extract_from_wav_8k_resnet34(bins, prec):
    wavs, _ = mg.model_wavs()
    m = from_synthetic("ResNet34", 0, precision=prec, feat_dim=bins)
    emb, feats = m.extract_from_wav(torch.from_numpy(wavs).to(DEV), return_feats=True, sample_rate=8000)
    assert feats.shape == (2, 198, bins)
    sd = syn.make_state_dict("ResNet34", 0, feat_dim=bins)
    ref = models_torch.forward("ResNet34", sd, feats.cpu()).numpy()
    rel = rel_l2(emb.cpu().numpy(), ref)
    print(f"ResNet34 feat_dim {bins} {prec} at 8 kHz: rel {rel.max():.2e}")
    assert rel.max() <= BARS[prec]
    # the features are the CMN'd fbank of the golden's waveforms (torchaudio-level agreement)
    assert np.abs(feats.cpu().numpy() - G[f"resnet34_fd{bins}_feats"]).max() < 2e-3
    # host input takes the same path
    eh = m.extract_from_wav(torch.from_numpy(wavs), sample_rate=8000)
    assert torch.equal(eh, emb.cpu())


@pytest.mark.gpu
def test_masked_and_ragged_8k_batches_equal_each_utterance_alone():
    m = from_synthetic("ResNet34", 0, precision="fp32", feat_dim=64)
    ns = [16000, 12345, 9001, 4000]
    wavs = [torch.from_numpy(syn.make_wavs(1, n, seed=40 + i)[0]) for i, n in enumerate(ns)]
    alone = torch.cat([m.extract_from_wav(w[None].to(DEV), sample_rate=8000) for w in wavs]).cpu().numpy()
    pad = torch.zeros((len(ns), max(ns)))
    for i, w in enumerate(wavs):
        pad[i, :ns[i]] = w
    masked = m.extract_from_wav_padded(pad.to(DEV), ns, sample_rate=8000).cpu().numpy()
    ragged = m.extract_from_wav_list_ragged(wavs, sample_rate=8000, device=DEV).cpu().numpy()
    bucketed = m.extract_from_wav_list(wavs, sample_rate=8000, device=DEV).cpu().numpy()
    print(f"8 kHz masked vs alone {rel_l2(masked, alone).max():.2e}, ragged {rel_l2(ragged, alone).max():.2e}")
    assert rel_l2(masked, alone).max() < 1e-5 and rel_l2(ragged, alone).max() < 1e-5
    assert np.array_equal(bucketed, alone)
    streamed = np.concatenate([e.numpy() for e in m.extract_stream([wavs[0][None], wavs[1][None]], sample_rate=8000)])
    assert np.array_equal(streamed, alone[:2])


def _write_wav(path, pcm, sr):
    import wave
    with wave.open(str(path), "wb") as f:
        f.setnchannels(1)
        f.setsampwidth(2)
        f.setframerate(sr)
        f.writeframes(np.asarray(pcm, dtype="<i2").tobytes())


@pytest.mark.gpu
def test_extract_sre_v3_raw_list_mixing_8k_and_16k(tmp_path):
    from wespeaker_b200.kaldi_io import read_vec_scp_file
    name, prec = "ResNet34", "fp32"
    args = dict(syn.DEFAULT_MODEL_ARGS[name], feat_dim=64)
    sd = syn.make_state_dict(name, 0, **args)
    torch.save({k: torch.from_numpy(np.asarray(v)) for k, v in sd.items()}, tmp_path / "model.pt")
    utts = [("a8k", 8000, 12000), ("b16k", 16000, 30000), ("c8k", 8000, 12000), ("d16k", 16000, 23000)]
    lines = []
    pcms = {}
    for i, (key, sr, n) in enumerate(utts):
        pcm = syn.make_wavs(1, n, seed=60 + i)[0].astype(np.int16)
        _write_wav(tmp_path / f"{key}.wav", pcm, sr)
        pcms[key] = (pcm, sr)
        lines.append(f'{{"key": "{key}", "wav": "{tmp_path / (key + ".wav")}", "spk": "s"}}')
    (tmp_path / "data.list").write_text("\n".join(lines) + "\n")
    cfg = {"model": name, "model_args": args, "model_path": str(tmp_path / "model.pt"), "precision": prec,
           "embed_ark": str(tmp_path / "out" / "emb.ark"), "data_list": str(tmp_path / "data.list"), "data_type": "raw",
           "batch_size": 1, "dataset_args": SRE_V3}
    (tmp_path / "config.yaml").write_text(yaml.safe_dump(cfg))
    assert extract.extract(str(tmp_path / "config.yaml")) == len(utts)
    got = read_vec_scp_file(str(tmp_path / "out" / "emb.scp"))
    for key, (pcm, sr) in pcms.items():
        x = pcm.astype(np.float32)
        if sr != 8000:
            x = resample_np.resample(x[None], sr, 8000)[0]
        feats = fbank_np.cmn(fbank_np.fbank(x, 64, sample_frequency=8000))
        ref = models_torch.forward(name, sd, torch.from_numpy(feats)[None]).numpy()[0]
        rel = rel_l2(got[key], ref)
        print(f"extract sre/v3 {key}: rel {rel:.2e}")
        assert rel < 1e-3


@pytest.mark.gpu
def test_speaker_set_resample_rate_8000(tmp_path):
    from wespeaker_b200.speaker import Speaker
    name = "ResNet34"
    m = from_synthetic(name, 0, precision="fp32")
    spk = Speaker(model=m)
    spk.set_resample_rate(8000)
    pcm = syn.make_wavs(1, 24000, seed=70)[0].astype(np.int16)
    _write_wav(tmp_path / "x.wav", pcm, 16000)
    emb = spk.extract_embedding(str(tmp_path / "x.wav")).numpy()
    x = resample_np.resample(pcm.astype(np.float32)[None], 16000, 8000)[0]
    ref = models_torch.forward(name, syn.make_state_dict(name, 0), torch.from_numpy(fbank_np.cmn(fbank_np.fbank(x, 80, sample_frequency=8000)))[None]).numpy()[0]
    rel = rel_l2(emb, ref)
    print(f"Speaker.set_resample_rate(8000): rel {rel:.2e}")
    assert rel < 1e-3
    f = spk.compute_features(torch.from_numpy(x[None]), sample_rate=8000).cpu().numpy()
    assert f.shape == (1, frontend.num_frames(x.shape[0], 8000), 80)
    assert np.abs(f[0] - fbank_np.cmn(fbank_np.fbank(x, 80, sample_frequency=8000))).max() < 2e-3
    with pytest.raises(NotImplementedError):
        spk.set_resample_rate(22050)


@pytest.mark.gpu
def test_speaker_engine_8k_64_matches_compiled_reference():
    """SpeakerEngine(model, 64, 8000, samples_per_chunk=16000) on the device against the reference's own compiled
    SpeakerEngine::ExtractFeature (+ ApplyMean per chunk) on the same int16 PCM, stored by make_golden_fbank_rates.py."""
    pcm = mg.engine_pcm()
    m = from_synthetic("ResNet34", 0, precision="fp32", feat_dim=64)
    full = SpeakerEngine(m, feat_dim=64, sample_rate=8000, samples_per_chunk=0).extract_feature(torch.from_numpy(pcm))
    want_full = G["engine_8000_64_full"]
    assert tuple(full.shape) == (1,) + want_full.shape
    d = np.abs(full[0].cpu().numpy() - want_full)
    print(f"SpeakerEngine 8 kHz / 64 full mode vs compiled reference: max {d.max():.2e} mean {d.mean():.2e}")
    assert d.max() < 5e-3 and d.mean() < 5e-5
    eng = SpeakerEngine(m, feat_dim=64, sample_rate=8000, samples_per_chunk=16000)
    chunks = eng.extract_feature(torch.from_numpy(pcm))
    got = (chunks - chunks.mean(dim=1, keepdim=True)).cpu().numpy()     # ApplyMean per chunk, as ExtractEmbedding does
    want = G["engine_8000_64_chunks_cmn"]
    assert got.shape == want.shape
    d = np.abs(got - want)
    print(f"SpeakerEngine 8 kHz / 64 chunks vs compiled reference: max {d.max():.2e} mean {d.mean():.2e}")
    assert d.max() < 5e-3 and d.mean() < 5e-5
    emb = eng.extract_embedding(pcm)
    ref = models_torch.forward("ResNet34", syn.make_state_dict("ResNet34", 0, feat_dim=64), torch.from_numpy(want)).numpy().mean(0)
    assert rel_l2(emb, ref) < 1e-3
