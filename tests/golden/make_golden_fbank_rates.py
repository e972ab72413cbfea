#!/usr/bin/env python
"""Goldens for the 8 kHz / any-bin-count frontend (run in the build container only):

    WESPEAKER_REFERENCE=<wespeaker checkout> PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_fbank_rates.py

* ``torchaudio.compliance.kaldi.fbank`` at 8 and 16 kHz x {40, 64, 80} bins x the four window types, plus a short 8 kHz
  utterance and an exactly-one-frame one;
* ``torchaudio.transforms.Resample(16000, 8000)`` followed by fbank (the SRE recipes' ``resample_rate: 8000``);
* the reference's ``resnet.py`` ``ResNet34(feat_dim=40 / 64)`` on the seeded synthetic weights and CMN'd 8 kHz features;
* ``SpeakerEngine::ExtractFeature`` at 8 kHz / 64 bins (the reference's own C++ fbank and chunking, compiled here from the
  checkout with ``ref_engine_rates_wrap.cc``), in full mode and in 2 s chunk mode after ``ApplyMean``.

Inputs are regenerated from seeds at test time (``wavs_for``); only outputs are stored, in tests/golden/fbank_rates.npz."""
import ctypes as C
import os
import subprocess
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

RATES = (8000, 16000)
BINS = (40, 64, 80)
WINDOWS = ("hamming", "povey", "hanning", "rectangular")


def wavs_for(rate, window):
    """The seeded waveforms of one (rate, window) case: 0.6 s each, two of them for hamming, one otherwise."""
    from wespeaker_b200 import synthetic as syn
    return syn.make_wavs(2 if window == "hamming" else 1, rate * 6 // 10, seed=rate // 1000 + WINDOWS.index(window))


def short_wavs():
    """An 8 kHz utterance of 1 s + 37 samples, and one of exactly one 200-sample frame."""
    from wespeaker_b200 import synthetic as syn
    return syn.make_wavs(1, 8037, seed=5)[0], syn.make_wavs(1, 200, seed=1)[0]


def model_wavs():
    """Two 2 s utterances at 8 kHz (the ResNet34 feat_dim 40 / 64 cases) and one 1 s utterance at 16 kHz (resampled)."""
    from wespeaker_b200 import synthetic as syn
    return syn.make_wavs(2, 16000, seed=21), syn.make_wavs(1, 16000, seed=22)[0]


def engine_pcm():
    """The int16 recording of the SpeakerEngine case: 40333 samples at 8 kHz (two full 2 s chunks and a padded third)."""
    from wespeaker_b200 import synthetic as syn
    return syn.make_wavs(1, 40333, seed=7)[0].astype(np.int16)


def load_ref_rates(reference_dir, out_dir):
    """Compile ref_engine_rates_wrap.cc with the reference's speaker_engine.cc / feature_pipeline.cc / fft.cc (the sources
    oracle/Makefile uses) into out_dir and load it."""
    core = os.path.join(reference_dir, "runtime", "core")
    so = os.path.join(out_dir, "libref_engine_rates.so")
    srcs = [os.path.join(core, "speaker", "speaker_engine.cc"), os.path.join(core, "frontend", "feature_pipeline.cc"),
            os.path.join(core, "frontend", "fft.cc"), os.path.join(HERE, "ref_engine_rates_wrap.cc")]
    subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-I" + os.path.join(ROOT, "oracle", "ref_shim"), "-I" + core,
                    "-o", so] + srcs + ["-lpthread"], check=True)
    L = C.CDLL(so)
    L.ref_extract_feature_at.restype = C.c_int
    L.ref_extract_feature_at.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                         C.POINTER(C.POINTER(C.c_float)), C.POINTER(C.c_int)]
    L.ref_rates_free.argtypes = [C.POINTER(C.c_float)]
    return L


def ref_features(L, pcm_i16, samples_per_chunk, apply_mean, rate, bins):
    out, shape = C.POINTER(C.c_float)(), (C.c_int * 3)()
    pcm = np.ascontiguousarray(pcm_i16, dtype=np.int16)
    nc = L.ref_extract_feature_at(pcm.ctypes.data, len(pcm), samples_per_chunk, apply_mean, rate, bins, C.byref(out), shape)
    assert nc >= 0
    a = np.ctypeslib.as_array(out, shape=(max(1, shape[0]) * max(1, shape[1]) * max(1, shape[2]),)).copy()
    L.ref_rates_free(out)
    return a[: shape[0] * shape[1] * shape[2]].reshape(shape[0], shape[1], shape[2])


def main():
    import torchaudio
    import torchaudio.compliance.kaldi as kaldi
    from make_golden import _import_reference
    from wespeaker_b200 import synthetic as syn

    def fb(w, rate, bins, wt="hamming"):
        return kaldi.fbank(torch.from_numpy(np.asarray(w, np.float32))[None], num_mel_bins=bins, frame_length=25,
                           frame_shift=10, dither=0.0, sample_frequency=rate, window_type=wt, use_energy=False).numpy()

    out = {}
    for rate in RATES:
        for wt in WINDOWS:
            wavs = wavs_for(rate, wt)
            for bins in BINS:
                out[f"fbank_{rate}_{bins}_{wt}"] = np.stack([fb(w, rate, bins, wt) for w in wavs])
    short, one = short_wavs()
    out["fbank_8000_64_short"] = fb(short, 8000, 64)
    out["fbank_8000_40_one"] = fb(one, 8000, 40)

    m8k, w16k = model_wavs()
    r = torchaudio.transforms.Resample(orig_freq=16000, new_freq=8000)(torch.from_numpy(w16k)[None].float())[0].numpy()
    out["resampled_16000_8000"] = r
    out["fbank_resampled_8000_64"] = fb(r, 8000, 64)

    _, resnet, _, du, _, _ = _import_reference()
    for bins in (40, 64):
        feats = du.apply_cmvn(torch.from_numpy(np.stack([fb(w, 8000, bins) for w in m8k])))
        args = dict(syn.DEFAULT_MODEL_ARGS["ResNet34"], feat_dim=bins)
        model = resnet.ResNet34(**args)
        sd = {k: torch.from_numpy(np.asarray(v)) for k, v in syn.make_state_dict("ResNet34", 0, **args).items()}
        model.load_state_dict(sd, strict=True)
        model.eval()
        with torch.no_grad():
            o = model(feats)
        out[f"resnet34_fd{bins}_feats"] = feats.numpy()
        out[f"resnet34_fd{bins}_emb"] = (o[-1] if isinstance(o, tuple) else o).numpy().astype(np.float32)

    with tempfile.TemporaryDirectory() as tmp:
        L = load_ref_rates(os.environ["WESPEAKER_REFERENCE"], tmp)
        pcm = engine_pcm()
        out["engine_8000_64_full"] = ref_features(L, pcm, 0, 0, 8000, 64)[0]
        out["engine_8000_64_chunks_cmn"] = ref_features(L, pcm, 16000, 1, 8000, 64)

    np.savez_compressed(os.path.join(HERE, "fbank_rates.npz"), **out)
    print({k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
