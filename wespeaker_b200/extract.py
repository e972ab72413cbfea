"""`extract(config, **kwargs)` — drop-in for `wespeaker/bin/extract.py:33-139` (seam B2, SURVEY.md §8b).

Reads the reference YAML keys (``model``, ``model_args``, ``dataset_args``), loads ``model_path`` with ``load_checkpoint``,
extracts embeddings and writes Kaldi ``ark,scp`` (scp path = ark path with ``.scp``).  Data lists are the reference's:

* ``raw``   JSON lines ``{key, wav, spk[, vad]}`` (`dataset/processor.py:112-166`; ``wav`` may be a ``cmd |`` pipe),
* ``shard`` a list of tar files whose members ``<key>.wav`` / ``<key>.spk`` are grouped by prefix (`processor.py:68-109`),
* ``feat``  JSON lines ``{key, feat, spk}`` with ``feat`` a Kaldi ``ark:offset`` matrix location (`processor.py:169-196`).

Like the reference, ``batch_size == 1`` extracts WHOLE utterances and ``batch_size > 1`` extracts one fixed-length chunk of
``num_frms`` frames per utterance (`dataset/dataset.py:213-242`, `processor.py:315-347`: random start, short utterances are
tiled) — that is what makes batches rectangular there.  What changes is where the work runs: the reference computes fbank in
DataLoader worker processes on the CPU and ships features to the GPU (`extract.py:99-134`); here a pool of reader threads
only decodes PCM, batches go through ``B200SpeakerModel.extract_stream`` (pinned int16 H2D of batch i+1 overlapping fbank +
CMN + forward of batch i on the device), and whole utterances of equal length are batched together.
Audio at another sample rate is resampled to ``resample_rate`` (16000, or 8000 as in the SRE recipes) on the device
(``frontend.resample`` = torchaudio's sinc resampler, `processor.py:242-262`).  The augmentation pipeline (``reverb_data`` / ``noise_data`` / ``aug_prob``),
``speed_perturb`` and SSL frontends are training-side features outside SURVEY.md section 8: requesting them raises.
"""
from __future__ import annotations

import io
import json
import os
import random
import subprocess
import tarfile
import wave
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch
import yaml

from . import frontend
from .kaldi_io import VectorWriter, load_mat
from .models import get_speaker_model, load_checkpoint

AUDIO_FORMAT_SETS = {"flac", "mp3", "m4a", "ogg", "opus", "wav", "wma"}   # processor.py:32


def parse_config_or_kwargs(config_file, **kwargs):
    """`wespeaker/utils/utils.py:37-51`: yaml dict overridden by kwargs."""
    with open(config_file) as f:
        cfg = yaml.load(f, Loader=yaml.FullLoader)
    return dict(cfg, **kwargs)


def _decode_wav_bytes(buf: bytes):
    """PCM16 WAV bytes -> (int16 (N,) first channel, sample_rate)."""
    with wave.open(io.BytesIO(buf), "rb") as w:
        if w.getsampwidth() != 2:
            raise ValueError("only 16-bit PCM WAV is supported")
        sr, ch, n = w.getframerate(), w.getnchannels(), w.getnframes()
        data = np.frombuffer(w.readframes(n), dtype="<i2").reshape(-1, ch)
    return np.ascontiguousarray(data[:, 0]), sr


def _read_audio(wav: str):
    """`processor.py:124-131`: a path, or a shell pipeline ending in '|' whose stdout is the audio file."""
    if wav.endswith("|"):
        return _decode_wav_bytes(subprocess.run(wav[:-1], shell=True, stdout=subprocess.PIPE, check=True).stdout)
    with open(wav, "rb") as f:
        return _decode_wav_bytes(f.read())


def _apply_vad(pcm, sr, vad):
    """`processor.py:133-141`: keep the listed [start, end] second ranges."""
    return np.concatenate([pcm[int(float(a) * sr):int(float(b) * sr)] for a, b in vad])


def get_random_chunk(data: np.ndarray, chunk_len: int, rng: random.Random) -> np.ndarray:
    """`processor.py:315-347`: random window of chunk_len; shorter inputs are tiled, then cut."""
    n = len(data)
    if n >= chunk_len:
        s = rng.randint(0, n - chunk_len)
        return data[s:s + chunk_len].copy()
    rep = chunk_len // n + 1
    return np.tile(data, rep if data.ndim == 1 else (rep, 1))[:chunk_len]


def frontend_args(test_conf: dict, feat_dim: int):
    """(resample_rate, num_mel_bins) of the ``dataset_args`` the fused wav path computes: fbank at 8 or 16 kHz, 25 ms frames
    every 10 ms, ``fbank_args.num_mel_bins`` equal to the model's feat_dim (the reference would fail in the forward pass on
    any other count)."""
    resample_rate = int(test_conf.get("resample_rate", 16000))
    if resample_rate not in frontend.SAMPLE_RATES:
        raise NotImplementedError(f"dataset_args.resample_rate {resample_rate}: the fbank kernel runs at "
                                  f"{frontend.SAMPLE_RATES} Hz")
    fb = test_conf.get("fbank_args", {}) or {}
    if (float(fb.get("frame_length", 25)), float(fb.get("frame_shift", 10))) != (25.0, 10.0):
        raise NotImplementedError("fbank_args frame_length / frame_shift other than 25 ms / 10 ms are outside the engine's "
                                  "hot path")
    num_mel_bins = int(fb.get("num_mel_bins", feat_dim))
    if num_mel_bins != feat_dim:
        raise ValueError(f"dataset_args.fbank_args.num_mel_bins = {num_mel_bins} does not match the model's feat_dim = "
                         f"{feat_dim}")
    frontend.check_rate_bins(resample_rate, num_mel_bins)
    return resample_rate, num_mel_bins


def _iter_raw(data_list):
    with open(data_list) as f:
        for line in f:
            if line.strip():
                obj = json.loads(line)
                yield obj["key"], obj


def _iter_shards(data_list):
    """(key, {wav bytes}) for every `<key>.<audio ext>` member of the listed tar files, grouped by prefix."""
    with open(data_list) as f:
        urls = [ln.strip() for ln in f if ln.strip()]
    for url in urls:
        with tarfile.open(url, mode="r:*") as tf:
            prev, example = None, {}
            for ti in tf:
                pos = ti.name.rfind(".")
                if pos <= 0 or not ti.isfile():
                    continue
                prefix, postfix = ti.name[:pos], ti.name[pos + 1:]
                if prev is not None and prefix != prev:
                    if "wav_bytes" in example:
                        yield prev, example
                    example = {}
                if postfix in AUDIO_FORMAT_SETS:
                    example["wav_bytes"] = tf.extractfile(ti).read()
                prev = prefix
            if prev is not None and "wav_bytes" in example:
                yield prev, example


def extract(config="conf/config.yaml", **kwargs):
    configs = parse_config_or_kwargs(config, **kwargs)
    model_path = configs["model_path"]
    embed_ark = os.path.abspath(configs["embed_ark"])
    batch_size = int(configs.get("batch_size", 1))
    num_workers = max(1, int(configs.get("num_workers", 1)))
    test_conf = dict(configs.get("dataset_args", {}))
    if test_conf.get("frontend", "fbank") != "fbank":
        raise NotImplementedError("only the fbank frontend is on the engine's hot path")
    if (configs.get("reverb_data") or configs.get("noise_data")) and float(configs.get("aug_prob", 0.0)) > 0.0:
        raise NotImplementedError("reverb / noise augmentation at extraction time is outside the engine's hot path")
    model = get_speaker_model(configs["model"])(precision=configs.get("precision"), **configs["model_args"])
    resample_rate, _ = frontend_args(test_conf, model.feat_dim)
    load_checkpoint(model, model_path)
    device = torch.device("cuda")
    model.to(device).eval()
    cmvn = test_conf.get("cmvn", True)
    cmvn_args = test_conf.get("cmvn_args", {})
    if cmvn_args.get("norm_var", False):
        raise NotImplementedError("cmvn_args.norm_var is outside the engine's hot path (reference default: mean only)")
    data_type = configs.get("data_type", "raw")
    whole_utt = batch_size == 1                       # extract.py:93: whole_utt=(batch_size == 1)
    num_frms = int(test_conf.get("num_frms", 200))
    chunk_samples = ((num_frms - 1) * 10 + 25) * resample_rate // 1000
    rng = random.Random(configs.get("seed", None))    # the reference draws chunk starts from the global `random` module
    os.makedirs(os.path.dirname(embed_ark), exist_ok=True)
    embed_scp = embed_ark[:-3] + "scp"
    n = 0

    with torch.no_grad(), VectorWriter(embed_ark, embed_scp) as writer:
        if data_type == "feat":
            # features are already computed: CMN + forward per utterance (whole) or per num_frms chunk (batched)
            pending = []

            def flush_feats(group):
                nonlocal n
                x = torch.from_numpy(np.stack([f for _, f in group]).astype(np.float32)).to(device)
                if cmvn:
                    x = x - x.mean(dim=1, keepdim=True)
                out = model(x)
                out = (out[-1] if isinstance(out, tuple) else out).cpu().numpy()
                for (k, _), e in zip(group, out):
                    writer(k, e)
                    n += 1

            for key, obj in _iter_raw(configs["data_list"]):
                feat = load_mat(obj["feat"])
                if not whole_utt:
                    feat = get_random_chunk(feat, num_frms, rng)
                if whole_utt:
                    flush_feats([(key, feat)])
                else:
                    pending.append((key, feat))
                    if len(pending) == batch_size:
                        flush_feats(pending)
                        pending = []
            if pending:
                flush_feats(pending)
            return n
        if data_type not in ("raw", "shard"):
            raise ValueError(f"unknown data_type {data_type!r} (shard | raw | feat)")
        if not cmvn:
            raise NotImplementedError("the fused wav path always applies CMN (reference default cmvn: True)")

        def decode(item):
            key, obj = item
            if "wav_bytes" in obj:
                pcm, sr = _decode_wav_bytes(obj["wav_bytes"])
            else:
                pcm, sr = _read_audio(obj["wav"])
                if "vad" in obj:
                    pcm = _apply_vad(pcm, sr, obj["vad"])
            return key, pcm, sr

        def batches():
            """Rectangular (keys, int16 (B, N)) batches: fixed-length chunks, or whole utterances grouped by length."""
            src = _iter_raw(configs["data_list"]) if data_type == "raw" else _iter_shards(configs["data_list"])
            groups = {}
            with ThreadPoolExecutor(num_workers) as pool:       # the DataLoader-worker analogue: PCM decoding only
                for key, pcm, sr in pool.map(decode, src):
                    if sr != resample_rate:   # processor.py:242-262 (torchaudio Resample), on the device, before chunking
                        pcm = frontend.resample(torch.from_numpy(np.array(pcm)), sr, resample_rate).cpu().numpy()
                    if not whole_utt:
                        pcm = get_random_chunk(pcm, chunk_samples, rng)
                    g = groups.setdefault(len(pcm), [])
                    g.append((key, pcm))
                    if len(g) >= (batch_size if not whole_utt else 64):
                        yield [k for k, _ in g], np.stack([p for _, p in g])
                        groups[len(pcm)] = []
            for g in groups.values():
                if g:
                    yield [k for k, _ in g], np.stack([p for _, p in g])

        keys_q = []

        def host_batches():
            for keys, arr in batches():
                keys_q.append(keys)
                yield torch.from_numpy(arr).pin_memory()

        for embs in model.extract_stream(host_batches(), sample_rate=resample_rate):
            keys = keys_q.pop(0)
            for k, e in zip(keys, embs.numpy()):
                writer(k, e)
                n += 1
    return n
