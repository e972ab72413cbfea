"""`Speaker` API mirror (seam B3, SURVEY.md §8b) of `wespeaker/cli/speaker.py:39-178,296-335` — the
embedding-extraction methods, and `:76-88,213-289` — diarization with the speech segments given by the caller (VAD and the
model hub are out of scope).  fbank, CMN, sub-segmentation and the model forward all run on the GPU through the C ABI; WAV
decoding uses the stdlib ``wave`` module so that no torchaudio IO backend is needed."""
from __future__ import annotations

import os
import wave

import numpy as np
import torch
import yaml

from .frontend import fbank_batch
from . import diar, frontend
from .models import get_speaker_model, load_checkpoint


def read_wav(path: str, normalize: bool = False):
    """PCM16 WAV -> (channels, N) tensor; int16-range float32 when normalize=False (torchaudio.load semantics
    used at cli/speaker.py:126-127)."""
    with wave.open(path, "rb") as w:
        if w.getsampwidth() != 2:
            raise ValueError("only 16-bit PCM WAV is supported")
        sr, ch, n = w.getframerate(), w.getnchannels(), w.getnframes()
        data = np.frombuffer(w.readframes(n), dtype="<i2").reshape(-1, ch).T
    pcm = torch.from_numpy(data.astype(np.float32))
    if normalize:
        pcm = pcm / 32768.0
    return pcm, sr


def load_model_pt(model_dir: str, precision: str | None = None):
    """`cli/speaker.py:306-335`: needs {config.yaml, avg_model.pt} in ``model_dir``."""
    for f in ("config.yaml", "avg_model.pt"):
        if not os.path.exists(os.path.join(model_dir, f)):
            raise FileNotFoundError(f"{f} not found in {model_dir}")
    with open(os.path.join(model_dir, "config.yaml")) as f:
        config = yaml.load(f, Loader=yaml.FullLoader)
    model = get_speaker_model(config["model"])(precision=precision, **config["model_args"])
    frontend_type = config.get("dataset_args", {}).get("frontend", "fbank")
    if frontend_type != "fbank":
        raise NotImplementedError("only the fbank frontend is on the engine's hot path (SURVEY.md §0)")
    load_checkpoint(model, os.path.join(model_dir, "avg_model.pt"))
    model.eval()
    model.frontend_type = frontend_type
    return model


class Speaker:
    def __init__(self, model_dir: str | None = None, model=None, precision: str | None = None):
        self.model = model if model is not None else load_model_pt(model_dir, precision)
        self.table = {}
        self.resample_rate = 16000
        self.apply_vad = False
        self.device = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() \
            else torch.device("cpu")
        self.wavform_norm = False
        self.window_type = "hamming"
        self.set_diarization_params(batch_size=256)

    def set_wavform_norm(self, wavform_norm: bool):
        self.wavform_norm = wavform_norm

    def set_window_type(self, window_type: str):
        self.window_type = window_type

    def set_resample_rate(self, resample_rate: int):
        """The rate audio is resampled to before fbank: 16000 or 8000 (the engine's fbank runs at those two)."""
        self.resample_rate = frontend.check_rate_bins(resample_rate)[0]

    def set_vad(self, apply_vad: bool):
        if apply_vad:
            raise NotImplementedError("silero VAD is out of scope for the engine's hot path")
        self.apply_vad = False

    def set_device(self, device: str):
        self.device = torch.device(device)
        self.model = self.model.to(self.device)

    def set_diarization_params(self, min_duration: float = 0.255, window_secs: float = 1.5, period_secs: float = 0.75,
                               frame_shift: int = 10, batch_size: int = 32, subseg_cmn: bool = True):
        """`cli/speaker.py:76-88`.  batch_size bounds the windows per engine launch; the result does not depend on it."""
        self.diar_min_duration = min_duration
        self.diar_window_secs = window_secs
        self.diar_period_secs = period_secs
        self.diar_frame_shift = frame_shift
        self.diar_batch_size = batch_size
        self.diar_subseg_cmn = subseg_cmn

    def compute_features(self, wavform: torch.Tensor, sample_rate: int = 16000, cmn: bool = True):
        """`cli/speaker.py:90-106`: (C,N) waveform at sample_rate (8000 or 16000) -> (1,T,80) features on the GPU."""
        w = wavform[:1].to(self._cuda_device())
        return fbank_batch(w, window_type=self.window_type, cmn=cmn, sample_rate=sample_rate, num_mel_bins=80)

    def _cuda_device(self):
        return self.device if self.device.type == "cuda" else torch.device("cuda", torch.cuda.current_device())

    def extract_embedding_from_feats(self, fbanks, batch_size: int, subseg_cmn: bool):
        """`cli/speaker.py:108-123`: list of (T,80) arrays -> (N,E) numpy."""
        arr = torch.from_numpy(np.stack(fbanks).astype(np.float32)).to(self._cuda_device())
        if subseg_cmn:
            arr = arr - arr.mean(dim=1, keepdim=True)
        embs = []
        for i in range(0, arr.shape[0], batch_size):
            out = self.model(arr[i:i + batch_size])
            out = out[-1] if isinstance(out, tuple) else out
            embs.append(out.detach().cpu().numpy())
        return np.vstack(embs)

    def extract_embedding(self, audio_path: str):
        pcm, sample_rate = read_wav(audio_path, normalize=self.wavform_norm)
        return self.extract_embedding_from_pcm(pcm, sample_rate)

    def extract_embedding_from_pcm(self, pcm: torch.Tensor, sample_rate: int):
        """`cli/speaker.py:130-167`: fused fbank + CMN + forward; returns a CPU (E,) tensor."""
        pcm = pcm.to(torch.float)[:1].to(self._cuda_device())
        if sample_rate != self.resample_rate:   # cli/speaker.py:157-159: torchaudio.transforms.Resample, here on the device
            pcm = frontend.resample(pcm, sample_rate, self.resample_rate)
        emb = self.model.extract_from_wav(pcm, window_type=self.window_type, sample_rate=self.resample_rate)
        return emb[0].to(torch.device("cpu"))

    def extract_embedding_list(self, scp_path: str):
        names, embeddings = [], []
        with open(scp_path) as read_scp:
            for line in read_scp:
                name, wav_path = line.strip().split()
                names.append(name)
                embeddings.append(self.extract_embedding(wav_path).detach().numpy())
        return names, embeddings

    def extract_embedding_batch(self, pcm_batch: torch.Tensor):
        """Addition: (B,N) equal-length int16/float waveforms at the resample rate -> (B,E) CUDA tensor in one fused pass."""
        return self.model.extract_from_wav(pcm_batch.to(self._cuda_device()), window_type=self.window_type,
                                           sample_rate=self.resample_rate)

    def compute_similarity(self, audio_path1: str, audio_path2: str) -> float:
        """`cli/speaker.py:180-186`."""
        e1 = self.extract_embedding(audio_path1)
        e2 = self.extract_embedding(audio_path2)
        if e1 is None or e2 is None:
            return 0.0
        return self.cosine_similarity(e1, e2)

    def cosine_similarity(self, e1, e2):
        """`cli/speaker.py:188-191`: cosine of two (E,) CPU embeddings mapped from [-1, 1] to [0, 1]."""
        cosine_score = torch.dot(e1, e2) / (torch.norm(e1) * torch.norm(e2))
        return (cosine_score.item() + 1.0) / 2

    def register(self, name: str, audio_path: str):
        """`cli/speaker.py:193-197`."""
        if name in self.table:
            print("Speaker {} already registered, ignore".format(name))
        else:
            self.table[name] = self.extract_embedding(audio_path)

    def recognize(self, audio_path: str):
        """`cli/speaker.py:199-211`: best-scoring registered speaker, `{'name', 'confidence'}`."""
        q = self.extract_embedding(audio_path)
        best_score = 0.0
        best_name = ""
        for name, e in self.table.items():
            score = self.cosine_similarity(q, e)
            if best_score < score:
                best_score = score
                best_name = name
        return {"name": best_name, "confidence": best_score}

    def diarize(self, audio_path: str, utt: str = "unk", segments=None):
        """`cli/speaker.py:213-270` with the speech segments [(begin_s, end_s)] given instead of found by VAD, and the
        reference's spectral clusterer in place of umap + hdbscan: -> [(utt, begin_s, end_s, label)].  subseg_cmn=False
        means no CMN at all, as there."""
        if segments is None:
            raise NotImplementedError("silero VAD is out of scope: pass the speech segments [(begin_s, end_s)]")
        if len(segments) == 0:
            return []
        pcm, sample_rate = read_wav(audio_path, normalize=False)
        pcm = pcm[:1].to(self._cuda_device())
        if sample_rate != 16000:
            pcm, sample_rate = frontend.resample(pcm, sample_rate, 16000), 16000
        subsegs, embeddings = diar.extract_subsegment_embeddings(
            self.model, pcm, segments, sample_rate, self.diar_window_secs, self.diar_period_secs, self.diar_frame_shift,
            self.diar_min_duration, self.diar_batch_size, "window" if self.diar_subseg_cmn else "none", self.window_type)
        labels = diar.cluster(embeddings)
        subseg2label = [(*diar.subseg_times(s, self.diar_frame_shift), int(la)) for s, la in zip(subsegs, labels)]
        return diar.merge_segments({utt: subseg2label})

    def diarize_list(self, scp_path: str, segments_path: str):
        """`cli/speaker.py:272-281`; segments_path is the recipe's `segments` file (`seg utt begin_s end_s`)."""
        utt_to_segments = diar.read_segments(segments_path)
        utts, segment2labels = [], []
        with open(scp_path, "r", encoding="utf-8") as read_scp:
            for line in read_scp:
                utt, wav_path = line.strip().split()
                utts.append(utt)
                segs = [(b, e) for _, b, e in utt_to_segments.get(utt, [])]
                segment2labels.append(self.diarize(wav_path, utt, segs))
        return utts, segment2labels

    def make_rttm(self, merged_segment_to_labels, outfile: str):
        diar.make_rttm(merged_segment_to_labels, outfile)


def load_model(model_dir: str, precision: str | None = None) -> Speaker:
    return Speaker(model_dir, precision=precision)
