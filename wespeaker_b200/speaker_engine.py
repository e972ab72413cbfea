"""Chunk-and-average long-audio extraction — mirror of the C++ `SpeakerEngine`
(`runtime/core/speaker/speaker_engine.h`, `speaker_engine.cc:30-172`; SURVEY.md §8f rank 4): fbank of the whole
recording, fixed-length chunks (the last one padded with head frames exactly as `ExtractFeature` :77-139 does), per-chunk
mean normalisation (`ApplyMean` :62-75), one embedding per chunk, average (`ExtractEmbedding` :141-159).

GPU shape of the same work: the reference runs its chunks one by one through a batch-1 ONNX session; here all chunks of
a recording are gathered on the device into ONE (nchunk, frames, 80) batch and go through a single engine forward.
"""
from __future__ import annotations

import math

import numpy as np
import torch


def chunk_frame_index(num_frames: int, num_chunk_frames: int) -> np.ndarray:
    """Source-frame index of every frame of every chunk, shape (nchunk, num_chunk_frames): `speaker_engine.cc:100-133`.
    Full chunks are consecutive; a trailing partial chunk is completed with the HEAD frames of the first chunk; a recording
    shorter than one chunk is repeated floor(chunk/len) times and completed with its own head frames."""
    if num_frames <= 0:
        return np.zeros((0, num_chunk_frames), dtype=np.int64)
    nfull = num_frames // num_chunk_frames
    rows = [np.arange(i * num_chunk_frames, (i + 1) * num_chunk_frames, dtype=np.int64) for i in range(nfull)]
    last = num_frames - nfull * num_chunk_frames
    if last > 0:
        own = np.arange(nfull * num_chunk_frames, num_frames, dtype=np.int64)
        if nfull == 0:
            num_pad = num_chunk_frames // last
            row = np.tile(own, max(num_pad, 1))
            row = np.concatenate([row, row[:num_chunk_frames - row.shape[0]]])
        else:
            row = np.concatenate([own, rows[0][:num_chunk_frames - last]])
        rows.append(row)
    return np.stack(rows)


class SpeakerEngine:
    """`SpeakerEngine(model_path, feat_dim, sample_rate, embedding_size, SamplesPerChunk)` with the model object in place
    of the ONNX path.  `fbank_fn(wav (1,N) int16/float tensor) -> (T,feat_dim)` and `embed_fn(feats (B,T,feat_dim)) -> (B,E)`
    default to the GPU frontend (feat_dim bins at sample_rate, 8000 or 16000) and the engine forward; tests inject the CPU
    oracle to check the host logic."""

    def __init__(self, model, feat_dim: int = 80, sample_rate: int = 16000, embedding_size: int | None = None,
                 samples_per_chunk: int = 32000, fbank_fn=None, embed_fn=None):
        from .frontend import check_rate_bins
        self.sample_rate, self.feat_dim = check_rate_bins(sample_rate, feat_dim)
        self.model = model
        self.per_chunk_samples = samples_per_chunk
        self._embedding_size = embedding_size
        self._fbank = fbank_fn or self._gpu_fbank
        self._embed = embed_fn or self._gpu_embed

    # ---- defaults: the GPU path
    def _gpu_fbank(self, wav):
        from .frontend import fbank_batch
        return fbank_batch(wav.cuda(), window_type="hamming", cmn=False, sample_rate=self.sample_rate,   # C++ frontend: hamming
                           num_mel_bins=self.feat_dim)[0]                                                # (fbank.h:90-95)

    def _gpu_embed(self, feats):
        out = self.model(feats)
        return out[-1] if isinstance(out, tuple) else out

    def embedding_size(self) -> int:
        return self._embedding_size if self._embedding_size is not None else self.model.embed_dim

    def num_chunk_frames(self) -> int:
        ms = self.sample_rate // 1000
        return 1 + (self.per_chunk_samples - ms * 25) // (ms * 10)          # speaker_engine.cc:97-99

    def extract_feature(self, pcm) -> torch.Tensor:
        """`ExtractFeature`: (N,) or (1,N) int16 / int16-range float samples -> (nchunk, T, feat_dim) un-normalised chunks."""
        wav = torch.as_tensor(pcm)
        wav = wav[None] if wav.dim() == 1 else wav[:1]
        feats = self._fbank(wav)
        if self.per_chunk_samples <= 0:                                      # full mode (:90-95)
            return feats[None]
        idx = chunk_frame_index(feats.shape[0], self.num_chunk_frames())
        return feats[torch.as_tensor(idx, device=feats.device)]

    def extract_embedding(self, pcm) -> np.ndarray:
        """`ExtractEmbedding`: per-chunk CMN, one forward over all chunks, average of the chunk embeddings."""
        chunks = self.extract_feature(pcm)
        if chunks.shape[0] == 0:
            raise ValueError("recording shorter than one 25 ms frame")
        chunks = chunks - chunks.mean(dim=1, keepdim=True)                   # ApplyMean per chunk
        embs = self._embed(chunks.contiguous())
        return embs.float().mean(dim=0).cpu().numpy()

    @staticmethod
    def cosine_similarity(emb1, emb2) -> float:
        """`CosineSimilarity` (:161-172): cosine mapped to [0, 1]."""
        e1, e2 = np.asarray(emb1, dtype=np.float64), np.asarray(emb2, dtype=np.float64)
        dot = float(e1 @ e2) / max(math.sqrt(float(e1 @ e1)) * math.sqrt(float(e2 @ e2)), float(np.finfo(np.float32).eps))
        return (dot + 1.0) / 2.0
