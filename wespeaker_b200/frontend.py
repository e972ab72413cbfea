"""GPU fbank + CMN with the reference call signatures.

`fbank` mirrors ``torchaudio.compliance.kaldi.fbank`` for the argument set the reference uses
(`wespeaker/dataset/processor.py:518-525`, `wespeaker/cli/speaker.py:92-97`); `apply_cmvn` mirrors
`wespeaker/dataset/dataset_utils.py:19-26`.  The arithmetic runs in ws_fbank.cu through the C ABI.
Sample rates: 16 kHz and 8 kHz (the SRE recipes' ``resample_rate: 8000``), 25 ms frames every 10 ms, 4 to 128 mel bins.
"""
from __future__ import annotations

import torch

from . import lib as _lib


SAMPLE_RATES = (8000, 16000)
MIN_BINS, MAX_BINS = 4, 128


def check_rate_bins(sample_rate, num_mel_bins=80):
    """Refuse what the fbank kernel does not compute: a rate other than 8000 / 16000 (resample first, as the reference does)
    or a mel bin count outside [4, 128]."""
    if float(sample_rate) not in SAMPLE_RATES:
        raise NotImplementedError(f"fbank runs at {SAMPLE_RATES} Hz; resample {sample_rate} Hz audio first")
    if int(num_mel_bins) != num_mel_bins or not MIN_BINS <= int(num_mel_bins) <= MAX_BINS:
        raise NotImplementedError(f"num_mel_bins must be an integer in [{MIN_BINS}, {MAX_BINS}], got {num_mel_bins}")
    return int(sample_rate), int(num_mel_bins)


def frame_geometry(sample_rate: int = 16000):
    """(frame length, frame shift) in samples: 25 ms every 10 ms (400 / 160 at 16 kHz, 200 / 80 at 8 kHz)."""
    sr, _ = check_rate_bins(sample_rate)
    return sr * 25 // 1000, sr // 100


def num_frames(num_samples: int, sample_rate: int = 16000) -> int:
    sr, _ = check_rate_bins(sample_rate)
    return int(_lib.load().ws_fbank_num_frames_at(int(num_samples), sr))


def fbank_batch(wav: torch.Tensor, window_type: str = "hamming", cmn: bool = False, sample_rate: int = 16000,
                num_mel_bins: int = 80) -> torch.Tensor:
    """wav (B,N) CUDA tensor, float32 in int16 range or int16 -> (B,T,num_mel_bins) float32 log-mel (dither 0)."""
    if not wav.is_cuda:
        raise _lib.B200Error("fbank_batch needs a CUDA tensor (no CPU fallback)")
    sr, nb = check_rate_bins(sample_rate, num_mel_bins)
    is_i16 = 1 if wav.dtype == torch.int16 else 0
    wav = wav.contiguous() if is_i16 else wav.float().contiguous()
    B, N = wav.shape
    T = num_frames(N, sr)
    feats = torch.empty((B, T, nb), dtype=torch.float32, device=wav.device)
    if T == 0 or B == 0:
        return feats
    with torch.cuda.device(wav.device.index):
        _lib.check(_lib.load().ws_fbank_at(wav.data_ptr(), is_i16, N, N, B, window_type.encode(), sr, nb, int(cmn),
                                           feats.data_ptr(), _lib.cur_stream_ptr(wav.device.index)), "ws_fbank_at")
    return feats


def fbank(waveform: torch.Tensor, num_mel_bins: int = 80, frame_length: float = 25, frame_shift: float = 10,
          dither: float = 0.0, sample_frequency: float = 16000, window_type: str = "povey",
          use_energy: bool = False, **unsupported) -> torch.Tensor:
    """Same positional meaning as kaldi.fbank for (1,N) input; returns (T, num_mel_bins).  Only the reference's
    argument set is implemented: 8 or 16 kHz, 4 to 128 bins, 25/10 ms, dither 0, no energy."""
    if (float(frame_length), float(frame_shift)) != (25.0, 10.0) or dither != 0.0 or use_energy or unsupported:
        raise NotImplementedError("wespeaker_b200.fbank implements the reference's extraction-time arguments only")
    sr, nb = check_rate_bins(sample_frequency, num_mel_bins)
    dev = waveform.device
    w = waveform[:1] if waveform.dim() == 2 else waveform[None]
    if not w.is_cuda:
        w = w.cuda()
    out = fbank_batch(w, window_type=window_type, sample_rate=sr, num_mel_bins=nb)[0]
    return out if dev.type == "cuda" else out.to(dev)


def compute_fbank(data, num_mel_bins=80, frame_length=25, frame_shift=10, dither=0.0):
    """Generator mirror of `wespeaker/dataset/processor.py:496-526` (sample dicts in, feat dicts out); each sample's
    ``sample_rate`` (8000 or 16000) sets the frame geometry, ``num_mel_bins`` the bin count."""
    for sample in data:
        waveform = sample["wav"] * (1 << 15)
        mat = fbank(waveform, num_mel_bins=num_mel_bins, frame_length=frame_length, frame_shift=frame_shift,
                    dither=dither, sample_frequency=sample["sample_rate"], window_type="hamming", use_energy=False)
        yield dict(key=sample["key"], label=sample["label"], feat=mat)


def apply_cmvn(feats: torch.Tensor, norm_mean: bool = True, norm_var: bool = False) -> torch.Tensor:
    """`wespeaker/dataset/dataset_utils.py:19-26` on a (B,T,F) batch (plain torch elementwise; the
    fused wav->embedding path applies CMN inside ws_fbank.cu instead)."""
    if norm_mean:
        feats = feats - torch.mean(feats, dim=1, keepdim=True)
    if norm_var:
        feats = feats / torch.sqrt(torch.var(feats, dim=1, keepdim=True) + 1e-7)
    return feats


def resample(waveform: torch.Tensor, orig_freq: int, new_freq: int) -> torch.Tensor:
    """`torchaudio.transforms.Resample(orig_freq, new_freq)(waveform)` as the reference applies it before fbank
    (`dataset/processor.py:242-262`, `cli/speaker.py:157-159`): (B, N) or (N,) int16 / float waveform -> float32 on the device,
    ceil(new * N / orig) samples per row (Hann-windowed sinc, lowpass_filter_width 6, rolloff 0.99 = torchaudio's defaults)."""
    if orig_freq == new_freq:
        return waveform.float() if waveform.dtype != torch.int16 else waveform
    L = _lib.load()
    w = waveform.detach()
    squeeze = w.dim() == 1
    if squeeze:
        w = w[None]
    if not w.is_cuda:
        w = w.cuda()
    is_i16 = 1 if w.dtype == torch.int16 else 0
    w = w.contiguous() if is_i16 else w.float().contiguous()
    B, N = w.shape
    n_out = int(L.ws_resample_out_len(N, int(orig_freq), int(new_freq)))
    out = torch.empty((B, n_out), dtype=torch.float32, device=w.device)
    idx = w.device.index if w.device.index is not None else torch.cuda.current_device()
    with torch.cuda.device(idx):
        _lib.check(L.ws_resample(w.data_ptr(), is_i16, N, N, B, int(orig_freq), int(new_freq), out.data_ptr(), n_out,
                                 _lib.cur_stream_ptr(idx)), "ws_resample")
    return out[0] if squeeze else out

