"""Drop-in model objects for the reference operator seam B1 (SURVEY.md §8b):

    model = get_speaker_model(name)(**model_args)      # wespeaker/models/speaker_model.py:31-62
    load_checkpoint(model, path)                       # wespeaker/utils/checkpoint.py:20-85
    model.to(device).eval()
    outputs = model(features)                          # features: float32 (B,T,feat_dim)
    embeds = outputs[-1] if isinstance(outputs, tuple) else outputs   # bin/extract.py:133-134

``B200SpeakerModel`` is an ``nn.Module``-shaped object holding the *reference* ``state_dict`` (same
key names / shapes) whose ``forward`` runs the hand-written sm_90a engine through the C ABI
(include/wespeaker_b200.h).  PyTorch is used for device memory and streams only.
"""
from __future__ import annotations

import ctypes as C
import os
from collections import OrderedDict, namedtuple

import numpy as np
import torch

from . import frontend as _frontend
from . import lib as _lib
from .synthetic import (CAMPP_NAMES, DEFAULT_MODEL_ARGS, ECAPA_NAMES, GEMINI_NAMES, RES2NET_NAMES, RESNET_NAMES, SIMAM_NAMES,
                        XVEC_NAMES, state_dict_spec)

_IncompatibleKeys = namedtuple("IncompatibleKeys", ["missing_keys", "unexpected_keys"])
SUPPORTED_MODELS = tuple(ECAPA_NAMES) + tuple(RESNET_NAMES) + tuple(CAMPP_NAMES) + tuple(XVEC_NAMES) + tuple(RES2NET_NAMES) \
    + tuple(SIMAM_NAMES) + tuple(GEMINI_NAMES)


class B200SpeakerModel(torch.nn.Module):
    """One reference speaker model executed by the GPU engine.

    precision: "tf32x3" (default: tensor cores with three error-compensated TF32 passes, embeddings <= 1e-4 rel of
    the reference - measured <= 4.9e-5), "fp32" (exact fp32 FFMA path, <= 6e-7), "tf32", "bf16", "fp16" (single-pass
    tensor-core paths, 16-bit activations for the last two).  Default from $WESPEAKER_B200_PRECISION or "tf32x3".
    """

    def __init__(self, model_name: str, precision: str | None = None, **model_args):
        super().__init__()
        if model_name not in SUPPORTED_MODELS:
            raise ValueError(f"{model_name} is not on the engine's hot path (supported: {SUPPORTED_MODELS})")
        args = dict(DEFAULT_MODEL_ARGS[model_name])
        args.update(model_args)
        self.model_name = model_name
        self.model_args = args
        self.precision = precision or os.environ.get("WESPEAKER_B200_PRECISION", "tf32x3")
        # SimAM-ResNet names its feature dimension acoustic_dim (samresnet.py:135)
        self.feat_dim = int(args["acoustic_dim"] if model_name in SIMAM_NAMES else args["feat_dim"])
        self.embed_dim = int(args["embed_dim"])
        self._spec = state_dict_spec(model_name, **args)
        self._sd: "OrderedDict[str, torch.Tensor]" = OrderedDict()
        self._device = torch.device("cpu")
        self._engine = None
        self._engine_device = None
        self.frontend_type = "fbank"
        self.options = {}

    # ------------------------------------------------------------------ nn.Module-compatible surface
    def state_dict(self, *a, **k):
        sd = OrderedDict()
        for key, shape in self._spec.items():
            if key in self._sd:
                sd[key] = self._sd[key]
            elif key.endswith("num_batches_tracked"):
                sd[key] = torch.zeros((), dtype=torch.long)
            else:
                sd[key] = torch.zeros(shape, dtype=torch.float32)
        return sd

    def load_state_dict(self, state_dict, strict: bool = True, **_):
        missing = [k for k in self._spec if k not in state_dict and not k.endswith("num_batches_tracked")]
        unexpected = [k for k in state_dict if k not in self._spec]
        errors = []
        for k, shape in self._spec.items():
            if k in state_dict:
                v = state_dict[k]
                v = torch.as_tensor(np.asarray(v)) if not torch.is_tensor(v) else v
                if tuple(v.shape) != tuple(shape):
                    errors.append(f"size mismatch for {k}: checkpoint {tuple(v.shape)} vs model {tuple(shape)}")
                    continue
                self._sd[k] = v.detach().to("cpu")
        if errors or (strict and (missing or unexpected)):
            raise RuntimeError("Error(s) in loading state_dict for {}:\n\t{}".format(
                self.model_name, "\n\t".join(errors + [f"missing: {missing}"] * bool(strict and missing)
                                             + [f"unexpected: {unexpected}"] * bool(strict and unexpected))))
        self._drop_engine()
        return _IncompatibleKeys(missing, unexpected)

    def to(self, device=None, *a, **k):
        if device is not None and not isinstance(device, torch.dtype):
            self._device = torch.device(device)
            if self._device.type == "cuda" and self._device.index is None:
                self._device = torch.device("cuda", torch.cuda.current_device())
        return self

    def cuda(self, device=None):
        return self.to(torch.device("cuda", device if device is not None else torch.cuda.current_device()))

    def eval(self):
        return self

    def train(self, mode: bool = True):
        if mode:
            raise NotImplementedError("wespeaker_b200 is an inference engine (training is out of scope)")
        return self

    def set_option(self, key: str, value: int):
        self.options[key] = int(value)
        self._drop_engine()

    def engine_options(self) -> dict:
        """The engine options of this model, in the order the engine receives them: the model_args flags two_emb_layer and
        emb_bn, then every set_option call (a later value wins)."""
        opts = {k: 1 for k in ("two_emb_layer", "emb_bn") if self.model_args.get(k)}
        opts.update(self.options)
        return opts

    # ------------------------------------------------------------------ engine
    def _drop_engine(self):
        if self._engine is not None:
            _lib.load().ws_engine_destroy(self._engine)
            self._engine = None

    def __del__(self):
        try:
            self._drop_engine()
        except Exception:
            pass

    def _ensure_engine(self, dev_index: int):
        if self._engine is not None and self._engine_device == dev_index:
            return self._engine
        self._drop_engine()
        L = _lib.load()
        if not torch.cuda.is_available():
            raise _lib.B200Error("wespeaker_b200 needs a CUDA device (no CPU fallback)")
        h = _lib.c_engine_p()
        _lib.check(L.ws_engine_create(self.model_name.encode(), self.precision.encode(), self.feat_dim,
                                      self.embed_dim, dev_index, C.byref(h)), "ws_engine_create")
        try:
            self._configure(L, h)
        except Exception:
            L.ws_engine_destroy(h)
            raise
        self._engine, self._engine_device = h, dev_index
        return h

    def _configure(self, L, h):
        """options + reference state_dict -> engine handle, then finalize (packs / folds / converts the weights)."""
        for k, v in self.engine_options().items():
            _lib.check(L.ws_engine_set_option(h, k.encode(), v), "ws_engine_set_option")
        for k, v in self._sd.items():
            if k.endswith("num_batches_tracked"):
                continue
            a = np.ascontiguousarray(v.detach().cpu().numpy(), dtype=np.float32)
            shape = (C.c_longlong * a.ndim)(*a.shape)
            _lib.check(L.ws_engine_set_tensor(h, k.encode(), a.ctypes.data, shape, a.ndim),
                       "ws_engine_set_tensor")
        _lib.check(L.ws_engine_finalize(h), "ws_engine_finalize")

    def plan_trace(self, path: str, batch: int = 1, frames: int = 200, masked: bool = False):
        """Write the (batch, frames) launch plan as data (ws_engine_plan_trace; no device, nothing computed): tests re-evaluate
        it on the host against the oracle (tests/plan_interp.py)."""
        L = _lib.load()
        h = _lib.c_engine_p()
        _lib.check(L.ws_engine_create_plan_check(self.model_name.encode(), self.precision.encode(), self.feat_dim,
                                                 self.embed_dim, C.byref(h)), "ws_engine_create_plan_check")
        try:
            self._configure(L, h)
            _lib.check(L.ws_engine_plan_trace(h, batch, frames, int(masked), path.encode()), "ws_engine_plan_trace")
        finally:
            L.ws_engine_destroy(h)

    def device_trace(self, path: str, batch: int = 1, frames: int = 200, masked: bool = False, device: int | None = None):
        """Write the (batch, frames) launch plan of the engine on `device` as data, with device addresses and every weight
        and plan-buffer allocation (ws_engine_plan_trace on a real engine; needs set_option("plan_trace", 1)).  With
        run_ops, tests check what each kernel of the plan writes."""
        L = _lib.load()
        idx = self._dev_index() if device is None else device
        h = self._ensure_engine(idx)
        with torch.cuda.device(idx):
            _lib.check(L.ws_engine_plan_trace(h, batch, frames, int(masked), path.encode()), "ws_engine_plan_trace")

    def run_ops(self, batch: int, frames: int, masked: bool, first: int, last: int, device: int | None = None):
        """Run ops [first, last) of the (batch, frames) plan eagerly (no CUDA graph) on the current stream; the caller has
        filled the plan's inputs (feats_in, and lens in a masked plan, as named by device_trace)."""
        L = _lib.load()
        idx = self._dev_index() if device is None else device
        h = self._ensure_engine(idx)
        with torch.cuda.device(idx):
            _lib.check(L.ws_engine_run_ops(h, batch, frames, int(masked), first, last, _lib.cur_stream_ptr(idx)),
                       "ws_engine_run_ops")

    def plan_check(self, batch: int = 1, frames: int = 200):
        """Validate the loaded checkpoint against the engine's plan builder WITHOUT a device (ws_engine_create_plan_check:
        nothing is computed): missing / mis-shaped tensors, kernel envelopes and tensor-map alignment rules raise B200Error.
        Returns the launch plan of a (batch, frames) input as a list of (op label, FLOPs)."""
        L = _lib.load()
        h = _lib.c_engine_p()
        _lib.check(L.ws_engine_create_plan_check(self.model_name.encode(), self.precision.encode(), self.feat_dim,
                                                 self.embed_dim, C.byref(h)), "ws_engine_create_plan_check")
        try:
            self._configure(L, h)
            ops, fl = [], C.c_double(0.0)
            while True:
                name = L.ws_engine_plan_op_name(h, batch, frames, len(ops), C.byref(fl))
                if name is None:
                    break
                ops.append((name.decode(), fl.value))
            if not ops:
                _lib.check(1, "ws_engine_plan_op_name")
            return ops
        finally:
            L.ws_engine_destroy(h)

    def _dev_index(self, t: torch.Tensor | None = None) -> int:
        if t is not None and t.is_cuda:
            return t.device.index
        if self._device.type == "cuda":
            return self._device.index
        return torch.cuda.current_device() if torch.cuda.is_available() else 0

    def _wav_engine(self, dev_index: int, sample_rate: int):
        """The engine on `dev_index`, its waveform entry points set to `sample_rate` (their fbank writes feat_dim bins)."""
        sr, _ = _frontend.check_rate_bins(sample_rate, self.feat_dim)
        h = self._ensure_engine(dev_index)
        _lib.check(_lib.load().ws_engine_set_option(h, b"sample_rate", sr), "ws_engine_set_option")
        return h

    # ------------------------------------------------------------------ forward paths
    def embed(self, features: torch.Tensor) -> torch.Tensor:
        """(B,T,feat_dim) float32 -> (B,embed_dim) float32 on the same device class as the input."""
        if features.dim() != 3 or features.shape[2] != self.feat_dim:
            raise ValueError(f"expected features (B,T,{self.feat_dim}), got {tuple(features.shape)}")
        L = _lib.load()
        B, T, _ = features.shape
        if features.is_cuda:
            idx = features.device.index
            h = self._ensure_engine(idx)
            x = features.detach().contiguous().float()
            out = torch.empty((B, self.embed_dim), dtype=torch.float32, device=features.device)
            with torch.cuda.device(idx):
                _lib.check(L.ws_engine_forward(h, x.data_ptr(), B, T, out.data_ptr(), _lib.cur_stream_ptr(idx)),
                           "ws_engine_forward")
            return out
        # host tensor (cli/speaker.py:160-166 hands CPU feats to the model): H2D + forward + D2H inside the ABI
        idx = self._dev_index()
        h = self._ensure_engine(idx)
        x = features.detach().contiguous().float()
        out = torch.empty((B, self.embed_dim), dtype=torch.float32)
        _lib.check(L.ws_engine_forward_host(h, x.data_ptr(), B, T, out.data_ptr()), "ws_engine_forward_host")
        return out

    def forward(self, features: torch.Tensor):
        emb = self.embed(features)
        if self.model_name in CAMPP_NAMES or self.model_name in RES2NET_NAMES or self.model_name in SIMAM_NAMES:
            return emb  # campplus.py:409-413, res2net.py:199, eres2net.py:391, samresnet.py:142-149 return a bare tensor
        # ecapa_tdnn.py:234 returns (out4, emb); resnet.py:204 and gemini_dfresnet.py:130-136 return (tensor(0.), embed_a).
        # Callers use [-1].
        return torch.tensor(0.0), emb

    def extract_from_wav(self, wav: torch.Tensor, window_type: str = "hamming", return_feats: bool = False,
                         sample_rate: int = 16000):
        """wav: (B,N) float32 (int16 range, i.e. ``wav * (1 << 15)``) or int16 PCM at sample_rate (8000 or 16000), CUDA or
        host.  fbank (feat_dim bins, dither 0) + CMN + forward entirely on the GPU."""
        if wav.dim() != 2:
            raise ValueError("wav must be (B, N)")
        L = _lib.load()
        is_i16 = 1 if wav.dtype == torch.int16 else 0
        if not is_i16:
            wav = wav.float()
        wav = wav.contiguous()
        B, N = wav.shape
        if wav.is_cuda:
            idx = wav.device.index
            h = self._wav_engine(idx, sample_rate)
            out = torch.empty((B, self.embed_dim), dtype=torch.float32, device=wav.device)
            T = _frontend.num_frames(N, sample_rate)
            feats = torch.empty((B, T, self.feat_dim), dtype=torch.float32, device=wav.device) if return_feats else None
            with torch.cuda.device(idx):
                _lib.check(L.ws_engine_extract_wav(h, wav.data_ptr(), is_i16, N, N, B, window_type.encode(),
                                                   out.data_ptr(), feats.data_ptr() if return_feats else None,
                                                   _lib.cur_stream_ptr(idx)), "ws_engine_extract_wav")
            return (out, feats) if return_feats else out
        h = self._wav_engine(self._dev_index(), sample_rate)
        out = torch.empty((B, self.embed_dim), dtype=torch.float32)
        _lib.check(L.ws_engine_extract_wav_host(h, wav.data_ptr(), is_i16, N, B, window_type.encode(),
                                                out.data_ptr()), "ws_engine_extract_wav_host")
        return out

    def extract_stream(self, host_batches, window_type: str = "hamming", depth: int = 4, sample_rate: int = 16000):
        """Pipelined extraction over an iterable of HOST waveform batches ((B,N) int16 or int16-range float32, ideally
        pinned).  Yields one pinned CPU (B, embed_dim) tensor per batch, in order.  The H2D copy of batch i+1 overlaps
        the kernels of batch i (`depth` <= 4 staging slots inside the C ABI) — the analogue of the reference's DataLoader
        prefetching (extract.py:99-103)."""
        L = _lib.load()
        h = self._wav_engine(self._dev_index(), sample_rate)
        pending = []  # (slot, wav_keepalive, pinned_out)
        slot = 0
        pool = getattr(self, "_pinned_out", None)
        if pool is None:
            pool = self._pinned_out = {}
        for wav in host_batches:
            if wav.is_cuda:
                raise ValueError("extract_stream takes host tensors; use extract_from_wav for CUDA tensors")
            is_i16 = 1 if wav.dtype == torch.int16 else 0
            w = wav.contiguous() if is_i16 else wav.float().contiguous()
            B, N = w.shape
            if len(pending) == depth:  # the slot we are about to reuse must have been collected
                s0, _, o0 = pending.pop(0)
                _lib.check(L.ws_engine_collect(h, s0), "ws_engine_collect")
                yield self._unpinned_copy(o0)
            key = (slot, B)
            if key not in pool:  # pinned result buffers are allocated once per (slot, batch size): cudaHostAlloc is slow
                pool[key] = torch.empty((B, self.embed_dim), dtype=torch.float32).pin_memory()
            out = pool[key]
            _lib.check(L.ws_engine_submit_wav_host(h, slot, w.data_ptr(), is_i16, N, B, window_type.encode(),
                                                   out.data_ptr()), "ws_engine_submit_wav_host")
            pending.append((slot, w, out))
            slot = (slot + 1) % depth
        for s0, _, o0 in pending:
            _lib.check(L.ws_engine_collect(h, s0), "ws_engine_collect")
            yield self._unpinned_copy(o0)

    @staticmethod
    def _unpinned_copy(t: torch.Tensor) -> torch.Tensor:
        # Tensor.clone() of a pinned tensor allocates pinned memory again (a cudaHostAlloc per batch, ~6 ms); copy into
        # ordinary pageable memory instead
        # numpy's single-threaded memcpy: a torch copy_ may wake a large intra-op thread pool whose spinning workers get
        # the process CPU-throttled on shared hosts, which shows up as multi-ms stalls of the next collect()
        return torch.from_numpy(t.numpy().copy())

    # ------------------------------------------------------------------ variable-length batches (BASELINE config 4)
    def _run_buckets(self, items, key_fn, stack_fn, launch, max_batch, device):
        """Bucket `items` by exact length, enqueue EVERY bucket through the *_async entry points (the engine spreads the
        per-(B,T) plans over several streams, so small buckets overlap on the GPU) and close with one ws_engine_join."""
        L = _lib.load()
        buckets = {}
        for i, it in enumerate(items):
            buckets.setdefault(key_fn(it), []).append(i)
        dev = torch.device(device) if device is not None else items[0].device
        if dev.type != "cuda":
            dev = torch.device("cuda", self._dev_index())
        h = self._ensure_engine(dev.index)
        out = torch.empty((len(items), self.embed_dim), dtype=torch.float32, device=dev)
        keep = []
        with torch.cuda.device(dev.index):
            st = _lib.cur_stream_ptr(dev.index)
            for _, idx in sorted(buckets.items()):
                for s0 in range(0, len(idx), max_batch):
                    sel = idx[s0:s0 + max_batch]
                    x = stack_fn([items[i] for i in sel]).to(dev)
                    o = torch.empty((len(sel), self.embed_dim), dtype=torch.float32, device=dev)
                    keep.append((sel, launch(L, h, x, o, st), o))   # inputs stay alive until the join
            _lib.check(L.ws_engine_join(h, st), "ws_engine_join")
            for sel, _, o in keep:
                out[torch.as_tensor(sel, device=dev)] = o
        return out

    # ------------------------------------------------------------------ length-masked batches
    def embed_padded(self, features: torch.Tensor, lengths) -> torch.Tensor:
        """(B, Tmax, feat_dim) features of utterances with `lengths[b]` valid frames each (rows behind are ignored, any
        content) -> (B, embed_dim): every row equals what the utterance produces on its own, unpadded (the reference has no
        masking and therefore extracts test sets at batch 1, extract_vox.sh:31)."""
        L = _lib.load()
        x = features.detach()
        if not x.is_cuda:
            x = x.to(torch.device("cuda", self._dev_index()))
        x = x.contiguous().float()
        B, T, _ = x.shape
        idx = x.device.index
        h = self._ensure_engine(idx)
        n = torch.as_tensor(lengths, dtype=torch.int32).to(x.device).contiguous()
        if n.numel() != B:
            raise ValueError("lengths must have one entry per utterance")
        out = torch.empty((B, self.embed_dim), dtype=torch.float32, device=x.device)
        with torch.cuda.device(idx):
            _lib.check(L.ws_engine_forward_masked(h, x.data_ptr(), n.data_ptr(), B, T, out.data_ptr(), _lib.cur_stream_ptr(idx)),
                       "ws_engine_forward_masked")
        return out

    def extract_from_wav_padded(self, wavs: torch.Tensor, n_samples, window_type: str = "hamming",
                                sample_rate: int = 16000) -> torch.Tensor:
        """(B, Nmax) waveforms (int16 or int16-range float32) with `n_samples[b]` valid samples each -> (B, embed_dim):
        fbank, CMN over each utterance's own frames, masked forward."""
        L = _lib.load()
        w = wavs.detach()
        if not w.is_cuda:
            w = w.to(torch.device("cuda", self._dev_index()))
        is_i16 = 1 if w.dtype == torch.int16 else 0
        w = w.contiguous() if is_i16 else w.float().contiguous()
        B, N = w.shape
        idx = w.device.index
        h = self._wav_engine(idx, sample_rate)
        n = torch.as_tensor(n_samples, dtype=torch.int32).to(w.device).contiguous()
        nmax = int(n.max().item())
        out = torch.empty((B, self.embed_dim), dtype=torch.float32, device=w.device)
        with torch.cuda.device(idx):
            _lib.check(L.ws_engine_extract_wav_masked(h, w.data_ptr(), is_i16, N, n.data_ptr(), nmax, B, window_type.encode(),
                                                      out.data_ptr(), _lib.cur_stream_ptr(idx)), "ws_engine_extract_wav_masked")
        return out

    @staticmethod
    def length_buckets(lengths, max_batch: int = 64, max_pad: float = 0.15):
        """Greedy grouping for padded batches: longest first; a batch takes utterances down to (1 - max_pad) of its longest
        member, at most max_batch of them.  Returns a list of index lists."""
        order = sorted(range(len(lengths)), key=lambda i: -int(lengths[i]))
        out, cur = [], []
        for i in order:
            if cur and (len(cur) >= max_batch or int(lengths[i]) < (1.0 - max_pad) * int(lengths[cur[0]])):
                out.append(cur)
                cur = []
            cur.append(i)
        if cur:
            out.append(cur)
        return out

    def embed_list_padded(self, feats_list, max_batch: int = 64, max_pad: float = 0.15, device=None):
        """Variable-length utterances through length-masked batches: a handful of (B, Tmax) plans serve ANY mix of lengths
        (exact-length bucketing needs one plan per distinct length).  Returns (N, embed_dim) in input order."""
        if len(feats_list) == 0:
            return torch.empty((0, self.embed_dim))
        dev = torch.device(device) if device is not None else feats_list[0].device
        if dev.type != "cuda":
            dev = torch.device("cuda", self._dev_index())
        lens = [int(f.shape[0]) for f in feats_list]
        out = torch.empty((len(feats_list), self.embed_dim), dtype=torch.float32, device=dev)
        for sel in self.length_buckets(lens, max_batch, max_pad):
            tmax = -(-lens[sel[0]] // 8) * 8                     # a few shapes, not one per length: round Tmax up to 8
            x = torch.zeros((len(sel), tmax, self.feat_dim), dtype=torch.float32, device=dev)
            for j, i in enumerate(sel):
                x[j, : lens[i]] = feats_list[i].to(dev)
            out[torch.as_tensor(sel, device=dev)] = self.embed_padded(x, [lens[i] for i in sel])
        return out

    def embed_list(self, feats_list, max_batch: int = 64, device=None):
        """Embeddings for utterances of DIFFERENT lengths.  The reference has no length masking (SURVEY §3.1: test sets
        run at batch 1), so padding would change results; instead utterances are bucketed by exact frame count, each bucket
        is one batch (one cached plan / CUDA graph per (B,T)) and the buckets run concurrently on the engine's streams.
        feats_list: list of (T_i, feat_dim) tensors.  Returns (N, embed_dim) in input order on the CUDA device."""
        if len(feats_list) == 0:
            return torch.empty((0, self.embed_dim))

        def launch(L, h, x, o, st):
            x = x.contiguous().float()
            _lib.check(L.ws_engine_forward_async(h, x.data_ptr(), x.shape[0], x.shape[1], o.data_ptr(), st), "ws_engine_forward_async")
            return x
        return self._run_buckets(feats_list, lambda f: int(f.shape[0]), torch.stack, launch, max_batch, device)

    def extract_from_wav_list(self, wavs, window_type: str = "hamming", max_batch: int = 64, device=None,
                              sample_rate: int = 16000):
        """Same bucketing for raw waveforms (1-D tensors of different lengths, int16 or int16-range float32)."""
        if len(wavs) == 0:
            return torch.empty((0, self.embed_dim))
        wt = window_type.encode()
        dev = torch.device(device) if device is not None else wavs[0].device
        self._wav_engine(dev.index if dev.type == "cuda" and dev.index is not None else self._dev_index(), sample_rate)

        def launch(L, h, x, o, st):
            is_i16 = 1 if x.dtype == torch.int16 else 0
            x = x.contiguous() if is_i16 else x.float().contiguous()
            _lib.check(L.ws_engine_extract_wav_async(h, x.data_ptr(), is_i16, x.shape[1], x.shape[1], x.shape[0], wt, o.data_ptr(), st),
                       "ws_engine_extract_wav_async")
            return x
        return self._run_buckets(wavs, lambda w: int(w.shape[-1]), lambda ws: torch.stack([w.reshape(-1) for w in ws]), launch,
                                 max_batch, device)

    @staticmethod
    def frame_grid(t: int, ratio: float = 1.15) -> int:
        """Smallest member >= t of the geometric frame grid 16, 24, 32, ... (each step x ratio, rounded up to 8 frames): the
        padded T of a length-masked bucket, so that ANY mix of durations runs through a bounded set of plans."""
        g = 16
        while g < t:
            g = -(-int(g * ratio + 0.999) // 8) * 8
        return g

    def extract_from_wav_list_ragged(self, wavs, window_type: str = "hamming", max_batch: int = 64, grid_ratio: float = 1.15,
                                     device=None, sample_rate: int = 16000) -> torch.Tensor:
        """Waveforms of ARBITRARY lengths (1-D tensors, int16 or int16-range float32) -> (N, embed_dim) in input order.
        The PCM is concatenated once (no padded copies); utterances are grouped by the frame grid above into length-masked
        buckets of <= max_batch (B rounded up to 8 by repeating an utterance, so the set of (B, T) plans stays small), each
        bucket is one ws_engine_extract_wav_ragged_async on the engine's streams, one join at the end.  With exact-length
        bucketing (extract_from_wav_list) every distinct length costs its own plan and launch; here the cost is the padding
        inside a grid cell (< grid_ratio - 1 of the frames, ~7 % on average)."""
        if len(wavs) == 0:
            return torch.empty((0, self.embed_dim))
        L = _lib.load()
        dev = torch.device(device) if device is not None else wavs[0].device
        if dev.type != "cuda":
            dev = torch.device("cuda", self._dev_index())
        idx = dev.index if dev.index is not None else torch.cuda.current_device()
        ns = [int(w.numel()) for w in wavs]
        flen, shift = _frontend.frame_geometry(sample_rate)
        if min(ns) < flen:
            raise ValueError(f"every waveform must hold at least one 25 ms frame ({flen} samples at {sample_rate} Hz)")
        is_i16 = 1 if all(w.dtype == torch.int16 for w in wavs) else 0
        flat = torch.cat([(w if is_i16 else w.float()).reshape(-1).to(dev) for w in wavs])
        starts = np.concatenate([[0], np.cumsum(ns)[:-1]]).astype(np.int64)
        cells = {}
        for i, n in enumerate(ns):
            cells.setdefault(self.frame_grid(1 + (n - flen) // shift, grid_ratio), []).append(i)
        slots, batches = [], []                      # slots: utterance index per launched row; batches: (rows, Tgrid)
        for tg in sorted(cells, reverse=True):
            members = cells[tg]
            for c in range(0, len(members), max_batch):
                chunk = members[c:c + max_batch]
                rows = min(max_batch, -(-len(chunk) // 8) * 8)
                chunk = chunk + [chunk[-1]] * (rows - len(chunk))
                batches.append((len(chunk), tg))
                slots.extend(chunk)
        slots_np = np.asarray(slots, dtype=np.int64)
        offs = torch.from_numpy(starts[slots_np]).to(dev)
        nsd = torch.from_numpy(np.asarray(ns, dtype=np.int32)[slots_np]).to(dev)
        out = torch.empty((len(slots), self.embed_dim), dtype=torch.float32, device=dev)
        first = np.full(len(wavs), -1, dtype=np.int64)
        first[slots_np[::-1]] = np.arange(len(slots) - 1, -1, -1)            # first launched row of each utterance
        h = self._wav_engine(idx, sample_rate)
        wt = window_type.encode()
        with torch.cuda.device(idx):
            st = _lib.cur_stream_ptr(idx)
            pos = 0
            for rows, tg in batches:
                _lib.check(L.ws_engine_extract_wav_ragged_async(h, flat.data_ptr(), is_i16, offs.data_ptr() + 8 * pos,
                                                                nsd.data_ptr() + 4 * pos, (tg - 1) * shift + flen, rows, wt,
                                                                out.data_ptr() + 4 * self.embed_dim * pos, st),
                           "ws_engine_extract_wav_ragged_async")
                pos += rows
            _lib.check(L.ws_engine_join(h, st), "ws_engine_join")
        return out[torch.from_numpy(first).to(dev)]

    def export_flat(self, path: str):
        """Write the flat weights file the C++ back-end seam reads (`csrc/runtime/b200_speaker_model.h`, seam B4:
        `wespeaker::B200SpeakerModel(path)` behind `runtime/core/speaker/speaker_model.h:25-32`)."""
        import struct

        def wstr(f, t: str):
            b = t.encode()
            f.write(struct.pack("<I", len(b)) + b)
        opts = self.engine_options()
        tensors = [(k, v) for k, v in self._sd.items() if not k.endswith("num_batches_tracked")]
        with open(path, "wb") as f:
            f.write(b"WSPKB200" + struct.pack("<I", 1))
            wstr(f, self.model_name)
            wstr(f, self.precision)
            f.write(struct.pack("<ii", self.feat_dim, self.embed_dim))
            f.write(struct.pack("<I", len(opts)))
            for k, v in opts.items():
                wstr(f, k)
                f.write(struct.pack("<q", v))
            f.write(struct.pack("<I", len(tensors)))
            for k, v in tensors:
                a = np.ascontiguousarray(v.detach().cpu().numpy(), dtype="<f4")
                wstr(f, k)
                f.write(struct.pack("<I", a.ndim) + struct.pack(f"<{a.ndim}q", *a.shape))
                f.write(a.tobytes())

    def last_launches(self) -> int:
        return int(_lib.load().ws_engine_last_launches(self._engine)) if self._engine is not None else 0


def get_speaker_model(model_name: str):
    """Mirror of `wespeaker/models/speaker_model.py:31-62`: name -> constructor taking **model_args."""
    if model_name not in SUPPORTED_MODELS:
        # the reference prints and exit(1)s (speaker_model.py:60-62); raising is the library-friendly equivalent
        raise ValueError(f"{model_name} not found / not on the engine's hot path; supported: {SUPPORTED_MODELS}")

    def ctor(**model_args):
        return B200SpeakerModel(model_name, **model_args)

    ctor.__name__ = model_name
    return ctor


def load_checkpoint(model, path: str):
    """Mirror of `wespeaker/utils/checkpoint.py:20-85`: torch.load, unwrap ``state_dict``, ignore
    ``projection.*`` (training head), ``load_state_dict(strict=False)`` with warnings."""
    import logging
    checkpoint = torch.load(path, map_location="cpu", weights_only=False)
    if isinstance(checkpoint, dict) and "state_dict" in checkpoint:
        checkpoint = checkpoint["state_dict"]
    missing, unexpected = model.load_state_dict(checkpoint, strict=False)
    for key in missing:
        if "projection" not in key:
            logging.warning("missing tensor: %s", key)
    for key in unexpected:
        if "projection" not in key:
            logging.warning("unexpected tensor: %s", key)


def from_synthetic(model_name: str, seed: int = 0, precision: str | None = None, **model_args):
    """Random-init model of the reference architecture (no pretrained checkpoints offline)."""
    from .synthetic import make_state_dict
    m = B200SpeakerModel(model_name, precision=precision, **model_args)
    m.load_state_dict({k: torch.from_numpy(np.asarray(v)) for k, v in make_state_dict(model_name, seed, **model_args).items()})
    return m
