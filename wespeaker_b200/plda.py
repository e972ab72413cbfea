"""Two-covariance PLDA scoring on the GPU — mirror of the scoring half of
`wespeaker/utils/plda/two_cov_plda.py` (seam B5, SURVEY.md §8b): ``load_model``, ``transform_embedding``,
``log_likelihood_ratio``, ``eval_sv``; plus the batched entry points the GPU makes worthwhile
(``transform_batch`` on (N,D) matrices, ``score_matrix`` all-pairs, ``score_trials``).  All arithmetic is fp64 on
the device (ws_plda.cu); numpy here is only file parsing and host<->device staging.  Training / adaptation
(`two_cov_plda.py:106-154,258-309`) live in plda_train.py.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import lib as _lib
from .kaldi_io import read_vec_scp_file


def read_label_file(label_file):
    """`wespeaker/utils/plda/plda_utils.py:32-43`."""
    labels = {}
    with open(label_file) as fin:
        for line in fin:
            tok = line.strip().split()
            if tok:
                labels[tok[0]] = tok[1]
    return labels


class TwoCovPLDA:
    def __init__(self, embed_dim: int = 256, normalize_length: bool = False, subtract_train_set_mean: bool = False,
                 device: int | None = None):
        self.dim = embed_dim
        self.normalize_length = normalize_length
        self.subtract_train_set_mean = subtract_train_set_mean
        self.mu = np.zeros(embed_dim)
        self.transform = np.zeros((embed_dim, embed_dim))
        self.psi = np.zeros(embed_dim)
        self.offset = np.zeros(embed_dim)
        self._device = device
        self._h = None

    # ------------------------------------------------------------------ model IO (two_cov_plda.py:341-363)
    @staticmethod
    def from_arrays(mu, transform, psi, offset=None, normalize_length=False, subtract_train_set_mean=False,
                    device=None, **_):
        p = TwoCovPLDA(len(mu), normalize_length, subtract_train_set_mean, device)
        p.mu = np.asarray(mu, dtype=np.float64)
        p.transform = np.ascontiguousarray(transform, dtype=np.float64)
        p.psi = np.asarray(psi, dtype=np.float64)
        p.offset = (-1.0 * p.transform @ p.mu) if offset is None else np.asarray(offset, dtype=np.float64)
        return p

    @staticmethod
    def load_model(model_name: str, from_kaldi: bool = False, device=None):
        """`two_cov_plda.py:341-363`: HDF5 with the reference's dataset names (needs h5py), a Kaldi `<Plda>` file
        (``from_kaldi=True``, `kaldi_utils.py:24-55`), or the h5py-free ``.npz`` twin written by save_model."""
        if from_kaldi:
            from .kaldi_io import read_plda
            mu, transform, psi = read_plda(model_name)
            return TwoCovPLDA.from_arrays(mu, transform, psi, None, False, False, device)
        if str(model_name).endswith(".npz"):
            with np.load(model_name) as z:
                return TwoCovPLDA.from_arrays(z["mu"], z["transform"], z["psi"], z["offset"],
                                              bool(z["normalize_length"]), bool(z["subtract_train_set_mean"]), device)
        try:
            import h5py
        except ImportError as e:
            raise ImportError(f"{model_name}: reading the reference's HDF5 PLDA format needs h5py (not installed); "
                              "use a .npz written by TwoCovPLDA.save_model or a Kaldi <Plda> file") from e
        with h5py.File(model_name, "r") as f:
            return TwoCovPLDA.from_arrays(f.get("mu")[()], f.get("transform")[()], f.get("psi")[()],
                                          f.get("offset")[()], bool(f.get("normalize_length")[()]),
                                          bool(f.get("subtract_train_set_mean")[()]), device)

    def save_model(self, output_file_name: str):
        """`two_cov_plda.py:311-339`.  ``*.npz`` -> numpy archive at exactly that path; anything else -> HDF5 with the
        reference's dataset names / filters (so the reference's load_model reads it), which needs h5py."""
        fields = dict(mu=self.mu, transform=self.transform, psi=self.psi, offset=self.offset)
        flags = dict(normalize_length=int(self.normalize_length),
                     subtract_train_set_mean=int(self.subtract_train_set_mean))
        if str(output_file_name).endswith(".npz"):
            with open(output_file_name, "wb") as f:   # a file object: np.savez never appends ".npz" to it
                np.savez(f, **fields, **flags)
            return
        try:
            import h5py
        except ImportError as e:
            raise ImportError(f"{output_file_name}: writing the reference's HDF5 PLDA format needs h5py (not "
                              "installed); pass a path ending in .npz") from e
        with h5py.File(output_file_name, "w") as f:
            for k, v in fields.items():
                v = np.asarray(v)
                f.create_dataset(k, data=v, maxshape=(None,) * v.ndim, compression="gzip", fletcher32=True)
            for k, v in flags.items():
                f.create_dataset(k, data=v)

    # ------------------------------------------------------------------ device handle
    def _dev(self) -> int:
        if self._device is None:
            if not torch.cuda.is_available():
                raise _lib.B200Error("TwoCovPLDA scoring needs a CUDA device (no CPU fallback)")
            self._device = torch.cuda.current_device()
        return int(self._device)

    def _handle(self):
        if self._h is None:
            L = _lib.load()
            h = _lib.c_plda_p()
            mu = np.ascontiguousarray(self.mu, dtype=np.float64)
            A = np.ascontiguousarray(self.transform, dtype=np.float64)
            psi = np.ascontiguousarray(self.psi, dtype=np.float64)
            off = np.ascontiguousarray(self.offset, dtype=np.float64)
            _lib.check(L.ws_plda_create(self.dim, mu.ctypes.data, A.ctypes.data, psi.ctypes.data, off.ctypes.data,
                                        int(self.normalize_length), self._dev(), C.byref(h)), "ws_plda_create")
            self._h = h
        return self._h

    def __del__(self):
        try:
            if self._h is not None:
                _lib.load().ws_plda_destroy(self._h)
        except Exception:
            pass

    def _cuda(self, x, dtype):
        t = x if torch.is_tensor(x) else torch.from_numpy(np.ascontiguousarray(x))
        return t.to(device=torch.device("cuda", self._dev()), dtype=dtype).contiguous()

    # ------------------------------------------------------------------ batched GPU API
    def transform_batch(self, embeddings, mean_vec=None, pre_norm: bool | None = None) -> torch.Tensor:
        """(N,D) fp32 embeddings -> fp64 CUDA (N,D): ``transform_embedding(pre(x - mean_vec))`` where pre is the
        sqrt(D) length-norm (default: iff normalize_length, as eval_sv :225-241 does; transform_embedding :156-163)."""
        if pre_norm is None:
            pre_norm = bool(self.normalize_length)
        x = self._cuda(embeddings, torch.float32)
        if x.dim() == 1:
            x = x[None]
        y = torch.empty(x.shape, dtype=torch.float64, device=x.device)
        mv = None
        if mean_vec is not None:
            mv = np.ascontiguousarray(mean_vec, dtype=np.float64)
        with torch.cuda.device(self._dev()):
            _lib.check(_lib.load().ws_plda_transform(self._handle(), x.data_ptr(), x.shape[0],
                                                     mv.ctypes.data if mv is not None else None, int(pre_norm),
                                                     y.data_ptr(),
                                                     _lib.cur_stream_ptr(self._dev())), "ws_plda_transform")
        return y

    def score_matrix(self, enroll_t, test_t, counts=1, out: torch.Tensor | None = None,
                     out_dtype=torch.float32) -> torch.Tensor:
        """All-pairs LLR (N,M).  ``counts`` = int (constant n, K=D GEMM) or (N,) int array (K=2D GEMM).
        ``out``: a float32 or float64 (N,M) CUDA tensor on this PLDA's device whose rows are unit-stride and do not
        overlap (stride(1) == 1, stride(0) >= M); the kernel writes it through its data pointer and row stride."""
        N, M = int(enroll_t.shape[0]), int(test_t.shape[0])
        if out is not None:
            self._check_out(out, N, M)
        e = self._cuda(enroll_t, torch.float64)
        t = self._cuda(test_t, torch.float64)
        if out is None:
            out = torch.empty((N, M), dtype=out_dtype, device=e.device)
        if N == 0 or M == 0:
            return out
        cnt, const_n = None, 1
        if np.isscalar(counts) or (torch.is_tensor(counts) and counts.dim() == 0):
            const_n = int(counts)
        else:
            cnt = self._cuda(counts, torch.int32)
        with torch.cuda.device(self._dev()):
            _lib.check(_lib.load().ws_plda_score_matrix(
                self._handle(), e.data_ptr(), cnt.data_ptr() if cnt is not None else None, const_n, N, t.data_ptr(),
                M, out.data_ptr(), 1 if out.dtype == torch.float64 else 0, out.stride(0),
                _lib.cur_stream_ptr(self._dev())), "ws_plda_score_matrix")
        return out

    def _check_out(self, out, N, M):
        """Refuse an ``out`` the kernel would write wrongly: another dtype would be written as fp32, fewer rows or
        overlapping rows past or over other data, a non-unit column stride in the wrong layout, a host or other-device
        tensor through a pointer the kernel cannot use."""
        if out.dtype not in (torch.float32, torch.float64):
            raise ValueError(f"score_matrix: out must be float32 or float64, got {out.dtype}")
        if tuple(out.shape) != (N, M):
            raise ValueError(f"score_matrix: out has shape {tuple(out.shape)}, the scores are ({N}, {M})")
        if out.stride(1) != 1 or out.stride(0) < M:
            raise ValueError(f"score_matrix: out needs stride(1) == 1 and stride(0) >= {M}, got strides {out.stride()}")
        dev = self._dev()
        if not out.is_cuda or out.device.index != dev:
            raise ValueError(f"score_matrix: out is on {out.device}, this PLDA scores on cuda:{dev}")

    def score_trials(self, enroll_t, test_t, enroll_idx, test_idx, counts=1) -> torch.Tensor:
        e = self._cuda(enroll_t, torch.float64)
        t = self._cuda(test_t, torch.float64)
        ei = self._cuda(enroll_idx, torch.int64)
        ti = self._cuda(test_idx, torch.int64)
        out = torch.empty((ei.shape[0],), dtype=torch.float64, device=e.device)
        cnt, const_n = None, 1
        if np.isscalar(counts):
            const_n = int(counts)
        else:
            cnt = self._cuda(counts, torch.int32)
        with torch.cuda.device(self._dev()):
            _lib.check(_lib.load().ws_plda_score_trials(
                self._handle(), e.data_ptr(), cnt.data_ptr() if cnt is not None else None, const_n, e.shape[0],
                t.data_ptr(), t.shape[0], ei.data_ptr(), ti.data_ptr(), ei.shape[0], out.data_ptr(),
                _lib.cur_stream_ptr(self._dev())), "ws_plda_score_trials")
        return out

    # ------------------------------------------------------------------ reference-shaped scalar API
    def transform_embedding(self, embedding):
        """two_cov_plda.py:156-163 for one (D,) vector: A x + offset (+ length-norm), fp64 throughout; like the reference,
        callers pre-normalise with norm_embeddings themselves (eval_sv :225-241)."""
        x = np.asarray(embedding, dtype=np.float64)
        return self.transform_batch64(x[None], pre_norm=False).cpu().numpy()[0]

    def log_likelihood_ratio(self, transformed_train_embedding, transformed_test_embedding, n):
        """two_cov_plda.py:165-184 for one trial (runs the same device kernel with one trial)."""
        e = np.asarray(transformed_train_embedding, dtype=np.float64)[None]
        t = np.asarray(transformed_test_embedding, dtype=np.float64)[None]
        cnt = np.asarray([int(n)], dtype=np.int32)
        return float(self.score_trials(e, t, np.zeros(1, np.int64), np.zeros(1, np.int64), cnt).cpu()[0])

    def transform_batch64(self, x64, pre_norm: bool | None = None) -> torch.Tensor:
        """fp64 twin of transform_batch for rows that are already mean-subtracted (speaker means of eval_sv)."""
        if pre_norm is None:
            pre_norm = bool(self.normalize_length)
        x = self._cuda(x64, torch.float64)
        if x.dim() == 1:
            x = x[None]
        y = torch.empty(x.shape, dtype=torch.float64, device=x.device)
        with torch.cuda.device(self._dev()):
            _lib.check(_lib.load().ws_plda_transform64(self._handle(), x.data_ptr(), x.shape[0], int(pre_norm),
                                                       y.data_ptr(), _lib.cur_stream_ptr(self._dev())),
                       "ws_plda_transform64")
        return y

    def adapt(self, adapt_scp, ac_scale=0.5, wc_scale=0.5):
        """`two_cov_plda.py:258-309` (unsupervised adaptation; algebra in plda_train.adapt)."""
        from .plda_train import adapt_model
        return adapt_model(self, adapt_scp, ac_scale, wc_scale)

    def eval_sv(self, enroll_scp, enroll_utt2spk, test_scp, trials, score_file, multisession_avg=True,
                indomain_scp=None):
        """`two_cov_plda.py:186-256` with the per-embedding transform loop and the per-trial LLR loop replaced by
        device launches.  The host part restates the reference's numpy lines on the parsed vectors with the SAME dtype
        flow (`value - mean_vec`, per-speaker `np.mean(value, 0)`: float32 data stays float32 when an in-domain mean is
        given, becomes float64 against the default `np.zeros` mean), and everything from the length-norm on is fp64 on
        the device."""
        enroll = read_vec_scp_file(enroll_scp)
        labels = read_label_file(enroll_utt2spk)
        test = read_vec_scp_file(test_scp)
        if indomain_scp is not None:
            mean_vec = np.vstack(list(read_vec_scp_file(indomain_scp).values())).mean(0)   # :203-206
        else:
            mean_vec = np.zeros(self.dim)
        spk_sessions = {}
        for key, vec in enroll.items():                                                    # get_data_for_plda
            if key in labels:
                spk_sessions.setdefault(labels[key], []).append(vec)
            else:
                print("WARNING: {} not in utt2spk ({}), skipping it.".format(key, enroll_utt2spk))
        spks = list(spk_sessions)
        counts = np.array([1 if multisession_avg else len(spk_sessions[s]) for s in spks], dtype=np.int32)  # :213-217
        spk_mean = np.stack([np.mean(np.vstack(spk_sessions[s]) - mean_vec, 0) for s in spks]).astype(np.float64)
        tkeys = list(test)
        test_rows = np.stack([test[k] - mean_vec for k in tkeys]).astype(np.float64)       # :236
        e_t = self.transform_batch64(spk_mean)
        t_t = self.transform_batch64(test_rows)
        sidx = {s: i for i, s in enumerate(spks)}
        tidx = {k: i for i, k in enumerate(tkeys)}
        lines, ei, ti = [], [], []
        with open(trials) as f:
            for line in f:
                seg = line.strip().split()
                lines.append(seg)
                ei.append(sidx[seg[0]])
                ti.append(tidx[seg[1]])
        scores = self.score_trials(e_t, t_t, np.asarray(ei, np.int64), np.asarray(ti, np.int64), counts).cpu().numpy()
        with open(score_file, "w") as w:
            for seg, sc in zip(lines, scores):
                w.write("{} {} {:.5f} {}\n".format(seg[0], seg[1], sc, seg[2]))
