"""Every compiled instance of the front-end and fp64 scoring kernels, checked against fp64 references with per-element
error bounds.

  * fbank (ws_fbank.cu): fbank_kernel<NFFT, NG> for NFFT in {256, 512} (8 / 16 kHz) and NG = ceil(bins / 32) in 1..4,
    empty mel filters, partial 8-frame blocks, scalar sample loads, the ragged entry point; CMN (cmn_kernel).
  * fp64 GEMM (ws_plda.cu): the FFMA-style dgemm_nt_kernel and the DMMA (fp64 mma.sync) kernel through transform_batch,
    transform_batch64, score_matrix (constant and per-speaker counts, fp32 / fp64 out, contiguous and strided out),
    score_trials and the AS-norm cohort statistics; tile tails and the DMMA scalar-store fallbacks.
  * top-N selection (ws_select.cuh, topn_stats_kernel): exact scores chosen so that ties, signed zeros and keys sharing
    their top 8 / 16 / 24 bits are pinned, at top_n below, at and above M.

Each GPU test prints the worst error / bound ratio of every branch it reaches (pytest -s).  The CPU tests prove that the
checkers reject plausible kernel bugs, that the branch map below is reached by the cases, and that score_matrix refuses an
`out` the kernel would write wrongly."""
import ctypes as C
import json
import math

import numpy as np
import pytest
import torch

from oracle import fbank_np, plda_np
from wespeaker_b200 import frontend, lib, score, synthetic as syn
from wespeaker_b200.plda import TwoCovPLDA

DEV = "cuda:0"
U32, U64 = 2.0 ** -24, 2.0 ** -53
EPS32 = float(fbank_np.EPS)
LOG_EPS32 = np.float32(math.log(EPS32))
WORST = {}      # branch key -> worst error / bound ratio over the cases run


def _note(key, ratio):
    WORST[key] = max(WORST.get(key, 0.0), float(ratio))


@pytest.fixture(scope="module", autouse=True)
def _print_worst():
    yield
    if WORST:
        print("\nworst error / bound per branch:", json.dumps({k: round(v, 4) for k, v in sorted(WORST.items())}))


# ============================================================================================== branch map
# Python mirrors of the host-side dispatch predicates.  A case names the branches it takes; test_branch_map_is_covered
# fails when a threshold moves and no case reaches a branch any more.
BRANCHES = {
    *(f"fbank:NFFT={n},NG={g}" for n in (256, 512) for g in (1, 2, 3, 4)),
    "fbank:empty-filter", "fbank:partial-block", "fbank:scalar-load", "fbank:ragged-tail", "cmn:T=1", "cmn:T>8",
    "dgemm:simt", "dgemm:dmma", "dgemm:simt-single-kstep", "dgemm:simt-tail", "dgemm:dmma-tail",
    "dgemm:f32-scalar-store", "dgemm:f64-scalar-store", "dgemm:dmma-odd-M",
    "select:ties-straddle", "select:top_n>=M", "select:top_n>M", "select:M=1", "select:top24-equal",
    "select:signed-zero", "select:ragged-tiles",
}


def fbank_branches(rate, bins, T, nsamples, B, ragged=False):
    """launch_fbank (ws_fbank.cu:242-246): NFFT from the rate (:264-266), NG = ceil(bins / 32) (:244-245), 8 frames per block
    (:242); ld_sample2 (ws_fbank.cu:39-40) takes scalar loads when a row starts at an odd sample (row b at b * nsamples);
    empty filters are the len = 0 rows of fbank_tables (ws_engine.cu:175); frames behind lens[b] return early (:99)."""
    nfft = 512 if rate == 16000 else 256
    out = {f"fbank:NFFT={nfft},NG={(bins + 31) // 32}"}
    if T % 8:
        out.add("fbank:partial-block")
    if B > 1 and nsamples % 2:
        out.add("fbank:scalar-load")
    if (kernel_mel_table(rate, bins) == 0).all(axis=1).any():
        out.add("fbank:empty-filter")
    if ragged:
        out.add("fbank:ragged-tail")
    return out


def dgemm_branches(K, rows, cols, out_ld, out_f64, simt_env=False):
    """ws_launch_dgemm_nt (ws_plda.cu:304-328): DMMA when K % 16 == 0 and the operands are 16-byte aligned (always so for
    the device buffers the entry points pass) unless WS_PLDA_SIMT is set; FFMA-style kernel otherwise, one k step when
    K <= TK = 8 (:39).  Tiles are 128 x 64 (FFMA) and 128 x 128 (DMMA).  DMMA stores a column pair with one 8- / 16-byte
    store when its address is aligned, else two scalar stores (:183-188): with an odd out_ld, odd rows are misaligned."""
    dmma = K % 16 == 0 and not simt_env
    out = {"dgemm:dmma" if dmma else "dgemm:simt"}
    if dmma:
        if rows % 128 or cols % 128:
            out.add("dgemm:dmma-tail")
        if cols % 2:
            out.add("dgemm:dmma-odd-M")
        if out_ld % 2 and rows > 1 and cols > 1:
            out.add("dgemm:f64-scalar-store" if out_f64 else "dgemm:f32-scalar-store")
    else:
        if K <= 8:
            out.add("dgemm:simt-single-kstep")
        if rows % 128 or cols % 64:
            out.add("dgemm:simt-tail")
    return out


def select_branches(M, top_n, pattern, rows, tile_rows):
    """ws_score_cohort_stats (ws_score.cu:145-163): n_eff = min(top_n, M) (:153), tiles of tile_rows rows (:156-160);
    radix_select_kth (ws_select.cuh:18-49) splits a tie group at the n-th position through *ties."""
    out = set()
    if M == 1:
        out.add("select:M=1")
    if top_n >= M:
        out.add("select:top_n>=M")
    if top_n > M:
        out.add("select:top_n>M")
    if rows % tile_rows:
        out.add("select:ragged-tiles")
    out |= {"straddle": {"select:ties-straddle"} if min(top_n, M) < M else set(), "bits24": {"select:top24-equal"},
            "pm0": {"select:signed-zero"}}.get(pattern, set())
    return out


# ============================================================================================== 1. fbank
FB_BINS = (4, 23, 32, 33, 64, 65, 72, 96, 97, 120, 128)
FB_CASES = [(r, b, "hamming") for r in (8000, 16000) for b in FB_BINS]
FB_CASES += [(r, b, w) for r in (8000, 16000) for w, bs in (("povey", (4, 64, 72, 128)), ("hanning", (23, 33, 96, 97)),
                                                             ("rectangular", (32, 65, 96, 120))) for b in bs]
FB_T = 97                                           # 97 = 12 * 8 + 1: the last 8-frame block holds one frame
FB_B = 3
_libm = C.CDLL("libm.so.6")
_libm.logf.restype, _libm.logf.argtypes = C.c_float, [C.c_float]
_TABLES = {}


def fb_nsamples(rate, T=FB_T):
    fl, sh = frontend.frame_geometry(rate)
    return (T - 1) * sh + fl + 1                    # odd: rows 1, 3, ... of a batch start at odd samples


def kernel_mel_table(rate, bins):
    """The mel table the kernel reads, as fbank_tables (ws_engine.cu:159-176) builds it: torchaudio's get_mel_banks in
    float32, with the C library's logf.  numpy's and torch's float32 log differ from it by one ulp at a few FFT bins
    (pinned by test_kernel_mel_table_is_torchaudios), which moves those weights by up to ~1e-5; the error bound below is
    for the kernel's arithmetic, so the reference uses the table the kernel was given.  (bins, Nfft / 2) float64."""
    key = (rate, bins)
    if key not in _TABLES:
        nfft = 512 if rate == 16000 else 256
        f32 = np.float32
        mel_low, mel_high = 1127.0 * math.log(1.0 + 20.0 / 700.0), 1127.0 * math.log(1.0 + 0.5 * rate / 700.0)
        delta, lowf, bw = f32((mel_high - mel_low) / (bins + 1)), f32(mel_low), f32(rate) / f32(nfft)
        arg = f32(1.0) + (bw * np.arange(nfft // 2, dtype=f32)) / f32(700.0)
        mel = f32(1127.0) * np.array([_libm.logf(float(a)) for a in arg], dtype=f32)
        m = np.arange(bins, dtype=f32)[:, None]
        left, center, right = lowf + m * delta, lowf + (m + f32(1.0)) * delta, lowf + (m + f32(2.0)) * delta
        w = np.maximum(f32(0.0), np.minimum((mel - left) / (center - left), (right - mel) / (right - center)))
        _TABLES[key] = w.astype(np.float64)
    return _TABLES[key]


# Error model of one frame.  The kernel works in fp32 (unit roundoff u = 2^-24):
#  * front end: y_n = w_n ((x_n - mu) - 0.97 (x_{n-1} - mu)).  Integer samples and their sums are exact; the mean, the two
#    subtractions, the product with the fp32 constant 0.97f (0.97 (1 + 3e-8)) and the window product each cost <= u of
#    the magnitude they touch, so |dy_n| <~ 3 u s_n with s_n = w_n (|x_n - mu| + |x_{n-1} - mu|).  An error vector dy
#    reaches each FFT bin with unit-modulus weights: RMS over bins ||dy||_2, i.e. ~3 u ||s||_2.
#  * FFT: log2(Nfft) butterfly levels (R-point register DIF, 32-point shuffle DIF, split step), each rounding every value
#    to ~u of its size with twiddles good to ~u; by Parseval each level's values have the norm of y, so the per-bin error
#    grows like u sqrt(log2 Nfft) ||y||_2 in RMS and is below u log2(Nfft) ||y||_2 in all but a vanishing fraction of bins.
#  Hence the per-bin bound  delta = C_FFT u (log2(Nfft) ||y||_2 + ||s||_2).  C_FFT = 4 leaves a factor >= 2 over the worst
#  bin of a plain fp32 pipeline (torch.fft, test_fp32_pipeline_meets_the_bound) and over the kernel on the H100, while it
#  keeps the bound ~100x below the change of a dropped edge tap of the widest filter (16 kHz / 4 bins: 175 taps).
#  * power: |P^_k - P_k| <= 2 |X_k| delta + delta^2, plus 2 u P_k for squaring and adding in fp32;
#  * mel sum: a chain of len_m fp32 FMAs: <= len_m u sum_k w_mk P_k.
#  So E_m = sum_k w_mk (2 |X_k| delta + delta^2) + (len_m + 2) u e_m, and the fp32 log output must lie in
#  [log max(e_m - E_m, eps), log max(e_m + E_m, eps)] widened by 2 ulp32 (logf is good to 1 ulp, the store rounds): an
#  element whose energy is within E_m of the eps floor may come out on either side of it.  An empty filter (len 0) must
#  give exactly float32(log(eps)).
C_FFT = 4.0


def fbank_ref(wav, rate, bins, wt, W=None):
    """fp64 energies e (T, bins) and their bounds E of one waveform with mel table W (default: the kernel's); restates
    fbank_np.fbank(dtype=np.float64), test_fbank_ref_is_the_oracle pins the two together."""
    fl, sh = frontend.frame_geometry(rate)
    nfft = 512 if rate == 16000 else 256
    wav = np.asarray(wav, dtype=np.float64)
    T = 1 + (wav.shape[0] - fl) // sh
    fr = wav[np.arange(T)[:, None] * sh + np.arange(fl)[None, :]]
    xc = fr - fr.mean(axis=1, keepdims=True)
    prev = np.concatenate([xc[:, :1], xc[:, :-1]], axis=1)
    win = fbank_np.window(wt, fl).astype(np.float64)
    y = (xc - 0.97 * prev) * win
    s = win * (np.abs(xc) + np.abs(prev))
    X = np.fft.rfft(y, n=nfft, axis=1)[:, :nfft // 2]
    W = kernel_mel_table(rate, bins) if W is None else W
    e = (np.abs(X) ** 2) @ W.T
    d = C_FFT * U32 * (math.log2(nfft) * np.linalg.norm(y, axis=1) + np.linalg.norm(s, axis=1))[:, None]
    lens = (W > 0).sum(axis=1)
    E = (2.0 * np.abs(X) * d + d * d) @ W.T + (lens + 2) * U32 * e
    return e, E


def fbank_ratio(out, e, E, W):
    """worst error / bound ratio of one (T, bins) fp32 output against fp64 energies e with bounds E (inf: an empty filter
    that is not exactly float32(log(eps)), or a non-finite output)"""
    out = np.asarray(out)
    empty = (W == 0).all(axis=1)
    if empty.any() and not (out[:, empty] == LOG_EPS32).all():
        return math.inf
    o, e, E = out[:, ~empty].astype(np.float64), e[:, ~empty], E[:, ~empty]
    if not np.isfinite(o).all():
        return math.inf
    ref = np.log(np.maximum(e, EPS32))
    tol = 2.0 * np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64)
    hi = np.log(np.maximum(e + E, EPS32)) - ref + tol
    lo = ref - np.log(np.maximum(e - E, EPS32)) + tol
    r = np.where(o >= ref, (o - ref) / hi, (ref - o) / lo)
    return float(r.max()) if r.size else 0.0


def fb_wavs(rate, n=None, B=FB_B, seed=11):
    return syn.make_wavs(B, n or fb_nsamples(rate), seed=seed + rate // 1000)


# ---------------------------------------------------------------------------------------------- CPU: model and checker
def test_kernel_mel_table_is_torchaudios():
    """the kernel's table (C logf) and the oracle's (numpy float32 log) have the same filters, the same empty filters and
    differ by at most one ulp of the mel value at a few bins"""
    for rate in (8000, 16000):
        for bins in FB_BINS:
            a = kernel_mel_table(rate, bins)
            b = fbank_np.mel_banks(bins, 512 if rate == 16000 else 256, rate)[:, :-1].astype(np.float64)
            assert ((a > 0) == (b > 0)).all(), (rate, bins)
            assert np.abs(a - b).max() < 3e-5, (rate, bins)
    # the empty filters (len-0 table rows) and the widest filter the cases rely on
    empties = {(r, b): int((kernel_mel_table(r, b) == 0).all(axis=1).sum()) for r in (8000, 16000) for b in FB_BINS}
    assert empties[(8000, 96)] == 1 and empties[(8000, 97)] == 1 and empties[(8000, 120)] == 3
    assert empties[(8000, 128)] == 4 and empties[(16000, 128)] == 1
    assert (kernel_mel_table(16000, 4) > 0).sum(axis=1).max() == 175


def test_fbank_ref_is_the_oracle():
    """fbank_ref with the oracle's table is fbank_np.fbank in fp64"""
    w = fb_wavs(8000, B=1)[0]
    for rate, bins, wt in ((8000, 97, "povey"), (16000, 4, "hamming")):
        W = fbank_np.mel_banks(bins, 512 if rate == 16000 else 256, rate)[:, :-1].astype(np.float64)
        e, _ = fbank_ref(w, rate, bins, wt, W)
        want = fbank_np.fbank(w, bins, sample_frequency=rate, window_type=wt, dtype=np.float64)
        assert np.abs(np.log(np.maximum(e, EPS32)) - want).max() < 1e-9


def _fp32_pipeline(wav, rate, bins, wt):
    """a plain fp32 implementation: fp32 framing and pre-emphasis, torch.fft.rfft in fp32, fp32 mel products"""
    fl, sh = frontend.frame_geometry(rate)
    nfft = 512 if rate == 16000 else 256
    x = torch.from_numpy(np.asarray(wav, np.float32))
    T = 1 + (x.shape[0] - fl) // sh
    fr = x[torch.arange(T)[:, None] * sh + torch.arange(fl)[None, :]]
    xc = fr - fr.mean(dim=1, keepdim=True)
    prev = torch.cat([xc[:, :1], xc[:, :-1]], dim=1)
    y = (xc - 0.97 * prev) * torch.from_numpy(fbank_np.window(wt, fl))
    P = torch.fft.rfft(y, n=nfft, dim=1)[:, :nfft // 2].abs() ** 2
    e = P @ torch.from_numpy(kernel_mel_table(rate, bins).astype(np.float32)).T
    return torch.log(torch.clamp(e, min=EPS32)).numpy()


@pytest.mark.parametrize("rate,bins,wt", [(8000, 97, "hamming"), (16000, 4, "povey"), (16000, 128, "rectangular")])
def test_fp32_pipeline_meets_the_bound(rate, bins, wt):
    """the bound is not tighter than fp32 arithmetic: an ordinary fp32 pipeline meets it with margin, and so does the
    fp64 reference rounded to fp32"""
    W = kernel_mel_table(rate, bins)
    for w in fb_wavs(rate):
        e, E = fbank_ref(w, rate, bins, wt)
        rounded = np.log(np.maximum(e, EPS32)).astype(np.float32)
        rounded[:, (W == 0).all(axis=1)] = LOG_EPS32
        assert fbank_ratio(rounded, e, E, W) <= 0.5
        r = fbank_ratio(_fp32_pipeline(w, rate, bins, wt), e, E, W)
        print(f"fp32 pipeline {rate} Hz {bins} bins {wt}: worst error / bound {r:.3f}")
        assert r <= 0.5


def _mutants(rate, bins, wt, w):
    """(name, output) of plausible kernel bugs, computed exactly and rounded to fp32"""
    W = kernel_mel_table(rate, bins)
    e, _ = fbank_ref(w, rate, bins, wt)

    def out_of(e2):
        o = np.log(np.maximum(e2, EPS32)).astype(np.float32)
        o[:, (W == 0).all(axis=1)] = LOG_EPS32
        return o

    def energies(W2):
        return fbank_ref(w, rate, bins, wt, W2)[0]
    out = []
    lens = (W > 0).sum(axis=1)
    m = int(np.argmax(lens))                                      # the widest filter loses its last tap
    W2 = W.copy()
    W2[m, np.nonzero(W[m])[0][-1]] = 0.0
    out.append(("last tap of the widest filter dropped", out_of(energies(W2))))
    if bins > 32:                                                 # lane owning the wrong bin across an NG boundary
        o = out_of(e)
        o[:, [1, 33]] = o[:, [33, 1]]
        out.append(("bins 1 and 33 swapped", o))
    W3 = W.copy()
    m3 = int(np.nonzero(lens)[0][len(np.nonzero(lens)[0]) // 2])
    W3[m3] = np.roll(W[m3], 1)
    out.append(("one filter's start shifted by one FFT bin", out_of(energies(W3))))
    empty = np.nonzero(lens == 0)[0]
    if len(empty):
        o = out_of(e)
        o[:, empty[0]] = 0.0
        out.append(("empty filter giving 0", o))
    o = out_of(e)
    o[5] = o[6]
    out.append(("frame 5 computed from frame 6's samples", o))
    return out


@pytest.mark.parametrize("rate,bins,wt", [(8000, 97, "hamming"), (16000, 4, "hamming"), (16000, 72, "povey")])
def test_fbank_checker_rejects_kernel_bugs(rate, bins, wt):
    w = fb_wavs(rate, B=1)[0]
    W = kernel_mel_table(rate, bins)
    e, E = fbank_ref(w, rate, bins, wt)
    for name, o in _mutants(rate, bins, wt, w):
        r = fbank_ratio(o, e, E, W)
        print(f"{rate} Hz {bins} bins, {name}: error / bound {r:.3g}")
        assert r > 1.0, f"the fbank checker accepts: {name}"


# ---------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
@pytest.mark.parametrize("rate,bins,wt", FB_CASES)
def test_fbank_kernel_instance(rate, bins, wt):
    n = fb_nsamples(rate)
    wavs = fb_wavs(rate)
    out = frontend.fbank_batch(torch.from_numpy(wavs).to(DEV), window_type=wt, sample_rate=rate, num_mel_bins=bins).cpu().numpy()
    out16 = frontend.fbank_batch(torch.from_numpy(wavs.astype(np.int16)).to(DEV), window_type=wt, sample_rate=rate,
                                 num_mel_bins=bins).cpu().numpy()
    assert out.shape == (FB_B, FB_T, bins)
    assert np.array_equal(out16.view(np.int32), out.view(np.int32)), "int16 input differs from float input"
    W = kernel_mel_table(rate, bins)
    worst = max(fbank_ratio(out[b], *fbank_ref(wavs[b], rate, bins, wt), W) for b in range(FB_B))
    for k in fbank_branches(rate, bins, FB_T, n, FB_B):
        _note(k, worst)
    print(f"fbank {rate} Hz {bins} bins {wt}: worst error / bound {worst:.3f}")
    assert worst <= 1.0


@pytest.mark.gpu
@pytest.mark.parametrize("rate,bins", [(8000, 23), (8000, 128), (16000, 4), (16000, 97)])
def test_fbank_ragged_instance(rate, bins):
    """ws_fbank_ragged_at: each utterance's rows equal the utterance alone and meet the bound; rows behind its end keep
    the sentinel"""
    fl, sh = frontend.frame_geometry(rate)
    ns = [fl, fl + 9 * sh + 3, fl + 40 * sh + 1, fl + 16 * sh]
    wavs = [syn.make_wavs(1, n, seed=80 + i)[0] for i, n in enumerate(ns)]
    nf = [frontend.num_frames(n, rate) for n in ns]
    T = max(nf)
    flat = torch.from_numpy(np.concatenate(wavs)).to(DEV)
    offs = torch.from_numpy(np.concatenate([[0], np.cumsum(ns)[:-1]]).astype(np.int64)).to(DEV)
    nfd = torch.tensor(nf, dtype=torch.int32, device=DEV)
    out = torch.full((len(ns), T, bins), -7.0, device=DEV)
    L = lib.load()
    lib.check(L.ws_fbank_ragged_at(flat.data_ptr(), 0, flat.numel(), offs.data_ptr(), nfd.data_ptr(), T, len(ns), b"hamming",
                                   rate, bins, out.data_ptr(), lib.cur_stream_ptr(0)), "ws_fbank_ragged_at")
    out = out.cpu().numpy()
    W = kernel_mel_table(rate, bins)
    worst = 0.0
    for i, w in enumerate(wavs):
        alone = frontend.fbank_batch(torch.from_numpy(w[None]).to(DEV), sample_rate=rate, num_mel_bins=bins).cpu().numpy()[0]
        assert np.array_equal(out[i, :nf[i]], alone)
        assert (out[i, nf[i]:] == -7.0).all(), "a row behind the utterance's end was written"
        worst = max(worst, fbank_ratio(out[i, :nf[i]], *fbank_ref(w, rate, bins, "hamming"), W))
    for k in fbank_branches(rate, bins, T, 0, 1, ragged=True):
        _note(k, worst)
    print(f"ragged fbank {rate} Hz {bins} bins: worst error / bound {worst:.3f}")
    assert worst <= 1.0


# ============================================================================================== 2. CMN
CMN_BINS = (4, 23, 33, 72, 97, 128)
CMN_T = (1, 7, 8, 9, 1001)


def cmn_ratio(x, got):
    """cmn_kernel sums each bin over T in fp32 (T / 8 per thread, then 8 partials: depth <= T) and divides by T, so the
    mean is within T u max_t |x| of the fp64 mean; the subtraction rounds to the output's ulp."""
    x = np.asarray(x, np.float64)
    ref = x - x.mean(axis=0, keepdims=True)
    bound = x.shape[0] * U32 * np.abs(x).max(axis=0, keepdims=True) + np.spacing(np.abs(ref).astype(np.float32))
    return float((np.abs(got.astype(np.float64) - ref) / bound).max())


def test_cmn_checker_rejects_kernel_bugs():
    x = np.random.default_rng(0).normal(5.0, 3.0, (9, 7)).astype(np.float32)
    ref = (x - x.astype(np.float64).mean(axis=0)).astype(np.float32)
    assert cmn_ratio(x, ref) <= 0.5
    assert cmn_ratio(x, (x - x[:8].mean(axis=0)).astype(np.float32)) > 1      # mean over T - 1 frames
    assert cmn_ratio(x, (x - x.sum(axis=0) / 8).astype(np.float32)) > 1        # divided by the block height
    assert cmn_ratio(x, x - x.mean(axis=1, keepdims=True)) > 1                  # mean over the bins


@pytest.mark.gpu
@pytest.mark.parametrize("bins", CMN_BINS)
def test_cmn(bins):
    for rate in (8000, 16000):
        fl, sh = frontend.frame_geometry(rate)
        for T in CMN_T:
            w = torch.from_numpy(syn.make_wavs(2, (T - 1) * sh + fl, seed=T)).to(DEV)
            raw = frontend.fbank_batch(w, sample_rate=rate, num_mel_bins=bins).cpu().numpy()
            got = frontend.fbank_batch(w, cmn=True, sample_rate=rate, num_mel_bins=bins).cpu().numpy()
            worst = max(cmn_ratio(raw[b], got[b]) for b in range(2))
            _note("cmn:T=1" if T == 1 else "cmn:T>8" if T > 8 else "cmn:T<=8", worst)
            assert worst <= 1.0, (rate, T, worst)


# ============================================================================================== 3. fp64 GEMM family
GEMM_D = (8, 24, 200, 16, 256)
GEMM_SHAPES = (1, 63, 64, 65, 127, 128, 129, 300)
NMAX = max(GEMM_SHAPES)
_LD = np.longdouble


class GemmRef:
    """score_matrix's refactored GEMM (ws_plda.cu:1-9) evaluated in long double, with the magnitudes its error bound needs.
    Error model of the device (fp64, u = 2^-53): each P / Q element carries a few roundings; the GEMM accumulates K
    products (depth <= K in either kernel); the row / column constants are sums of D terms of a few roundings each
    (warp-strided: depth <= D / 32 + 5), with log good to 1 ulp; the epilogue adds the three.  So
        |S^ - S| <= 2 u (K (|P| |Q|^T)_ij + D (R_i + C_j)) + u |S_ij|,
    R_i and C_j the sums of the constants' absolute terms; the factor 2 absorbs the per-element roundings of P and Q
    (<= 4 u each against K >= 8) and the epilogue's two additions.  An fp32 out is that fp64 result rounded once, so it
    may add half an ulp32 of the stored value; the ratio reported for it is the error beyond that half ulp over the fp64
    bound (a ratio of the whole error would sit at ~1 by construction, the half ulp dwarfing the fp64 error)."""

    def __init__(self, D, counts, seed=5):
        pm = syn.make_plda(D, seed=seed, normalize_length=False)
        self.pm, self.D = pm, D
        g = np.random.default_rng(seed + D)
        self.e = g.standard_normal((NMAX, D)) * 1.5
        self.t = g.standard_normal((NMAX, D)) * 1.5
        self.counts = g.integers(1, 9, NMAX).astype(np.int32) if counts == "per-speaker" else None
        self.const_n = 3 if counts == "const" else 1
        psi, e, t = pm["psi"].astype(_LD), self.e.astype(_LD), self.t.astype(_LD)
        n = (self.counts if self.counts is not None else np.full(NMAX, self.const_n)).astype(_LD)[:, None]
        m = n * psi / (n * psi + 1) * e
        v = 1 + psi / (n * psi + 1)
        rterms = np.concatenate([np.log(v), m * m / v], axis=1)
        self.rowc = -0.5 * rterms.sum(axis=1)
        cterms = [np.log(psi + 1) + 0 * t, t * t / (psi + 1)]
        if self.counts is None:
            self.P, self.Q = m / v, t
            cterms.append(-(t * t) / (1 + psi / (self.const_n * psi + 1)))
        else:
            self.P, self.Q = np.concatenate([m / v, -0.5 / v], axis=1), np.concatenate([t, t * t], axis=1)
        cterms = np.concatenate(cterms, axis=1)
        self.colc = 0.5 * cterms.sum(axis=1)
        self.K = self.P.shape[1]
        self.S = (self.P @ self.Q.T + self.rowc[:, None] + self.colc[None, :]).astype(np.float64)
        P64, Q64 = np.abs(self.P.astype(np.float64)), np.abs(self.Q.astype(np.float64))
        R, Cc = 0.5 * np.abs(rterms.astype(np.float64)).sum(1), 0.5 * np.abs(cterms.astype(np.float64)).sum(1)
        self.bound = 2 * U64 * (self.K * (P64 @ Q64.T) + D * (R[:, None] + Cc[None, :])) + U64 * np.abs(self.S)

    def ratio(self, got, N, M):
        S, b = self.S[:N, :M], self.bound[:N, :M]
        got = np.asarray(got)
        err = np.abs(got.astype(np.float64) - S)
        if got.dtype == np.float32:
            err = np.maximum(0.0, err - 0.5 * np.spacing(np.abs(got)).astype(np.float64))
        r = err / b
        return math.inf if not np.isfinite(r).all() else float(r.max())


def test_gemm_ref_is_the_oracle_and_checker_rejects_bugs():
    """the refactored reference equals plda_np.llr_matrix (the reference's per-trial formula); the bound rejects an fp32
    accumulation, a dropped k step, a lost row constant and a transposed tile"""
    for counts in ("const", "per-speaker"):
        g = GemmRef(24, counts)
        n = g.counts if g.counts is not None else g.const_n
        want = plda_np.llr_matrix(g.pm, g.e, g.t, n)
        assert np.abs(want - g.S).max() <= 1e-9 * np.abs(g.S).max()
        assert g.ratio(g.S, NMAX, NMAX) == 0.0
        assert g.ratio(g.S.astype(np.float32), NMAX, NMAX) <= 1.0
        P, Q = g.P.astype(np.float64), g.Q.astype(np.float64)
        rc, cc = g.rowc.astype(np.float64), g.colc.astype(np.float64)
        f32acc = (P.astype(np.float32) @ Q.astype(np.float32).T).astype(np.float64) + rc[:, None] + cc[None, :]
        assert g.ratio(f32acc, NMAX, NMAX) > 1, "fp32 accumulation accepted"
        assert g.ratio(P[:, 8:] @ Q[:, 8:].T + rc[:, None] + cc[None, :], NMAX, NMAX) > 1, "dropped k step accepted"
        assert g.ratio(P @ Q.T + cc[None, :], NMAX, NMAX) > 1, "lost row constant accepted"
        tr = g.S.copy()
        tr[:64, :64] = g.S[:64, :64].T
        assert g.ratio(tr, NMAX, NMAX) > 1, "transposed tile accepted"


_GEMM = {}


def _gemm_ref(D, counts):
    if (D, counts) not in _GEMM:
        _GEMM[(D, counts)] = GemmRef(D, counts)
    return _GEMM[(D, counts)]


def _plda(g):
    return TwoCovPLDA.from_arrays(**g.pm, device=0)


def _simt_modes(K):
    """DMMA-eligible shapes run again on the FFMA-style kernel (WS_PLDA_SIMT is read at every launch)"""
    return (False, True) if K % 16 == 0 else (False,)


@pytest.mark.gpu
@pytest.mark.parametrize("D", GEMM_D)
def test_transform_batch(D, monkeypatch):
    """y = x A^T + offset (no row constant, column constant = offset, fp64 out) through transform_batch (fp32 rows) and
    transform_batch64 (fp64 rows); bound 2 u (D (|x| |A|^T) + D |offset|) + u |y|"""
    pm = syn.make_plda(D, seed=7, normalize_length=False)
    p = TwoCovPLDA.from_arrays(**pm, device=0)
    x32 = syn.make_embeddings(NMAX, D, seed=D)
    x64 = np.random.default_rng(D).standard_normal((NMAX, D))
    A, off = pm["transform"], pm["offset"]
    for simt in _simt_modes(D):
        if simt:
            monkeypatch.setenv("WS_PLDA_SIMT", "1")
        for name, x in (("transform_batch", x32), ("transform_batch64", x64)):
            xl = x.astype(_LD)
            ref = (xl @ A.astype(_LD).T + off.astype(_LD)).astype(np.float64)
            bnd = 2 * U64 * D * (np.abs(x.astype(np.float64)) @ np.abs(A).T + np.abs(off)) + U64 * np.abs(ref)
            for N in GEMM_SHAPES:
                fn = p.transform_batch if name == "transform_batch" else p.transform_batch64
                y = fn(x[:N], pre_norm=False).cpu().numpy()
                r = float((np.abs(y - ref[:N]) / bnd[:N]).max())
                for k in dgemm_branches(D, N, D, D, True, simt):
                    _note(k, r)
                assert r <= 1.0, (name, D, N, simt, r)
        monkeypatch.delenv("WS_PLDA_SIMT", raising=False)


SM_CASES = [(D, c) for D in GEMM_D for c in ("const", "per-speaker")]


@pytest.mark.gpu
@pytest.mark.parametrize("D,counts", SM_CASES)
def test_score_matrix(D, counts, monkeypatch):
    g = _gemm_ref(D, counts)
    p = _plda(g)
    cnt = g.counts if g.counts is not None else g.const_n
    for simt in _simt_modes(g.K):
        if simt:
            monkeypatch.setenv("WS_PLDA_SIMT", "1")
        for N in GEMM_SHAPES:
            c = cnt if np.isscalar(cnt) else cnt[:N]
            for M in GEMM_SHAPES:
                for dt in (torch.float32, torch.float64):
                    got = p.score_matrix(g.e[:N], g.t[:M], c, out_dtype=dt).cpu().numpy()
                    r = g.ratio(got, N, M)
                    big = torch.full((N + 1, M + 1), float("nan"), dtype=dt, device=DEV)
                    view = big[:N, :M]                                   # row stride M + 1: odd whenever M is even
                    ret = p.score_matrix(g.e[:N], g.t[:M], c, out=view)
                    assert ret.data_ptr() == view.data_ptr()
                    bigh = big.cpu().numpy()
                    assert np.isnan(bigh[N]).all() and np.isnan(bigh[:, M]).all(), "score_matrix wrote outside out"
                    rv = g.ratio(bigh[:N, :M], N, M)
                    f64 = dt == torch.float64
                    for k in dgemm_branches(g.K, N, M, M, f64, simt):
                        _note(k, r)
                    for k in dgemm_branches(g.K, N, M, M + 1, f64, simt):
                        _note(k, rv)
                    assert r <= 1.0 and rv <= 1.0, (D, counts, N, M, dt, simt, r, rv)
        monkeypatch.delenv("WS_PLDA_SIMT", raising=False)


@pytest.mark.gpu
@pytest.mark.parametrize("D,counts", SM_CASES)
def test_score_trials_matches_score_matrix(D, counts):
    """score_trials over ~1000 pairs, first and last rows included, meets the bound and matches score_matrix"""
    g = _gemm_ref(D, counts)
    p = _plda(g)
    rng = np.random.default_rng(D)
    ei = np.concatenate([[0, NMAX - 1, 0, NMAX - 1], rng.integers(0, NMAX, 1000)]).astype(np.int64)
    ti = np.concatenate([[0, NMAX - 1, NMAX - 1, 0], rng.integers(0, NMAX, 1000)]).astype(np.int64)
    cnt = g.counts if g.counts is not None else g.const_n
    got = p.score_trials(g.e, g.t, ei, ti, cnt).cpu().numpy()
    mat = p.score_matrix(g.e, g.t, cnt, out_dtype=torch.float64).cpu().numpy()
    b = g.bound[ei, ti]
    r = float((np.abs(got - g.S[ei, ti]) / b).max())
    _note("trials", r)
    assert r <= 1.0
    assert (np.abs(got - mat[ei, ti]) <= 2 * b).all()


# ============================================================================================== 4. top-N selection, exact
SEL_M = (1, 2, 255, 256, 257, 4097, 100003)
SEL_PATTERNS = ("equal", "straddle", "pm0", "bits8", "bits16", "bits24", "negative")


def sel_topns(M):
    return sorted({1, M - 1, M, M + 7} - {0})


def _key_pattern(rng, M, keep_bits):
    """positive fp32 values whose order keys agree in their top keep_bits bits (the key of a positive float is its bit
    pattern with the sign bit set, so the float's top keep_bits - 1 bits are shared)"""
    base = np.array([0.75], np.float32).view(np.uint32)[0]
    low = 32 - (keep_bits - 1)
    u = (base & ~np.uint32((1 << low) - 1)) | rng.integers(0, 1 << low, M, dtype=np.uint32)
    return u.view(np.float32)


def sel_pattern(name, M, top_n, rng):
    """the fp64 dot products of one row (exactly representable, so the device's fp32 score is float32(value))"""
    if name == "equal":
        return np.full(M, 0.3125)
    if name == "straddle":       # a tie group around the n-th largest
        v = np.sort(rng.uniform(-1, 1, M).astype(np.float32).astype(np.float64))[::-1].copy()
        n = min(top_n, M)
        lo, hi = max(0, n - 3), min(M, n + 2)
        v[lo:hi] = v[n - 1]
        return rng.permutation(v)
    if name == "pm0":            # +-1e-300 round to +0.0f / -0.0f; some values above and below zero
        v = rng.choice([1e-300, -1e-300, 0.0, 0.5, -0.25], M)
        return v
    if name.startswith("bits"):
        return _key_pattern(rng, M, int(name[4:])).astype(np.float64)
    if name == "negative":
        return -rng.uniform(0.01, 1, M).astype(np.float32).astype(np.float64)
    raise ValueError(name)


def sel_expected(scores32, top_n):
    """mean and population std of the top min(top_n, M) fp32 scores, in long double"""
    v = np.sort(scores32.astype(_LD))[::-1][:min(top_n, scores32.shape[0])]
    mean = v.mean()
    return float(mean), float(np.sqrt(((v - mean) ** 2).mean())), v


def sel_ratio(mean, std, scores32, top_n):
    """error / bound of the device's (mean, std).  topn_stats_kernel sums the selected scores per thread (M / 256 each),
    over 32 lanes and 8 warps, then adds ties * thr: depth d <= M / 256 + 16, so the mean is within (d + 2) u sum|v| / n.
    var = sum v^2 / n - mean^2 is within delta = (3 d + 8) u sum v^2 / n (the cancellation of the two terms is the bulk of
    it), and the std within min(sqrt(delta), delta / std) + 2 u std."""
    _, _, v = sel_expected(scores32, top_n)
    n = v.shape[0]
    m_ref, s_ref = float(v.mean()), float(np.sqrt(((v - v.mean()) ** 2).mean()))
    d = math.ceil(scores32.shape[0] / 256) + 16
    bm = (d + 2) * U64 * float(np.abs(v).sum()) / n + 1e-300
    delta = (3 * d + 8) * U64 * float((v * v).sum()) / n
    bs = (min(math.sqrt(delta), delta / s_ref) if s_ref > 0 else math.sqrt(delta)) + 2 * U64 * s_ref + 1e-300
    return max(abs(mean - m_ref) / bm, abs(std - s_ref) / bs)


def test_select_checker_rejects_kernel_bugs():
    rng = np.random.default_rng(3)
    for M in (257, 4097):
        for pattern in ("bits24", "straddle"):
            s = sel_pattern(pattern, M, 100, rng).astype(np.float32)
            m, sd, v = sel_expected(s, 100)
            assert sel_ratio(m, sd, s, 100) == 0.0
            srt = np.sort(s.astype(np.float64))[::-1]
            if pattern == "bits24":   # the (n+1)-th value in place of the n-th (a key compared on its top 24 bits only)
                k = int(np.nonzero(srt[:100] != srt[100])[0].max())     # last of the top 100 that differs from the 101st
                w = np.concatenate([srt[:k], srt[k + 1:101]])
                assert sel_ratio(w.mean(), w.std(), s, 100) > 1
            else:                     # a tie group counted once
                u = np.unique(srt[:100])
                w = np.concatenate([u, srt[srt < srt[99]][:100 - u.size]])
                assert sel_ratio(w.mean(), w.std(), s, 100) > 1
    s = rng.uniform(-1, 1, 50).astype(np.float32)
    assert sel_ratio(s.astype(np.float64).sum() / 57, s.astype(np.float64).std(), s, 57) > 1   # divided by top_n > M


@pytest.mark.gpu
@pytest.mark.parametrize("D", (16, 24))
@pytest.mark.parametrize("M", SEL_M)
def test_topn_selection_exact(M, D):
    """rows e_r of the identity, cohort row j = sum_r s_rj e_r: every dot product is exactly s_rj in any summation order,
    so each row of the fp32 score tile holds the chosen pattern; several rows per call in ragged tiles"""
    dev = torch.device(DEV)
    rows = len(SEL_PATTERNS)
    tile_rows = 3
    for top_n in sel_topns(M):
        rng = np.random.default_rng(M * 31 + top_n)
        S = np.stack([sel_pattern(p, M, top_n, rng) for p in SEL_PATTERNS])
        unit = torch.eye(rows, D, dtype=torch.float64, device=dev)
        coh = np.zeros((M, D))
        coh[:, :rows] = S.T
        mean, std = score._cohort_stats(unit, torch.from_numpy(coh).to(dev), top_n, dev, tile_bytes=tile_rows * 4 * M)
        mean, std = mean.cpu().numpy(), std.cpu().numpy()
        for r, p in enumerate(SEL_PATTERNS):
            s32 = S[r].astype(np.float32)
            ratio = sel_ratio(float(mean[r]), float(std[r]), s32, top_n)
            for k in select_branches(M, top_n, p, rows, tile_rows) | dgemm_branches(D, rows, M, M, False):
                _note(k, ratio)
            assert ratio <= 1.0, (M, D, top_n, p, mean[r], std[r], sel_expected(s32, top_n)[:2])


# ============================================================================================== 5. score_matrix `out`
def _cpu_plda(D=8):
    return TwoCovPLDA.from_arrays(**syn.make_plda(D, seed=1, normalize_length=False))


@pytest.mark.parametrize("bad,match", [
    pytest.param(lambda N, M: torch.empty((N, M), dtype=torch.float16), "float32 or float64", id="fp16"),
    pytest.param(lambda N, M: torch.empty((N, M), dtype=torch.bfloat16), "float32 or float64", id="bf16"),
    pytest.param(lambda N, M: torch.empty((N - 1, M), dtype=torch.float32), "shape", id="short"),
    pytest.param(lambda N, M: torch.empty((N, M + 1), dtype=torch.float64), "shape", id="wide"),
    pytest.param(lambda N, M: torch.empty((M, N), dtype=torch.float32).t(), "stride", id="transposed"),
    pytest.param(lambda N, M: torch.empty((N, 2 * M), dtype=torch.float64)[:, ::2], "stride", id="column-step"),
    pytest.param(lambda N, M: torch.empty((N, 1), dtype=torch.float32).expand(N, M), "stride", id="broadcast"),
])
def test_score_matrix_refuses_bad_out(bad, match):
    """refused before anything touches a device (these run without one): the kernel would write an fp16 / bf16 out as
    fp32, write past a short one, and write a non-unit-stride view in the wrong layout"""
    p = _cpu_plda()
    e, t = np.zeros((5, 8)), np.zeros((7, 8))
    with pytest.raises(ValueError, match=match):
        p.score_matrix(e, t, 1, out=bad(5, 7))


@pytest.mark.gpu
def test_score_matrix_refuses_host_out():
    p = _cpu_plda()
    e, t = np.zeros((5, 8)), np.zeros((7, 8))
    with pytest.raises(ValueError, match="cuda:0"):
        p.score_matrix(e, t, 1, out=torch.empty((5, 7), dtype=torch.float64))


# ============================================================================================== 6. branch map
def test_branch_map_is_covered():
    seen = set()
    for rate, bins, _ in FB_CASES:
        seen |= fbank_branches(rate, bins, FB_T, fb_nsamples(rate), FB_B)
    seen |= fbank_branches(8000, 23, 41, 0, 1, ragged=True)
    seen |= {"cmn:T=1" if T == 1 else "cmn:T>8" if T > 8 else "cmn:T<=8" for T in CMN_T}
    for D in GEMM_D:
        for simt in _simt_modes(D):
            seen |= set().union(*(dgemm_branches(D, N, D, D, True, simt) for N in GEMM_SHAPES))
    for D, counts in SM_CASES:
        K = 2 * D if counts == "per-speaker" else D
        for simt in _simt_modes(K):
            for N in GEMM_SHAPES:
                for M in GEMM_SHAPES:
                    for ld in (M, M + 1):
                        for f64 in (False, True):
                            seen |= dgemm_branches(K, N, M, ld, f64, simt)
    for M in SEL_M:
        for top_n in sel_topns(M):
            for p in SEL_PATTERNS:
                seen |= select_branches(M, top_n, p, len(SEL_PATTERNS), 3)
    assert not BRANCHES - seen, f"no case reaches {sorted(BRANCHES - seen)}"
    # the dimensions of the GEMM cases: D = 8, 24, 200 (200: a Kaldi PLDA after LDA) take the FFMA kernel at K = D,
    # D = 16, 256 take DMMA, and every D takes DMMA at K = 2D
    assert [("dgemm:dmma" in dgemm_branches(D, 1, 1, 1, True)) for D in GEMM_D] == [False, False, False, True, True]
    assert all("dgemm:dmma" in dgemm_branches(2 * D, 1, 1, 1, True) for D in GEMM_D)
