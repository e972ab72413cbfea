"""Verification metrics on the GPU — mirror of `wespeaker/utils/score_metrics.py` (compute_pmiss_pfa_rbst, compute_eer,
compute_c_norm, compute_c_dcf, plot_det_curve), `wespeaker/bin/compute_metrics.py` and `wespeaker/bin/compute_det.py`
(SURVEY.md §2 row 18).

`evaluate` is the device entry: one call of `ws_metrics_eval` (csrc/ws_metrics.cu) sorts the trials, builds the miss /
false-alarm curves, finds the EER crossing and the minimum detection cost of every operating point, and one copy brings
back the handful of numbers the EER interpolation and the c_def division need; those two are scalar float arithmetic here,
as in the reference.  Scores that are already on the device never leave it.

Tie policy (the one deviation from the reference): trials are ordered by (score, trial line) ascending — what the reference
computes with `np.argsort(kind="stable")`; its default argsort leaves equal scores in an order that depends on numpy's sort
and the CPU.  -0.0 equals +0.0, +-inf are ordered, a NaN score, a label other than 0 / 1 and an empty class are refused.

`compute_eer`, `compute_c_norm` and `compute_c_dcf` keep the reference's signatures over curves the caller already holds
(arrays in, scalars out: a search and one expression over the given values); the sort and the curves, the part that grows
with the trial count, come from the device through `compute_pmiss_pfa_rbst` / `evaluate`.  There is no CPU fallback.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import NamedTuple, Optional

import numpy as np
import torch

from . import lib as _lib

MAX_POINTS = 16
MAX_N = (1 << 31) - 1
_NO_X2 = 8
_CAUSES = ((1, "a NaN score"), (2, "a label other than 0 or 1"), (4, "no target or no non-target trial"),
           (8, "fnr - fpr is never negative, so the EER has no lower crossing point (x2)"))


class Metrics(NamedTuple):
    eer: float
    threshold: float             # the score at x1 (compute_eer's second result)
    min_dcf: tuple               # compute_c_norm per operating point
    c_det: tuple                 # compute_c_dcf per operating point
    x1: int
    x2: int
    fnr: Optional[torch.Tensor]  # fp64 [n] on the device when curve=True
    fpr: Optional[torch.Tensor]
    order: Optional[torch.Tensor]   # int32 [n]: trial indices in sorted order, when curve=True


def _device(device=None) -> torch.device:
    if not torch.cuda.is_available():
        raise _lib.B200Error("wespeaker_b200.metrics needs a CUDA device (no CPU fallback)")
    return torch.device("cuda", torch.cuda.current_device() if device is None else device)


def _scores_tensor(scores, dev) -> torch.Tensor:
    t = scores if isinstance(scores, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(scores))
    if t.dtype not in (torch.float64, torch.float32):
        raise _lib.B200Error(f"metrics: scores must be fp64 or fp32, got {t.dtype}")
    return t.reshape(-1).to(dev).to(torch.float64).contiguous()      # fp32 -> fp64 is exact


def _labels_tensor(labels, dev) -> torch.Tensor:
    t = labels if isinstance(labels, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(labels))
    t = t.reshape(-1).to(dev)
    if t.dtype != torch.bool:     # anything but 0 / 1 becomes 2, which the device refuses
        t = torch.where(t == 1, 1, torch.where(t == 0, 0, 2))
    return t.to(torch.uint8).contiguous()


def _points(operating_points):
    pts = [tuple(p) for p in operating_points]
    if not 1 <= len(pts) <= MAX_POINTS or any(len(p) != 3 for p in pts):
        raise _lib.B200Error(f"metrics: operating_points must be 1..{MAX_POINTS} (p_target, c_miss, c_fa) triples")
    return pts


def _launch(s: torch.Tensor, lab: torch.Tensor, pts, out=None, order=None, fnr=None, fpr=None, stage_events=None):
    """One ws_metrics_eval call on the current stream; returns the fp64 [8 + P] result buffer (still on the device)."""
    L = _lib.load()
    n = s.numel()
    if n == 0:
        raise _lib.B200Error("metrics: no trials")
    if lab.numel() != n:
        raise _lib.B200Error(f"metrics: {n} scores but {lab.numel()} labels")
    P = len(pts)
    arr = C.c_double * P
    p, cm, cf = (arr(*[float(q[k]) for q in pts]) for k in range(3))
    wb = L.ws_metrics_work_bytes(n)
    if wb == 0:
        raise _lib.B200Error(f"metrics: n = {n} trials is outside [1, 2^31 - 1]")
    work = torch.empty((wb,), dtype=torch.uint8, device=s.device)
    if out is None:
        out = torch.empty((8 + P,), dtype=torch.float64, device=s.device)
    ev = None
    if stage_events is not None:
        ev = (C.c_void_p * len(stage_events))(*[e.cuda_event for e in stage_events])
    ptr = lambda t: t.data_ptr() if t is not None else None   # noqa: E731
    _lib.check(L.ws_metrics_eval(s.data_ptr(), lab.data_ptr(), n, p, cm, cf, P, work.data_ptr(), wb, out.data_ptr(),
                                 ptr(order), ptr(fnr), ptr(fpr), _lib.cur_stream_ptr(s.device), ev), "ws_metrics_eval")
    return out


def status_causes(status: int) -> str:
    return "; ".join(msg for bit, msg in _CAUSES if status & bit)


def evaluate(scores, labels, operating_points=((0.01, 1, 1),), curve=False, device=None) -> Metrics:
    """EER, its threshold, and c_det / minDCF (c_norm) per (p_target, c_miss, c_fa) operating point of a trial list;
    with curve=True also the fnr / fpr curves and the sorted order, left on the device.  `scores`: fp64 or fp32 tensor or
    array; `labels`: 1 / True for a target trial, 0 / False for a non-target one."""
    pts = _points(operating_points)
    dev = scores.device if isinstance(scores, torch.Tensor) and scores.is_cuda else _device(device)
    with torch.cuda.device(dev):
        s = _scores_tensor(scores, dev)
        lab = _labels_tensor(labels, dev)
        n = s.numel()
        fnr = fpr = order = None
        if curve:
            fnr = torch.empty((n,), dtype=torch.float64, device=dev)
            fpr = torch.empty((n,), dtype=torch.float64, device=dev)
            order = torch.empty((n,), dtype=torch.int32, device=dev)
        r = _launch(s, lab, pts, order=order, fnr=fnr, fpr=fpr).cpu().numpy()
    status = int(r[7])
    if status:
        raise _lib.B200Error(f"metrics: refused: {status_causes(status)}")
    fnr1, fpr1, fnr2, fpr2 = (np.float64(v) for v in r[:4])
    a = (fnr1 - fpr1) / (fpr2 - fpr1 - (fnr2 - fnr1))                  # score_metrics.py:87-91
    eer = fnr1 + a * (fnr2 - fnr1)
    c_det = tuple(float(v) for v in r[8:8 + len(pts)])
    min_dcf = tuple(float(np.float64(c) / min(cm * p, cf * (1 - p))) for c, (p, cm, cf) in zip(c_det, pts))
    return Metrics(float(eer), float(r[4]), min_dcf, c_det, int(r[5]), int(r[6]), fnr, fpr, order)


# ------------------------------------------------------------------------------------------------- score_metrics.py
def compute_pmiss_pfa_rbst(scores, labels, weights=None):
    """`score_metrics.py:58-76`: (fnr, fpr) as fp64 numpy arrays, computed on the device."""
    if weights is not None:
        raise _lib.B200Error("compute_pmiss_pfa_rbst: weighted curves are not supported (weights must be None)")
    dev = scores.device if isinstance(scores, torch.Tensor) and scores.is_cuda else _device()
    with torch.cuda.device(dev):
        s = _scores_tensor(scores, dev)
        lab = _labels_tensor(labels, dev)
        fnr = torch.empty((s.numel(),), dtype=torch.float64, device=dev)
        fpr = torch.empty_like(fnr)
        status = int(_launch(s, lab, [(0.01, 1, 1)], fnr=fnr, fpr=fpr)[7].item())
    if status & ~_NO_X2:      # the curves are written without an EER crossing; only compute_eer needs one
        raise _lib.B200Error(f"compute_pmiss_pfa_rbst: refused: {status_causes(status)}")
    return fnr.cpu().numpy(), fpr.cpu().numpy()


def compute_eer(fnr, fpr, scores=None):
    """`score_metrics.py:79-93` over given curves; the threshold is the score at x1 in the stable (score, line) order."""
    fnr, fpr = np.asarray(fnr), np.asarray(fpr)
    diff_pm_fa = fnr - fpr
    x1 = np.flatnonzero(diff_pm_fa >= 0)[0]
    x2 = np.flatnonzero(diff_pm_fa < 0)[-1]
    a = (fnr[x1] - fpr[x1]) / (fpr[x2] - fpr[x1] - (fnr[x2] - fnr[x1]))
    if scores is not None:
        s = np.asarray(scores)
        return fnr[x1] + a * (fnr[x2] - fnr[x1]), s[np.argsort(s, kind="stable")][x1]
    return fnr[x1] + a * (fnr[x2] - fnr[x1])


def compute_c_dcf(fnr, fpr, p_target, c_miss=1, c_fa=1):
    """`score_metrics.py:108-116` over given curves."""
    return min(c_miss * np.asarray(fnr) * p_target + c_fa * np.asarray(fpr) * (1 - p_target))


def compute_c_norm(fnr, fpr, p_target, c_miss=1, c_fa=1):
    """`score_metrics.py:96-105` over given curves."""
    return compute_c_dcf(fnr, fpr, p_target, c_miss, c_fa) / min(c_miss * p_target, c_fa * (1 - p_target))


def plot_det_curve(fnr, fpr, save_path=None):
    """`score_metrics.py:119-160`; needs matplotlib, which is imported here and only here."""
    try:
        import matplotlib
        if save_path is not None:
            matplotlib.use("Agg")
        import matplotlib.pyplot as plt
    except ImportError as e:
        raise ImportError("plot_det_curve needs matplotlib, which is not installed") from e
    from scipy.stats import norm
    p_miss = norm.ppf(fnr)
    p_fa = norm.ppf(fpr)
    xytick = [0.0001, 0.0002, 0.0005, 0.001, 0.002, 0.005, 0.01, 0.02, 0.05, 0.1, 0.2, 0.4]
    xytick_labels = map(str, [x * 100 for x in xytick])
    plt.plot(p_fa, p_miss, "r")
    plt.xticks(norm.ppf(xytick), xytick_labels)
    plt.yticks(norm.ppf(xytick), xytick_labels)
    plt.xlim(norm.ppf([0.00051, 0.5]))
    plt.ylim(norm.ppf([0.00051, 0.5]))
    plt.xlabel("false-alarm rate [%]", fontsize=12)
    plt.ylabel("false-reject rate [%]", fontsize=12)
    eer = compute_eer(fnr, fpr)
    plt.plot(norm.ppf(eer), norm.ppf(eer), "o")
    plt.annotate("EER = %.2f%%" % (eer * 100), xy=(norm.ppf(eer), norm.ppf(eer)), xycoords="data",
                 xytext=(norm.ppf(eer + 0.05), norm.ppf(eer + 0.05)), textcoords="data",
                 arrowprops=dict(arrowstyle="-|>", connectionstyle="arc3, rad=+0.2", fc="w"), size=12, va="center",
                 ha="center", bbox=dict(boxstyle="round4", fc="w"))
    plt.grid()
    if save_path is not None:
        plt.savefig(save_path)
        plt.clf()
    else:
        plt.show()


# ------------------------------------------------------------------------------------------------- compute_metrics.py / compute_det.py
def read_scores(scores_file):
    """Column 2 is the score, column 3 == "target" the label (compute_metrics.py:26-37)."""
    scores, labels = [], []
    with open(scores_file) as readlines:
        for line in readlines:
            tokens = line.strip().split()
            scores.append(float(tokens[2]))
            labels.append(tokens[3] == "target")
    return np.array(scores, dtype=np.float64), np.array(labels, dtype=bool)


def compute_metrics(scores_file, p_target=0.01, c_miss=1, c_fa=1):
    """`compute_metrics.py:25-50`: prints the file name, the EER and minDCF in the reference's format."""
    scores, labels = read_scores(scores_file)
    m = evaluate(scores, labels, ((p_target, c_miss, c_fa),))
    print("---- {} -----".format(os.path.basename(scores_file)))
    print("EER = {0:.3f}".format(100 * m.eer))
    print("minDCF (p_target:{} c_miss:{} c_fa:{}) = {:.3f}".format(p_target, c_miss, c_fa, m.min_dcf[0]))


def main(p_target=0.01, c_miss=1, c_fa=1, *scores_files):
    """`compute_metrics.py:53-55`."""
    for scores_file in scores_files:
        compute_metrics(scores_file, p_target, c_miss, c_fa)


def compute_det(scores_file, det_file):
    """`compute_det.py:22-38`: the DET curve of a score file, curves from the device."""
    scores, labels = read_scores(scores_file)
    fnr, fpr = compute_pmiss_pfa_rbst(scores, labels)
    plot_det_curve(fnr, fpr, det_file)
    print("DET curve saved in {}".format(det_file))


def det_main(*scores_files):
    """`compute_det.py:41-44` (its `main`)."""
    for scores_file in scores_files:
        compute_det(scores_file, scores_file + ".det.png")
