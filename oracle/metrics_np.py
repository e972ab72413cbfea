"""numpy restatement of the verification metrics of `wespeaker/utils/score_metrics.py:58-116` (compute_pmiss_pfa_rbst,
compute_eer, compute_c_norm) and of `cllr` in `wespeaker/bin/score_calibration.py:82-92`.

One deviation, the project's tie policy: trials are ordered by `np.argsort(scores, kind="stable")`, i.e. ascending by
(score, trial line), where the reference's default argsort leaves equal scores in an order that depends on numpy's sort
algorithm and the CPU.  The arithmetic is otherwise the reference's, operation for operation, so with unit weights every
curve value, the EER, the threshold and minDCF are reproduced bit for bit.
"""
import numpy as np
import torch


def order(scores):
    return np.argsort(np.asarray(scores, dtype=np.float64), kind="stable")


def pmiss_pfa_rbst(scores, labels):
    """score_metrics.py:58-76 with unit weights, stable order."""
    labels = np.asarray(labels)[order(scores)]
    tgt = (labels == 1).astype("f8")
    imp = (labels == 0).astype("f8")
    fnr = np.cumsum(tgt) / np.sum(tgt)
    fpr = 1 - np.cumsum(imp) / np.sum(imp)
    return fnr, fpr


def eer(fnr, fpr, scores=None):
    """score_metrics.py:79-93; the threshold is the score at x1 in the stable order."""
    diff_pm_fa = fnr - fpr
    x1 = np.flatnonzero(diff_pm_fa >= 0)[0]
    x2 = np.flatnonzero(diff_pm_fa < 0)[-1]
    a = (fnr[x1] - fpr[x1]) / (fpr[x2] - fpr[x1] - (fnr[x2] - fnr[x1]))
    e = fnr[x1] + a * (fnr[x2] - fnr[x1])
    if scores is not None:
        s = np.asarray(scores, dtype=np.float64)
        return e, s[order(s)][x1]
    return e


def c_det(fnr, fpr, p_target, c_miss=1, c_fa=1):
    """score_metrics.py:108-116 (compute_c_dcf)."""
    return min(c_miss * fnr * p_target + c_fa * fpr * (1 - p_target))


def c_norm(fnr, fpr, p_target, c_miss=1, c_fa=1):
    """score_metrics.py:96-105."""
    return c_det(fnr, fpr, p_target, c_miss, c_fa) / min(c_miss * p_target, c_fa * (1 - p_target))


def cllr(target_llrs, nontarget_llrs):
    """score_calibration.py:82-92 on torch tensors."""
    def negative_log_sigmoid(lodds):
        return torch.log1p(torch.exp(-lodds))
    return 0.5 * (torch.mean(negative_log_sigmoid(target_llrs)) + torch.mean(negative_log_sigmoid(-nontarget_llrs))) / np.log(2)
