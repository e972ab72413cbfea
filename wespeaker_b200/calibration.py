"""Score calibration — mirror of `wespeaker/bin/score_calibration.py` (gather_calibration_factors, LinearModel, cllr,
train_calibration_model, infer_calibration) and `tools/generate_calibration_trial.py`, which the recipes'
`local/score_calibration.sh` runs ahead of `compute_metrics`.

The factor file is a text transformation of `score.score_norm_main`'s output (its four calibration columns), byte for byte
the reference's.  The model is the reference's linear logistic calibration: LBFGS (lr 0.01) on the CLLR for at most 50
epochs, stopping when an epoch improves the best loss by less than 1e-4, in torch fp64 on the device (a one-off job of a
few thousand rows, the precedent of `plda_train`).  Saved models hold CPU tensors under the reference's keys
(`linear.weight`, `linear.bias`), so either implementation loads the other's.
"""
from __future__ import annotations

import logging
import os
import random

import numpy as np
import torch
import torch.nn as nn
import torch.optim as optim

from . import lib as _lib
from .score import read_table


def _device(device=None) -> torch.device:
    if device is not None:
        return torch.device(device)
    if not torch.cuda.is_available():
        raise _lib.B200Error("wespeaker_b200.calibration needs a CUDA device (no CPU fallback)")
    return torch.device("cuda", torch.cuda.current_device())


def gather_calibration_factors(wav_dur_scp, max_dur, score_norm_file, calibration_factor_file, drop_duration=False):
    """`score_calibration.py:30-66`: `enroll test label score [dur x4] mag x4 cohort_mean x4`, each group as
    min, max, max - min, max / min."""
    if not drop_duration:
        wav_idx, dur_list = zip(*read_table(wav_dur_scp))
        wavidx2dur = {idx: min(float(dur), max_dur) for idx, dur in zip(wav_idx, dur_list)}

    def reorder_values(value_1, value_2):
        max_value = max(value_1, value_2)
        min_value = min(value_1, value_2)
        return "{:.4f} {:.4f} {:.4f} {:.4f}".format(min_value, max_value, max_value - min_value, max_value / min_value)

    assert os.path.exists(score_norm_file), "score norm file ({}) does not exist !!!".format(score_norm_file)
    with open(score_norm_file, "r", encoding="utf-8") as fin:
        with open(calibration_factor_file, "w", encoding="utf-8") as fout:
            for line in fin.readlines():
                line = line.strip().split()
                idx1, idx2 = line[0], line[1]
                dur_str = "" if drop_duration else reorder_values(wavidx2dur[idx1], wavidx2dur[idx2])
                mag_str = reorder_values(float(line[4]), float(line[5]))
                cohort_mean_str = reorder_values(float(line[6]), float(line[7]))
                fout.write("{} {} {} {} {} {} {}\n".format(line[0], line[1], line[3], line[2], dur_str, mag_str,
                                                          cohort_mean_str))


class LinearModel(nn.Module):
    """`score_calibration.py:69-79`."""

    def __init__(self, input_dim):
        super().__init__()
        self.linear = nn.Linear(input_dim, 1)
        nn.init.constant_(self.linear.weight, 1.0 / input_dim)
        nn.init.constant_(self.linear.bias, 0)

    def forward(self, x):
        return self.linear(x)


def cllr(target_llrs, nontarget_llrs):
    """`score_calibration.py:82-92`: the CLLR of target / non-target log-likelihood ratios, in bits."""
    def negative_log_sigmoid(lodds):
        return torch.log1p(torch.exp(-lodds))
    return 0.5 * (torch.mean(negative_log_sigmoid(target_llrs)) + torch.mean(negative_log_sigmoid(-nontarget_llrs))) / np.log(2)


def _read_factors(calibration_factor_file):
    with open(calibration_factor_file, "r", encoding="utf-8") as fin:
        return [line.strip().split() for line in fin.readlines()]


def train_calibration_model(calibration_factor_file, save_model_path, device=None):
    """`score_calibration.py:95-139`; returns the loss of every epoch that ran (the reference returns nothing)."""
    dev = _device(device)
    tgt, non = [], []
    for line in _read_factors(calibration_factor_file):
        (tgt if line[2] in ("tgt", "target") else non).append([float(v) for v in line[3:]])
    target_llrs = torch.tensor(tgt, dtype=torch.float64, device=dev)
    nontarget_llrs = torch.tensor(non, dtype=torch.float64, device=dev)
    model = LinearModel(target_llrs.shape[-1]).double().to(dev)
    optimizer = optim.LBFGS(model.parameters(), lr=0.01)
    losses = []
    best_loss = 1000000.0
    for _ in range(50):
        def closure():
            optimizer.zero_grad()
            loss = cllr(model(target_llrs), model(nontarget_llrs))
            loss.backward()
            return loss

        loss = float(optimizer.step(closure))
        losses.append(loss)
        if best_loss - loss < 1e-4:
            break
        if loss < best_loss:
            best_loss = loss
    torch.save({k: v.detach().cpu() for k, v in model.state_dict().items()}, save_model_path)
    return losses


def infer_calibration(calibration_factor_file, save_model_path, calibration_score_file, device=None):
    """`score_calibration.py:142-164`: `enroll test calibrated_score label`, the score as a Python float repr."""
    dev = _device(device)
    lines = _read_factors(calibration_factor_file)
    llrs = torch.tensor([[float(v) for v in line[3:]] for line in lines], dtype=torch.float64, device=dev)
    model = LinearModel(llrs.shape[-1])
    model.load_state_dict(torch.load(save_model_path, map_location="cpu"))
    model.eval()
    model = model.double().to(dev)
    with torch.no_grad():
        outputs = model(llrs).cpu()
    with open(calibration_score_file, "w", encoding="utf-8") as fout:
        for line, out in zip(lines, outputs):
            fout.write("{} {} {} {}\n".format(line[0], line[1], out.item(), line[2]))


def generate_calibration_trial(utt2dur, trial_path, each_trial_num=10000, seed=None):
    """`tools/generate_calibration_trial.py:22-83`: the same draws in the same order, so a seed gives the reference's file
    (seed=None draws from the `random` module's own state, as the reference does)."""
    rng = random if seed is None else random.Random(seed)
    logging.info("Generate calibration trial ...")
    short_spk2utt, long_spk2utt = {}, {}
    with open(utt2dur, "r") as f:
        for line in f.readlines():
            utt, dur = line.strip().split()
            dur = float(dur)
            spk = utt.split("/")[0]
            if 2 < dur < 6:
                short_spk2utt.setdefault(spk, []).append(utt)
            if dur > 6:
                long_spk2utt.setdefault(spk, []).append(utt)
    short_spks = list(short_spk2utt.keys())
    for spk in list(long_spk2utt.keys()):
        if spk not in short_spks:
            long_spk2utt.pop(spk, None)
    long_spks = list(long_spk2utt.keys())
    for spk in short_spks:
        if spk not in long_spks:
            short_spk2utt.pop(spk, None)
    short_spks = list(short_spk2utt.keys())
    with open(trial_path, "w") as f:
        for _ in range(each_trial_num // 2):
            enroll_spk = rng.choice(short_spks)
            spk_index = short_spks.index(enroll_spk)
            nontarget_spk = rng.choice(short_spks[:spk_index] + short_spks[spk_index + 1:])
            # short2short
            enroll_utt, test_utt = rng.choices(short_spk2utt[enroll_spk], k=2)
            f.write("{} {} {}\n".format(enroll_utt, test_utt, "target"))
            test_utt = rng.choice(short_spk2utt[nontarget_spk])
            f.write("{} {} {}\n".format(enroll_utt, test_utt, "nontarget"))
            # short2long
            enroll_utt = rng.choice(short_spk2utt[enroll_spk])
            test_utt = rng.choice(long_spk2utt[enroll_spk])
            f.write("{} {} {}\n".format(enroll_utt, test_utt, "target"))
            test_utt = rng.choice(long_spk2utt[nontarget_spk])
            f.write("{} {} {}\n".format(enroll_utt, test_utt, "nontarget"))
            # long2long
            enroll_utt, test_utt = rng.choices(long_spk2utt[enroll_spk], k=2)
            f.write("{} {} {}\n".format(enroll_utt, test_utt, "target"))
            test_utt = rng.choice(long_spk2utt[nontarget_spk])
            f.write("{} {} {}\n".format(enroll_utt, test_utt, "nontarget"))
