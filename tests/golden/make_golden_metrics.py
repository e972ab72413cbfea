"""Generate tests/golden/metrics.npz by running the REAL reference metrics and calibration code.

Runs only in the build container (reads the reference checkout named by $WESPEAKER_REFERENCE).  Imported with the package
__init__ bypassed: `wespeaker/utils/score_metrics.py` (matplotlib / matplotlib.pyplot are stubs: only plot_det_curve uses
them), `wespeaker/bin/compute_metrics.py` (fire is a stub; stdout captured), `wespeaker/bin/score_calibration.py` and
`tools/generate_calibration_trial.py` (the `random` module seeded before the call).

Metric fixtures (every value from the reference's own compute_pmiss_pfa_rbst / compute_eer / compute_c_norm):
  * tie-free fp64 scores, n = 3 and 1000: balanced labels, a single target, a single non-target; n = 2 and 37 720:
    balanced.  Curves longer than 1200 are kept as the sha256 of their fp64 bytes.  Where the
    reference's compute_eer fails (no index with fnr - fpr < 0, e.g. every n = 2 list) only the curves are kept.
  * 5-decimal score files with ties: kept only when the reference as is and the reference with np.argsort patched to
    kind="stable" give the same curves, so the golden does not depend on this machine's unstable sort.
  * one file whose ties mix target and non-target trials: its golden is made WITH the stable patch (key "stable_only").
Calibration fixtures: a synthetic score-norm file (score_norm_main's 8 columns) of 6000 trials plus a wav duration table;
the factor files with and without duration, the loss of every epoch (LBFGS.step wrapped), the trained weights and the
inferred scores (the files as sha256, the scores as fp64).  Every stopping decision `best_loss - loss < 1e-4` is kept at
least 2e-5 away from the threshold (seeds are skipped until it is).  Run on the CPU, calibration.train_calibration_model
then reproduces every loss and weight; on a GPU the LBFGS trajectory drifts further than that, so the GPU test pins only
the first epochs and the final CLLR.
"""
import contextlib
import hashlib
import io
import os
import random
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.environ["WESPEAKER_REFERENCE"]   # a checkout of wenet-e2e/wespeaker
REF = os.path.join(ROOT, "wespeaker")


def _import_reference():
    for pkg, path in [("wespeaker", REF), ("wespeaker.bin", REF + "/bin"), ("wespeaker.utils", REF + "/utils")]:
        m = types.ModuleType(pkg)
        m.__path__ = [path]
        sys.modules[pkg] = m
    sys.modules["fire"] = types.ModuleType("fire")
    mpl = types.ModuleType("matplotlib")
    mpl.pyplot = types.ModuleType("matplotlib.pyplot")
    sys.modules["matplotlib"] = mpl
    sys.modules["matplotlib.pyplot"] = mpl.pyplot
    import wespeaker.utils.score_metrics as sm
    import wespeaker.bin.compute_metrics as cm
    import wespeaker.bin.score_calibration as sc
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import generate_calibration_trial as gct
    return sm, cm, sc, gct


@contextlib.contextmanager
def stable_argsort():
    """np.argsort and np.sort (compute_eer's threshold: the sign of a zero score at x1) with kind="stable"."""
    orig_argsort, orig_sort = np.argsort, np.sort
    np.argsort = lambda a, *args, **kw: orig_argsort(a, kind="stable")
    np.sort = lambda a, *args, **kw: orig_sort(a, kind="stable")
    try:
        yield
    finally:
        np.argsort, np.sort = orig_argsort, orig_sort


def same(a, b):
    return a.keys() == b.keys() and all(np.array_equal(a[k], b[k]) and np.signbit(a[k]).tolist() == np.signbit(b[k]).tolist()
                                        for k in a)


def run_metrics(sm, scores, labels, points):
    fnr, fpr = sm.compute_pmiss_pfa_rbst(scores, labels)
    r = {"fnr": fnr, "fpr": fpr}
    try:
        eer, thr = sm.compute_eer(fnr, fpr, scores)
    except IndexError:
        return r
    r["eer"], r["thr"] = np.float64(eer), np.float64(thr)
    r["min_dcf"] = np.array([sm.compute_c_norm(fnr, fpr, p, cmiss, cfa) for p, cmiss, cfa in points])
    r["c_det"] = np.array([sm.compute_c_dcf(fnr, fpr, p, cmiss, cfa) for p, cmiss, cfa in points])
    return r


POINTS = ((0.01, 1, 1), (0.001, 1, 1), (0.05, 2, 0.5))


def score_file_text(scores, labels, rng):
    return "".join(f"e{rng.integers(0, 500):03d} t{rng.integers(0, 900):03d} {s:.5f} {'target' if l else 'nontarget'}\n"
                   for s, l in zip(scores, labels))


def main():
    sm, cm, sc, gct = _import_reference()
    out = {"points": np.array(POINTS, dtype=np.float64)}
    rng = np.random.default_rng(11)
    # ---- tie-free fp64 lists
    cases = []
    for n in (2, 3, 1000, 37720):
        for kind in ("balanced", "one_target", "one_nontarget"):
            if n in (2, 37720) and kind != "balanced":
                continue
            lab = np.zeros(n, dtype=bool)
            if kind == "balanced":
                lab[rng.permutation(n)[: n // 2]] = True
            elif kind == "one_target":
                lab[rng.integers(0, n)] = True
            else:
                lab[:] = True
                lab[rng.integers(0, n)] = False
            s = rng.standard_normal(n) + 1.5 * lab
            assert np.unique(s).size == n
            cases.append((f"free_{n}_{kind}", s, lab))
    # ---- 5-decimal files with ties; the first two agree under both sorts, the third mixes labels in its ties
    for name, n, scale in (("ties_a", 3000, 0.05), ("ties_b", 20000, 0.3)):
        for _ in range(100):
            lab = rng.random(n) < 0.1
            # ties only inside a class (the last decimal tells the classes apart): any tie order gives the same curves
            s = np.round(np.round(scale * (rng.standard_normal(n) + 2.0 * lab), 4) + 1e-5 * lab, 5)
            text = score_file_text(s, lab, rng)
            s = np.array([float(ln.split()[2]) for ln in text.splitlines()])
            a = run_metrics(sm, s, lab, POINTS)
            with stable_argsort():
                b = run_metrics(sm, s, lab, POINTS)
            if same(a, b) and "eer" in a and np.unique(s).size < n:
                break
        else:
            raise RuntimeError(name + ": no fixture where both sorts agree")
        cases.append((name, s, lab))
        out[name + "_text"] = np.array(text.encode())
    n = 4000
    lab = rng.random(n) < 0.3
    s = np.round(0.01 * rng.integers(-40, 40, n) + 0.0 * lab, 5)
    s[:50] = -0.0
    s[50:100] = 0.0
    text = score_file_text(s, lab, rng)
    out["stable_only_text"] = np.array(text.encode())
    cases.append(("stable_only", np.array([float(ln.split()[2]) for ln in text.splitlines()]), lab))

    names = []
    for name, s, lab in cases:
        ctx = stable_argsort() if name == "stable_only" else contextlib.nullcontext()
        with ctx:
            r = run_metrics(sm, s, lab, POINTS)
        names.append(name)
        if name + "_text" not in out:     # the score files carry their scores and labels
            out[name + "_scores"], out[name + "_labels"] = s, lab
        big = s.size > 1200
        for k, v in r.items():
            if big and k in ("fnr", "fpr"):
                out[f"{name}_{k}_sha256"] = np.array(hashlib.sha256(np.ascontiguousarray(v).tobytes()).hexdigest())
            else:
                out[f"{name}_{k}"] = v
    out["cases"] = np.array(names)
    # ---- compute_metrics stdout
    with tempfile.TemporaryDirectory() as td:
        for name in ("ties_a", "ties_b", "stable_only"):
            path = os.path.join(td, name + ".score")
            open(path, "wb").write(out[name + "_text"].item())
            buf = io.StringIO()
            ctx = stable_argsort() if name == "stable_only" else contextlib.nullcontext()
            with ctx, contextlib.redirect_stdout(buf):
                cm.compute_metrics(path, 0.01, 1, 1)
                cm.compute_metrics(path, 0.05, 2, 1)
            out[name + "_stdout"] = np.array(buf.getvalue())

        # ---- calibration
        for seed in range(100):
            crng = np.random.default_rng(1000 + seed)
            nutt = 400
            utts = [f"spk{u % 40:02d}/utt{u:03d}.wav" for u in range(nutt)]
            durs = crng.uniform(1.0, 20.0, nutt)
            mag = crng.uniform(5.0, 30.0, nutt)
            cmean = crng.uniform(0.01, 0.3, nutt)
            rows = []
            for _ in range(6000):
                i, j = crng.integers(0, nutt, 2)
                tgt = crng.random() < 0.2
                sc_ = (0.6 if tgt else 0.0) + 0.25 * crng.standard_normal() + 0.01 * (mag[i] - 15) - 0.5 * cmean[j]
                rows.append(f"{utts[i]} {utts[j]} {sc_ * 5:.5f} {'target' if tgt else 'nontarget'} "
                            f"{mag[i]:.4f} {mag[j]:.4f} {cmean[i]:.4f} {cmean[j]:.4f}\n")
            norm_path, dur_path = os.path.join(td, "norm.score"), os.path.join(td, "utt2dur")
            open(norm_path, "w").write("".join(rows))
            open(dur_path, "w").write("".join(f"{u} {d:.3f}\n" for u, d in zip(utts, durs)))
            fac, fac_nodur = os.path.join(td, "factor"), os.path.join(td, "factor_nodur")
            sc.gather_calibration_factors(dur_path, 10.0, norm_path, fac)
            sc.gather_calibration_factors(dur_path, 10.0, norm_path, fac_nodur, drop_duration=True)
            losses = []
            orig = sc.optim.LBFGS

            class Rec(orig):
                def step(self, closure):
                    loss = super().step(closure)
                    losses.append(float(loss))
                    return loss

            sc.optim.LBFGS = Rec
            model_path = os.path.join(td, "model.pt")
            try:
                sc.train_calibration_model(fac, model_path)
            finally:
                sc.optim.LBFGS = orig
            best, margin = 1000000.0, np.inf
            for loss in losses:
                margin = min(margin, abs((best - loss) - 1e-4))
                if best - loss < 1e-4:
                    break
                best = min(best, loss)
            if margin >= 2e-5 and 2 < len(losses) < 50:
                break
        else:
            raise RuntimeError("no calibration fixture with a clear stopping margin")
        import torch
        sd = torch.load(model_path)
        cal = os.path.join(td, "cal.score")
        sc.infer_calibration(fac, model_path, cal)
        sha = lambda path: np.array(hashlib.sha256(open(path, "rb").read()).hexdigest())   # noqa: E731
        cal_lines = [ln.split() for ln in open(cal)]
        fac_lines = [ln.split() for ln in open(fac)]
        assert [c[:2] + c[3:] for c in cal_lines] == [f[:3] for f in fac_lines]
        out.update(cal_norm_text=np.array("".join(rows).encode()), cal_utt2dur_text=np.array(open(dur_path).read().encode()),
                   cal_factor_sha256=sha(fac), cal_factor_nodur_sha256=sha(fac_nodur), cal_score_sha256=sha(cal),
                   cal_losses=np.array(losses), cal_weight=sd["linear.weight"].numpy(), cal_bias=sd["linear.bias"].numpy(),
                   cal_scores=np.array([float(c[2]) for c in cal_lines]), cal_stop_margin=np.float64(margin))
        tgt = [[float(v) for v in ln.split()[3:]] for ln in open(fac) if ln.split()[2] == "target"]
        non = [[float(v) for v in ln.split()[3:]] for ln in open(fac) if ln.split()[2] != "target"]
        m = sc.LinearModel(len(tgt[0])).double()
        m.load_state_dict(sd)
        with torch.no_grad():
            out["cal_final_cllr"] = np.float64(sc.cllr(m(torch.tensor(tgt, dtype=torch.float64)),
                                                       m(torch.tensor(non, dtype=torch.float64))).item())
        # ---- calibration trial list
        trial = os.path.join(td, "trial")
        random.seed(7)
        gct.main(dur_path, trial, each_trial_num=300)
        out["cal_trial_seed"] = np.int64(7)
        out["cal_trial_text"] = np.array(open(trial).read().encode())
    np.savez_compressed(os.path.join(HERE, "metrics.npz"), **out)
    print({k: (v.shape, v.dtype) for k, v in out.items() if v.ndim > 0}, "stop margin", out["cal_stop_margin"],
          "epochs", len(out["cal_losses"]))


if __name__ == "__main__":
    main()
