"""Verification metrics (EER / minDCF / DET curves) and score calibration (SURVEY.md §2 row 18).

CPU part: the oracle (oracle/metrics_np.py) against goldens produced by the reference's own score_metrics.py,
compute_metrics.py, score_calibration.py and generate_calibration_trial.py (tests/golden/make_golden_metrics.py); the
calibration text files byte for byte; argument refusals of the C ABI.  GPU part: ws_metrics_eval (csrc/ws_metrics.cu)
through wespeaker_b200.metrics against torch's stable sort, the oracle and the goldens, bit for bit; calibration training and
inference against the reference's model and scores."""
import contextlib
import ctypes as C
import hashlib
import io
import os

import numpy as np
import pytest
import torch

from oracle import metrics_np
from wespeaker_b200 import calibration, lib, metrics

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "metrics.npz"))
CASES = [str(c) for c in G["cases"]]
POINTS = [tuple(p) for p in G["points"]]
gpu = pytest.mark.gpu


def _text(key):
    return G[key].item().decode()


def _case(name):
    if name + "_text" in G:
        rows = [ln.split() for ln in _text(name + "_text").splitlines()]
        return np.array([float(r[2]) for r in rows]), np.array([r[3] == "target" for r in rows])
    return G[name + "_scores"], G[name + "_labels"]


def _same_bits(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return a.shape == b.shape and a.tobytes() == b.tobytes()


def _same_curve(name, key, got):
    if f"{name}_{key}_sha256" in G:
        return hashlib.sha256(np.ascontiguousarray(got, dtype=np.float64).tobytes()).hexdigest() == str(G[f"{name}_{key}_sha256"])
    return _same_bits(got, G[f"{name}_{key}"])


# ------------------------------------------------------------------------------------------------- CPU: oracle pinned
@pytest.mark.parametrize("name", CASES)
def test_oracle_reproduces_reference_bit_for_bit(name):
    s, lab = _case(name)
    fnr, fpr = metrics_np.pmiss_pfa_rbst(s, lab)
    assert _same_curve(name, "fnr", fnr) and _same_curve(name, "fpr", fpr)
    if name + "_eer" not in G:
        with pytest.raises(IndexError):
            metrics_np.eer(fnr, fpr, s)
        return
    eer, thr = metrics_np.eer(fnr, fpr, s)
    assert _same_bits(eer, G[name + "_eer"]) and _same_bits(thr, G[name + "_thr"])
    assert _same_bits([metrics_np.c_norm(fnr, fpr, *p) for p in POINTS], G[name + "_min_dcf"])
    assert _same_bits([metrics_np.c_det(fnr, fpr, *p) for p in POINTS], G[name + "_c_det"])


def test_calibration_text_files_are_byte_identical(tmp_path):
    norm, dur = tmp_path / "norm.score", tmp_path / "utt2dur"
    norm.write_bytes(G["cal_norm_text"].item())
    dur.write_bytes(G["cal_utt2dur_text"].item())
    for drop, key in ((False, "cal_factor_sha256"), (True, "cal_factor_nodur_sha256")):
        fac = tmp_path / f"factor_{drop}"
        calibration.gather_calibration_factors(str(dur), 10.0, str(norm), str(fac), drop_duration=drop)
        assert hashlib.sha256(fac.read_bytes()).hexdigest() == str(G[key])
    trial = tmp_path / "trial"
    calibration.generate_calibration_trial(str(dur), str(trial), each_trial_num=300, seed=int(G["cal_trial_seed"]))
    assert trial.read_bytes() == G["cal_trial_text"].item()


def test_oracle_cllr_of_reference_model():
    rows = [ln.split() for ln in _factor_lines()]
    x = torch.tensor([[float(v) for v in r[3:]] for r in rows], dtype=torch.float64)
    is_t = torch.tensor([r[2] == "target" for r in rows])
    w, b = torch.from_numpy(G["cal_weight"]), torch.from_numpy(G["cal_bias"])
    llr = x @ w.T + b
    assert abs(float(metrics_np.cllr(llr[is_t], llr[~is_t])) - float(G["cal_final_cllr"])) <= 1e-12


def _factor_lines(drop=False):
    import tempfile
    with tempfile.TemporaryDirectory() as td:
        norm, dur, fac = (os.path.join(td, f) for f in ("norm", "dur", "fac"))
        open(norm, "wb").write(G["cal_norm_text"].item())
        open(dur, "wb").write(G["cal_utt2dur_text"].item())
        calibration.gather_calibration_factors(dur, 10.0, norm, fac, drop_duration=drop)
        return open(fac).read().splitlines()


def _abi_args(n=10, p=(0.01,), cm=(1.0,), cf=(1.0,), n_points=None, work_bytes=None, null=None):
    L = lib.load()
    P = len(p)
    arr = C.c_double * max(P, 1)
    fake = C.c_void_p(256)                       # never dereferenced: every case is refused before a launch
    args = [fake, fake, n, arr(*p), arr(*cm), arr(*cf), P if n_points is None else n_points, fake,
            (L.ws_metrics_work_bytes(n) or 1 << 40) if work_bytes is None else work_bytes, fake, None, None, None, None, None]
    if null is not None:
        args[null] = None
    return args


@pytest.mark.parametrize("case,msg", [
    (dict(n=0), "n must be"), (dict(n=-5), "n must be"), (dict(n=1 << 31), "n must be"),
    (dict(n_points=0), "n_points"), (dict(n_points=17), "n_points"),
    (dict(p=(0.0,)), "p_target"), (dict(p=(1.0,)), "p_target"), (dict(p=(float("nan"),)), "p_target"),
    (dict(cm=(-1.0,)), "costs"), (dict(cf=(float("inf"),)), "costs"), (dict(cf=(float("nan"),)), "costs"),
    (dict(work_bytes=1000), "workspace"), (dict(null=0), "null"), (dict(null=1), "null"), (dict(null=7), "null"),
    (dict(null=9), "null")])
def test_abi_refuses_bad_arguments_before_launch(case, msg):
    L = lib.load()
    assert L.ws_metrics_eval(*_abi_args(**case)) == 1
    assert msg in L.ws_last_error().decode()


def test_abi_work_bytes_bounds():
    L = lib.load()
    assert L.ws_metrics_work_bytes(0) == 0 and L.ws_metrics_work_bytes(1 << 31) == 0
    assert L.ws_metrics_work_bytes(1) > 0 and L.ws_metrics_work_bytes((1 << 31) - 1) > 24 * ((1 << 31) - 1)


def test_python_refusals_without_device():
    with pytest.raises(lib.B200Error, match="weights"):
        metrics.compute_pmiss_pfa_rbst(np.zeros(4), np.array([0, 1, 0, 1]), weights=np.ones(4))
    for bad in ((), [(0.01, 1, 1)] * 17, [(0.01, 1)]):
        with pytest.raises(lib.B200Error, match="operating_points"):
            metrics.evaluate(np.zeros(4), np.array([0, 1, 0, 1]), bad)


def test_metrics_and_calibration_need_gpu_and_fail_loudly(tmp_path):
    if torch.cuda.is_available():
        pytest.skip("CPU-only check")
    s, lab = _case("free_1000_balanced")
    with pytest.raises(lib.B200Error):
        metrics.evaluate(s, lab)
    with pytest.raises(lib.B200Error):
        metrics.compute_pmiss_pfa_rbst(s, lab)
    f = tmp_path / "x.score"
    f.write_bytes(G["ties_a_text"].item())
    with pytest.raises(lib.B200Error):
        metrics.compute_metrics(str(f))
    fac = tmp_path / "fac"
    fac.write_text("\n".join(_factor_lines()) + "\n")
    with pytest.raises(lib.B200Error):
        calibration.train_calibration_model(str(fac), str(tmp_path / "m.pt"))
    with pytest.raises(lib.B200Error):
        calibration.infer_calibration(str(fac), str(tmp_path / "m.pt"), str(tmp_path / "o"))


# ------------------------------------------------------------------------------------------------- GPU
TILE = 4096
SIZES = [2, 3, TILE - 1, TILE, TILE + 1, (1 << 20) + 3, 30_000_000]
KINDS = ["normal", "decimals5", "all_equal", "two_values", "signed_zeros", "infinities", "subnormals", "sorted", "reversed"]


def _make(kind, n, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(n, dtype=torch.float64, device="cuda", generator=g)
    if kind == "decimals5":
        x = torch.round(x * 0.3, decimals=5)
    elif kind == "all_equal":
        x = torch.full_like(x, 0.25)
    elif kind == "two_values":
        x = torch.where(x > 0, 0.5, -1.5).to(torch.float64)
    elif kind == "signed_zeros":
        x = torch.where(x > 0.5, 0.0, torch.where(x < -0.5, -0.0, x)).to(torch.float64)
        if n > 1000:
            assert bool(torch.signbit(x[x == 0]).any()) and not bool(torch.signbit(x[x == 0]).all())
    elif kind == "infinities":
        x = torch.where(x > 1.5, float("inf"), torch.where(x < -1.5, float("-inf"), x)).to(torch.float64)
    elif kind == "subnormals":
        x = x * 1e-310
    elif kind == "sorted":
        x = torch.sort(x).values
    elif kind == "reversed":
        x = torch.sort(x, descending=True).values
    lab = (torch.rand(n, device="cuda", generator=g) < 0.3).to(torch.uint8)
    lab[0], lab[-1] = 1, 0                     # both classes present
    return x.contiguous(), lab


def _raw(s, lab, pts=((0.01, 1, 1),), curve=True, fill=None):
    n = s.numel()
    f = (lambda shape, dt: torch.full(shape, fill, dtype=dt, device=s.device)) if fill is not None else \
        (lambda shape, dt: torch.empty(shape, dtype=dt, device=s.device))
    out = f((8 + len(pts),), torch.float64)
    order = f((max(n, 1),), torch.int32) if curve else None
    fnr = f((max(n, 1),), torch.float64) if curve else None
    fpr = f((max(n, 1),), torch.float64) if curve else None
    metrics._launch(s, lab, pts, out=out, order=order, fnr=fnr, fpr=fpr)
    torch.cuda.synchronize()
    return out, order, fnr, fpr


@gpu
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("n", SIZES)
def test_gpu_order_equals_torch_stable_sort(n, kind):
    s, lab = _make(kind, n, seed=n % 1000 + len(kind))
    out, order, fnr, fpr = _raw(s, lab)
    assert int(out[7].item()) & 7 == 0
    want = torch.sort(s + 0.0, stable=True).indices.to(torch.int32)      # + 0.0: -0.0 -> +0.0, equal as in numpy
    assert torch.equal(order, want)
    if n <= (1 << 20) + 3:
        rf, rp = metrics_np.pmiss_pfa_rbst(s.cpu().numpy(), lab.cpu().numpy())
        assert _same_bits(fnr.cpu().numpy(), rf) and _same_bits(fpr.cpu().numpy(), rp)
    else:
        t = torch.cumsum(lab[want.long()].to(torch.int64), 0).cpu().numpy()   # numpy: correctly rounded divisions
        f = np.arange(1, n + 1) - t
        assert _same_bits(fnr.cpu().numpy(), t / float(t[-1]))
        assert _same_bits(fpr.cpu().numpy(), 1 - f / float(f[-1]))


@gpu
@pytest.mark.parametrize("name", CASES)
def test_gpu_evaluate_matches_reference_goldens(name):
    s, lab = _case(name)
    fnr, fpr = metrics.compute_pmiss_pfa_rbst(s, lab)
    assert _same_curve(name, "fnr", fnr) and _same_curve(name, "fpr", fpr)
    if name + "_eer" not in G:
        with pytest.raises(lib.B200Error, match="x2"):
            metrics.evaluate(s, lab, POINTS)
        return
    runs = [metrics.evaluate(s, lab, POINTS, curve=True) for _ in range(2)]
    for m in runs:
        assert _same_bits(m.eer, G[name + "_eer"]) and _same_bits(m.threshold, G[name + "_thr"])
        assert _same_bits(m.min_dcf, G[name + "_min_dcf"]) and _same_bits(m.c_det, G[name + "_c_det"])
    a, b = runs
    assert torch.equal(a.order, b.order) and a.fnr.cpu().numpy().tobytes() == b.fnr.cpu().numpy().tobytes()
    assert a.fpr.cpu().numpy().tobytes() == b.fpr.cpu().numpy().tobytes()
    assert _same_bits(metrics.compute_eer(fnr, fpr, s)[0], G[name + "_eer"])
    assert _same_bits(metrics.compute_c_norm(fnr, fpr, *POINTS[0]), G[name + "_min_dcf"][0])


@gpu
@pytest.mark.parametrize("n", [37720, 579818])
def test_gpu_evaluate_matches_oracle_with_mixed_ties(n):
    rng = np.random.default_rng(n)
    lab = rng.random(n) < 0.05
    s = np.round(0.2 * rng.standard_normal(n) + 0.3 * lab, 3)            # ties that mix the classes
    s[rng.random(n) < 0.01] = -0.0
    fnr, fpr = metrics_np.pmiss_pfa_rbst(s, lab)
    eer, thr = metrics_np.eer(fnr, fpr, s)
    for scores in (s, torch.from_numpy(s).cuda(), torch.from_numpy(s.astype(np.float32)).cuda()):
        ref = (fnr, fpr, eer, thr)
        if isinstance(scores, torch.Tensor) and scores.dtype == torch.float32:
            s32 = scores.cpu().numpy().astype(np.float64)
            f32, p32 = metrics_np.pmiss_pfa_rbst(s32, lab)
            ref = (f32, p32) + tuple(metrics_np.eer(f32, p32, s32))
        m = metrics.evaluate(scores, lab, POINTS, curve=True)
        assert _same_bits(m.fnr.cpu().numpy(), ref[0]) and _same_bits(m.fpr.cpu().numpy(), ref[1])
        assert _same_bits(m.eer, ref[2]) and _same_bits(m.threshold, ref[3])
        assert _same_bits(m.c_det, [metrics_np.c_det(ref[0], ref[1], *p) for p in POINTS])
        assert _same_bits(m.min_dcf, [metrics_np.c_norm(ref[0], ref[1], *p) for p in POINTS])


@gpu
@pytest.mark.parametrize("case,bit,cause", [
    ("nan", 1, "NaN"), ("label2", 2, "label"), ("no_target", 4, "no target"), ("no_nontarget", 4, "no target"),
    ("n1", 4, "no target")])
def test_gpu_data_refusals_write_only_the_status(case, bit, cause):
    n = 1 if case == "n1" else 5000
    s = torch.randn(n, dtype=torch.float64, device="cuda")
    lab = (torch.arange(n, device="cuda") % 3 == 0).to(torch.uint8)
    if case == "nan":
        s[1234] = float("nan")
    elif case == "label2":
        lab[4000] = 2
    elif case == "no_target":
        lab.zero_()
    elif case == "no_nontarget":
        lab.fill_(1)
    out, order, fnr, fpr = _raw(s, lab, fill=7)
    assert int(out[7].item()) == bit
    assert (out[:7] == 7).all() and (out[8:] == 7).all()
    assert (order == 7).all() and (fnr == 7).all() and (fpr == 7).all()
    with pytest.raises(lib.B200Error, match=cause):
        metrics.evaluate(s, lab)
    if case == "label2":
        with pytest.raises(lib.B200Error, match="label"):
            metrics.evaluate(s.cpu().numpy(), np.where(lab.cpu().numpy() == 2, 300, lab.cpu().numpy()).astype(np.int64))


@gpu
def test_gpu_empty_trial_list_is_refused():
    with pytest.raises(lib.B200Error, match="no trials"):
        metrics.evaluate(np.zeros(0), np.zeros(0, dtype=bool))


@gpu
@pytest.mark.parametrize("name", ["ties_a", "ties_b", "stable_only"])
def test_gpu_compute_metrics_prints_the_reference_text(tmp_path, name):
    path = tmp_path / (name + ".score")
    path.write_bytes(G[name + "_text"].item())
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        metrics.main(0.01, 1, 1, str(path))
        metrics.compute_metrics(str(path), 0.05, 2, 1)
    assert buf.getvalue() == str(G[name + "_stdout"])


@gpu
def test_gpu_compute_det_needs_matplotlib_or_writes_the_plot(tmp_path):
    path = tmp_path / "t.score"
    path.write_bytes(G["ties_a_text"].item())
    try:
        import matplotlib  # noqa: F401
    except ImportError:
        with pytest.raises(ImportError, match="matplotlib"):
            metrics.det_main(str(path))
        return
    metrics.det_main(str(path))
    assert os.path.getsize(str(path) + ".det.png") > 0


@gpu
def test_gpu_calibration_training_matches_reference(tmp_path):
    fac = tmp_path / "factor"
    fac.write_text("\n".join(_factor_lines()) + "\n")
    model = tmp_path / "model.pt"
    losses = calibration.train_calibration_model(str(fac), str(model))
    # The loop is the reference's (on the CPU it reproduces every golden loss bit for bit), but LBFGS amplifies the GPU's
    # different rounding over the epochs: the first epochs agree closely, the stopping epoch and the final weights need
    # not.  What is pinned is the trajectory's start and the quality of the optimum.
    assert np.allclose(losses[:8], G["cal_losses"][:8], rtol=1e-6, atol=0), (losses, G["cal_losses"])
    sd = torch.load(str(model))
    assert set(sd) == {"linear.weight", "linear.bias"} and all(v.device.type == "cpu" and v.dtype == torch.float64
                                                             for v in sd.values())
    rows = [ln.split() for ln in fac.read_text().splitlines()]
    x = torch.tensor([[float(v) for v in r[3:]] for r in rows], dtype=torch.float64)
    is_t = torch.tensor([r[2] == "target" for r in rows])
    llr = x @ sd["linear.weight"].T + sd["linear.bias"]
    assert abs(float(calibration.cllr(llr[is_t], llr[~is_t])) - float(G["cal_final_cllr"])) <= 1e-3
    # our model file in the reference's layout loads into the reference-shaped LinearModel, and the reverse
    m = calibration.LinearModel(x.shape[1]).double()
    m.load_state_dict(sd)


@gpu
def test_gpu_calibration_inference_with_reference_weights(tmp_path):
    fac = tmp_path / "factor"
    lines = _factor_lines()
    fac.write_text("\n".join(lines) + "\n")
    model = tmp_path / "ref_model.pt"
    torch.save({"linear.weight": torch.from_numpy(G["cal_weight"]), "linear.bias": torch.from_numpy(G["cal_bias"])},
               str(model))
    out = tmp_path / "cal.score"
    calibration.infer_calibration(str(fac), str(model), str(out))
    got = [ln.split() for ln in out.read_text().splitlines()]
    assert [g[:2] + g[3:] for g in got] == [ln.split()[:3] for ln in lines]
    s = np.array([float(g[2]) for g in got])
    assert np.abs(s - G["cal_scores"]).max() <= 1e-12 * max(1.0, np.abs(G["cal_scores"]).max())
