"""CPU: the engine's model table and the refusals every compute entry point shares (plan-check engines, no device)."""
import ctypes as C

import numpy as np
import pytest

from wespeaker_b200 import lib
from wespeaker_b200.models import SUPPORTED_MODELS, from_synthetic


@pytest.mark.parametrize("name", SUPPORTED_MODELS)
def test_every_supported_model_builds_a_plan(name):
    """Every name the package supports is a row of the engine's model table: a plan-check engine accepts it and its family's
    builder turns the synthetic checkpoint into a launch plan."""
    ops = from_synthetic(name, precision="bf16").plan_check(2, 200)
    assert len(ops) >= 5 and all(isinstance(n, str) and n for n, _ in ops)


@pytest.mark.parametrize("name", ["ECAPA_TDNN_c256", "ResNet", "ResNet35", "Res2Net50", "CAMPPlus2", "ERes2Net34", ""])
def test_a_name_outside_the_model_table_is_refused(name):
    """No name reaches a builder by falling through: near misses of table rows are unknown models."""
    L = lib.load()
    h = lib.c_engine_p()
    assert L.ws_engine_create_plan_check(name.encode(), b"bf16", 80, 192, C.byref(h)) != 0
    assert b"unknown / out-of-scope model name" in L.ws_last_error()


def test_every_compute_entry_point_refuses_on_a_plan_check_engine():
    """The eleven compute entry points (and the two test / tuning ones that run ops) refuse on a plan-check engine before
    they touch any buffer.  Every pointer argument is a real host buffer, so a regression fails the call instead of
    crashing the test."""
    L = lib.load()
    h = lib.c_engine_p()
    lib.check(L.ws_engine_create_plan_check(b"ECAPA_TDNN_c512", b"bf16", 80, 192, C.byref(h)), "create")
    B, T, ns = 2, 200, 32000
    feats = np.zeros((B, T, 80), np.float32)
    embs = np.zeros((B, 192), np.float32)
    wav = np.zeros((B, ns), np.float32)
    nfr = np.full(B, T, np.int32)
    nsm = np.full(B, ns, np.int32)
    offs = np.arange(B, dtype=np.int64) * ns
    ms = np.zeros(4096, np.float32)
    f, o, w = feats.ctypes.data, embs.ctypes.data, wav.ctypes.data
    calls = {
        "ws_engine_forward": lambda: L.ws_engine_forward(h, f, B, T, o, None),
        "ws_engine_forward_async": lambda: L.ws_engine_forward_async(h, f, B, T, o, None),
        "ws_engine_forward_masked": lambda: L.ws_engine_forward_masked(h, f, nfr.ctypes.data, B, T, o, None),
        "ws_engine_forward_host": lambda: L.ws_engine_forward_host(h, f, B, T, o),
        "ws_engine_extract_wav": lambda: L.ws_engine_extract_wav(h, w, 0, ns, ns, B, b"hamming", o, f, None),
        "ws_engine_extract_wav_async": lambda: L.ws_engine_extract_wav_async(h, w, 0, ns, ns, B, b"hamming", o, None),
        "ws_engine_extract_wav_host": lambda: L.ws_engine_extract_wav_host(h, w, 0, ns, B, b"hamming", o),
        "ws_engine_submit_wav_host": lambda: L.ws_engine_submit_wav_host(h, 0, w, 0, ns, B, b"hamming", o),
        "ws_engine_extract_wav_masked": lambda: L.ws_engine_extract_wav_masked(h, w, 0, ns, nsm.ctypes.data, ns, B, b"hamming", o,
                                                                               None),
        "ws_engine_extract_wav_ragged": lambda: L.ws_engine_extract_wav_ragged(h, w, 0, offs.ctypes.data, nsm.ctypes.data, ns, B,
                                                                               b"hamming", o, None),
        "ws_engine_extract_wav_ragged_async": lambda: L.ws_engine_extract_wav_ragged_async(h, w, 0, offs.ctypes.data,
                                                                                           nsm.ctypes.data, ns, B, b"hamming", o,
                                                                                           None),
        "ws_engine_run_ops": lambda: L.ws_engine_run_ops(h, B, T, 0, 0, 1, None),
        "ws_engine_profile_ops": lambda: L.ws_engine_profile_ops(h, B, T, 1, ms.ctypes.data, ms.size),
    }
    try:
        for name, call in calls.items():
            assert call() != 0, name
            err = L.ws_last_error()
            assert err.startswith(name.encode()) and b"plan-check engine" in err, (name, err)
    finally:
        L.ws_engine_destroy(h)
    assert not embs.any() and not feats.any()
