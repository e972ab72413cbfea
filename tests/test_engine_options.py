"""CPU: the engine options on plan-check engines (no device).  The header's option list names every option the engine
accepts; each documented default is the engine's default, and each other value reaches the field that changes the plan."""
import ctypes as C
import functools
import os
import re
import sys
import tempfile

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from plan_digest import canonical  # noqa: E402
from wespeaker_b200 import lib  # noqa: E402
from wespeaker_b200.models import from_synthetic  # noqa: E402

OPTIONS = ("two_emb_layer", "emb_bn", "cuda_graph", "res2_fused", "se_fused", "se_colsum", "conv3x3", "cam_fused", "cam_block",
           "astp_fused", "plan_trace", "tc_version", "sample_rate")
MODEL_ARGS = ("two_emb_layer", "emb_bn")
# option -> a case whose plan the option changes: (model, precision, B, T, a value other than the default).  tc_version needs
# a batch at which some layer reaches the cluster kernel's 132 x 128 output positions.
PLAN_OPTIONS = {
    "two_emb_layer": ("ResNet34", "fp16", 2, 200, 1),
    "emb_bn": ("ECAPA_TDNN_c512", "bf16", 2, 200, 1),
    "res2_fused": ("ECAPA_TDNN_c512", "bf16", 2, 200, 0),
    "se_fused": ("ECAPA_TDNN_c512", "bf16", 2, 200, 0),
    "se_colsum": ("ECAPA_TDNN_c512", "bf16", 2, 200, 0),
    "astp_fused": ("ECAPA_TDNN_c512", "bf16", 2, 200, 0),
    "tc_version": ("ECAPA_TDNN_c512", "bf16", 128, 200, 2),
    "conv3x3": ("ResNet34", "fp16", 2, 200, 0),
    "cam_fused": ("CAMPPlus", "bf16", 2, 200, 0),
    "cam_block": ("CAMPPlus", "bf16", 2, 200, 0),
}


def header_options():
    """{name: default} of the option list in include/wespeaker_b200.h"""
    hdr = open(os.path.join(ROOT, "include", "wespeaker_b200.h")).read()
    block = hdr[hdr.index("/* Engine options"):hdr.index("int ws_engine_set_option")]
    return {n: int(d) for n, d in re.findall(r'^ \*   "(\w+)" \((\d+)\)', block, re.M)}


@functools.lru_cache(maxsize=None)
def plan(name, prec, B, T, option=None, value=None):
    """the canonical plan (tools/plan_digest.py) of a synthetic model, with one option set (model_args for two_emb_layer and
    emb_bn) or none"""
    args = {option: bool(value)} if option in MODEL_ARGS else {}
    m = from_synthetic(name, 0, precision=prec, **args)
    if option is not None and option not in MODEL_ARGS:
        m.set_option(option, value)
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "plan.wspt")
        m.plan_trace(path, B, T)
        return canonical(path)


def plan_check_engine(precision=b"bf16"):
    L = lib.load()
    h = lib.c_engine_p()
    lib.check(L.ws_engine_create_plan_check(b"ECAPA_TDNN_c512", precision, 80, 192, C.byref(h)), "create")
    return L, h


def test_the_header_lists_every_option_and_each_is_accepted():
    assert tuple(header_options()) == OPTIONS
    L, h = plan_check_engine()
    try:
        for name, default in header_options().items():
            assert L.ws_engine_set_option(h, name.encode(), default) == 0, (name, L.ws_last_error())
    finally:
        L.ws_engine_destroy(h)


@pytest.mark.parametrize("option", sorted(PLAN_OPTIONS))
def test_the_documented_default_is_the_default_and_another_value_changes_the_plan(option):
    name, prec, B, T, other = PLAN_OPTIONS[option]
    default = header_options()[option]
    assert other != default
    unset = plan(name, prec, B, T)
    assert plan(name, prec, B, T, option, default) == unset
    assert plan(name, prec, B, T, option, other) != unset


@pytest.mark.parametrize("key,value,message", [
    ("se_fuse", 1, b"unknown option se_fuse"),
    ("tc_versions", 3, b"unknown option tc_versions"),
    ("Cuda_graph", 0, b"unknown option Cuda_graph"),
    ("emb-bn", 1, b"unknown option emb-bn"),
    ("", 1, b"unknown option "),
    ("tc_version", 1, b"tc_version must be 2"),
    ("tc_version", 4, b"tc_version must be 2"),
    ("sample_rate", 11025, b"sample_rate must be 8000 or 16000"),
])
def test_unknown_names_and_values_are_refused(key, value, message):
    L, h = plan_check_engine()
    try:
        assert L.ws_engine_set_option(h, key.encode(), value) != 0
        assert L.ws_last_error().startswith(message), L.ws_last_error()
    finally:
        L.ws_engine_destroy(h)


def test_an_unknown_precision_is_refused():
    L = lib.load()
    h = lib.c_engine_p()
    assert L.ws_engine_create_plan_check(b"ECAPA_TDNN_c512", b"bf32", 80, 192, C.byref(h)) != 0
    assert L.ws_last_error() == b"unknown precision (fp32|tf32x3|tf32|bf16|fp16): bf32"


def test_tc_version_leaves_fp32_on_ffma():
    """fp32 runs FFMA whatever tc_version says: at the batch where tc_version selects the bf16 plan's kernels, the fp32 plan is
    the same with tc_version 2 as without it, and has no tensor-core conv."""
    unset = plan("ECAPA_TDNN_c512", "fp32", 128, 200)
    assert plan("ECAPA_TDNN_c512", "fp32", 128, 200, "tc_version", 2) == unset
    labels = re.findall(r'"label": "(\w+)', unset)
    assert "conv_simt" in labels and not any(n.startswith("conv_tc") for n in labels)
