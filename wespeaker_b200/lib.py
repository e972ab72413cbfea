"""ctypes binding of the C ABI in include/wespeaker_b200.h (the only way the Python host code reaches
the CUDA kernels).  There is no CPU fallback: if the in-tree shared library is missing or no CUDA
device is present, calls fail loudly."""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libwespeaker_b200.so")
_lib = None

c_engine_p = C.c_void_p
c_plda_p = C.c_void_p


class B200Error(RuntimeError):
    pass


class ConvDesc(C.Structure):
    """ws_conv_desc (include/wespeaker_b200.h)."""
    _fields_ = [
        ("x", C.c_void_p), ("B", C.c_int), ("F", C.c_int), ("T", C.c_int), ("Cin", C.c_int),
        ("x_ld", C.c_longlong), ("w", C.c_void_p), ("Cout", C.c_int), ("kf", C.c_int), ("kt", C.c_int),
        ("dil_f", C.c_int), ("dil_t", C.c_int), ("pad_f", C.c_int), ("pad_t", C.c_int),
        ("stride_f", C.c_int), ("stride_t", C.c_int), ("bias", C.c_void_p), ("act1", C.c_int),
        ("scale", C.c_void_p), ("shift", C.c_void_p), ("res", C.c_void_p), ("res_ld", C.c_longlong),
        ("act2", C.c_int), ("out", C.c_void_p), ("out_ld", C.c_longlong), ("dtype", C.c_int),
        ("use_tc", C.c_int), ("x_lo", C.c_void_p), ("w_lo", C.c_void_p), ("out_lo", C.c_void_p),
        ("colsum", C.c_void_p),
    ]


class SimamDesc(C.Structure):
    """ws_simam_desc (include/wespeaker_b200.h)."""
    _fields_ = [
        ("y", C.c_void_p), ("y_ld", C.c_longlong), ("B", C.c_int), ("F", C.c_int), ("T", C.c_int), ("C", C.c_int),
        ("lens", C.c_void_p), ("lambda_p", C.c_float), ("res", C.c_void_p), ("res_sb", C.c_longlong),
        ("res_sf", C.c_longlong), ("res_st", C.c_longlong), ("out", C.c_void_p), ("out_sb", C.c_longlong),
        ("out_sf", C.c_longlong), ("out_st", C.c_longlong), ("out_lo", C.c_void_p), ("dtype", C.c_int),
        ("stats", C.c_void_p), ("partial", C.c_void_p),
    ]


class DwConvDesc(C.Structure):
    """ws_dwconv_desc (include/wespeaker_b200.h)."""
    _fields_ = [
        ("x", C.c_void_p), ("x_ld", C.c_longlong), ("B", C.c_int), ("F", C.c_int), ("T", C.c_int), ("C", C.c_int),
        ("lens", C.c_void_p), ("w", C.c_void_p), ("shift", C.c_void_p), ("out", C.c_void_p), ("out_ld", C.c_longlong),
        ("out_lo", C.c_void_p), ("dtype", C.c_int),
    ]


_PROTOS = {
    "ws_version": (C.c_int, []),
    "ws_last_error": (C.c_char_p, []),
    "ws_engine_create": (C.c_int, [C.c_char_p, C.c_char_p, C.c_int, C.c_int, C.c_int, C.POINTER(c_engine_p)]),
    "ws_engine_create_plan_check": (C.c_int, [C.c_char_p, C.c_char_p, C.c_int, C.c_int, C.POINTER(c_engine_p)]),
    "ws_engine_set_option": (C.c_int, [c_engine_p, C.c_char_p, C.c_longlong]),
    "ws_engine_set_tensor": (C.c_int, [c_engine_p, C.c_char_p, C.c_void_p, C.POINTER(C.c_longlong), C.c_int]),
    "ws_engine_finalize": (C.c_int, [c_engine_p]),
    "ws_engine_embed_dim": (C.c_int, [c_engine_p]),
    "ws_engine_forward": (C.c_int, [c_engine_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "ws_engine_forward_masked": (C.c_int, [c_engine_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "ws_engine_extract_wav_masked": (C.c_int, [c_engine_p, C.c_void_p, C.c_int, C.c_longlong, C.c_void_p, C.c_int, C.c_int,
                                               C.c_char_p, C.c_void_p, C.c_void_p]),
    "ws_engine_extract_wav_ragged": (C.c_int, [c_engine_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                               C.c_char_p, C.c_void_p, C.c_void_p]),
    "ws_engine_extract_wav_ragged_async": (C.c_int, [c_engine_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                                     C.c_char_p, C.c_void_p, C.c_void_p]),
    "ws_resample_out_len": (C.c_int, [C.c_int, C.c_int, C.c_int]),
    "ws_resample": (C.c_int, [C.c_void_p, C.c_int, C.c_longlong, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_longlong, C.c_void_p]),
    "ws_engine_forward_async": (C.c_int, [c_engine_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "ws_engine_extract_wav_async": (C.c_int, [c_engine_p, C.c_void_p, C.c_int, C.c_longlong, C.c_int, C.c_int,
                                              C.c_char_p, C.c_void_p, C.c_void_p]),
    "ws_engine_join": (C.c_int, [c_engine_p, C.c_void_p]),
    "ws_engine_forward_host": (C.c_int, [c_engine_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]),
    "ws_engine_extract_wav": (C.c_int, [c_engine_p, C.c_void_p, C.c_int, C.c_longlong, C.c_int, C.c_int,
                                        C.c_char_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ws_engine_extract_wav_host": (C.c_int, [c_engine_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_char_p,
                                             C.c_void_p]),
    "ws_engine_submit_wav_host": (C.c_int, [c_engine_p, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_char_p,
                                            C.c_void_p]),
    "ws_engine_collect": (C.c_int, [c_engine_p, C.c_int]),
    "ws_engine_plan_op_name": (C.c_char_p, [c_engine_p, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "ws_engine_plan_trace": (C.c_int, [c_engine_p, C.c_int, C.c_int, C.c_int, C.c_char_p]),
    "ws_engine_run_ops": (C.c_int, [c_engine_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "ws_engine_profile_ops": (C.c_int, [c_engine_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int]),
    "ws_engine_last_launches": (C.c_longlong, [c_engine_p]),
    "ws_engine_destroy": (None, [c_engine_p]),
    "ws_fbank_num_frames": (C.c_int, [C.c_int]),
    "ws_fbank_num_frames_at": (C.c_int, [C.c_int, C.c_int]),
    "ws_fbank_at": (C.c_int, [C.c_void_p, C.c_int, C.c_longlong, C.c_int, C.c_int, C.c_char_p, C.c_int, C.c_int, C.c_int,
                              C.c_void_p, C.c_void_p]),
    "ws_fbank_ragged_at": (C.c_int, [C.c_void_p, C.c_int, C.c_longlong, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_char_p,
                                     C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "ws_fbank": (C.c_int, [C.c_void_p, C.c_int, C.c_longlong, C.c_int, C.c_int, C.c_char_p, C.c_int, C.c_void_p,
                           C.c_void_p]),
    "ws_fbank_ragged": (C.c_int, [C.c_void_p, C.c_int, C.c_longlong, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_char_p,
                                  C.c_void_p, C.c_void_p]),
    "ws_conv": (C.c_int, [C.POINTER(ConvDesc), C.c_void_p]),
    "ws_simam": (C.c_int, [C.POINTER(SimamDesc), C.c_void_p]),
    "ws_dwconv": (C.c_int, [C.POINTER(DwConvDesc), C.c_void_p]),
    "ws_plda_create": (C.c_int, [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                 C.POINTER(c_plda_p)]),
    "ws_plda_transform": (C.c_int, [c_plda_p, C.c_void_p, C.c_longlong, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "ws_plda_transform64": (C.c_int, [c_plda_p, C.c_void_p, C.c_longlong, C.c_int, C.c_void_p, C.c_void_p]),
    "ws_plda_score_matrix": (C.c_int, [c_plda_p, C.c_void_p, C.c_void_p, C.c_int, C.c_longlong, C.c_void_p,
                                       C.c_longlong, C.c_void_p, C.c_int, C.c_longlong, C.c_void_p]),
    "ws_plda_score_trials": (C.c_int, [c_plda_p, C.c_void_p, C.c_void_p, C.c_int, C.c_longlong, C.c_void_p,
                                       C.c_longlong, C.c_void_p, C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p]),
    "ws_plda_destroy": (None, [c_plda_p]),
    "ws_score_unit_rows": (C.c_int, [C.c_void_p, C.c_longlong, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ws_score_cosine_trials": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong, C.c_int, C.c_void_p, C.c_void_p]),
    "ws_score_cohort_stats": (C.c_int, [C.c_void_p, C.c_longlong, C.c_void_p, C.c_longlong, C.c_int, C.c_int, C.c_void_p,
                                        C.c_longlong, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ws_score_asnorm": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_longlong, C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.c_void_p, C.c_void_p, C.c_void_p]),
    "ws_diar_col_means": (C.c_int, [C.c_void_p, C.c_longlong, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "ws_diar_windows": (C.c_int, [C.c_void_p, C.c_longlong, C.c_int, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int,
                                  C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "ws_diar_laplacian": (C.c_int, [C.c_void_p, C.c_longlong, C.c_int, C.c_longlong, C.c_void_p, C.c_longlong, C.c_void_p,
                                    C.c_void_p, C.c_void_p]),
    "ws_metrics_work_bytes": (C.c_size_t, [C.c_longlong]),
    "ws_metrics_eval": (C.c_int, [C.c_void_p, C.c_void_p, C.c_longlong, C.POINTER(C.c_double), C.POINTER(C.c_double),
                                  C.POINTER(C.c_double), C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p,
                                  C.c_void_p, C.c_void_p, C.c_void_p]),
}
EXPORTED_SYMBOLS = tuple(_PROTOS.keys())


def build(verbose: bool = False) -> str:
    """Compile the CUDA library in-tree for sm_90a (nvcc cross-compiles without a GPU)."""
    script = os.path.join(os.path.dirname(_HERE), "build.sh")
    r = subprocess.run(["bash", script], capture_output=True, text=True)
    if verbose or r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
    if r.returncode != 0:
        raise B200Error("building libwespeaker_b200.so failed")
    return LIB_PATH


def load():
    """Load the shared library (no CUDA call happens at load time)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise B200Error(f"{LIB_PATH} is missing: run `bash build.sh` (or __graft_entry__.build()); "
                        "wespeaker_b200 has no CPU fallback")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in _PROTOS.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc: int, what: str = ""):
    if rc != 0:
        msg = load().ws_last_error()
        raise B200Error(f"{what}: {msg.decode() if msg else 'unknown error'}")


def cur_stream_ptr(device=None) -> int:
    import torch
    return int(torch.cuda.current_stream(device).cuda_stream)
