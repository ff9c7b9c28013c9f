"""ctypes binding of libbanet.so (C-ABI declared in include/banet_abi.h).

There is NO fallback: if the shared library is missing or a call fails, an exception is raised.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("BANET_LIB_PATH") or os.path.join(_HERE, "libbanet.so")      # the override is for kernel-variant timing scripts only

BANET_OK = 0
PREC_AUTO, PREC_FP32_SIMT, PREC_TF32X1, PREC_TF32X2, PREC_TF32X3, PREC_TF32_LEVELWISE = -1, 0, 1, 2, 3, 4

c_float_p = C.c_void_p      # raw device pointers
c_stream = C.c_void_p


class BanetLevel(C.Structure):
    """struct banet_level (include/banet_abi.h)."""
    _fields_ = [("nb", C.c_int), ("N", C.c_int), ("C", C.c_int), ("K", C.c_int),
                ("h", C.c_int), ("w", C.c_int), ("conv2_channels", C.c_int),
                ("conv1", C.c_void_p), ("conv2", C.c_void_p), ("intr", C.c_void_p),
                ("p", C.c_void_p), ("D", C.c_void_p), ("B", C.c_void_p),
                ("grid_w", C.c_int), ("grid_h", C.c_int)]


class BanetSolveOpts(C.Structure):
    """struct banet_solve_opts (include/banet_abi.h)."""
    _fields_ = [("damping_eps", C.c_float), ("undamped_last", C.c_int), ("vmatrix_batch_scramble", C.c_int)]


class BanetTuning(C.Structure):
    """struct banet_tuning (include/banet_abi.h): diagnostic knobs, defaults = production."""
    _fields_ = [("tc_generation", C.c_int), ("tc7_force_direct", C.c_int), ("tc7_band_rows", C.c_int),
                ("tc6_band_rows", C.c_int), ("tc6_l2_hints", C.c_int), ("tc6_tap_prefetch", C.c_int)]


class BanetLegacyOpts(C.Structure):
    """struct banet_legacy_opts (include/banet_abi.h): the module-level knobs of legacy/ba.py:5-8."""
    _fields_ = [("early_termination", C.c_int), ("angle_change", C.c_float), ("translation_change", C.c_float), ("residual_ratio", C.c_float)]


class BanetError(RuntimeError):
    pass


# name -> (restype, argtypes); every symbol declared in include/banet_abi.h
SIGNATURES = {
    "banet_abi_version": (C.c_int, []),
    "banet_last_error": (C.c_char_p, []),
    "banet_device_check": (C.c_int, []),
    "banet_num_sms": (C.c_int, []),
    "banet_set_tuning": (C.c_int, [C.POINTER(BanetTuning)]),
    "banet_get_tuning": (C.c_int, [C.POINTER(BanetTuning)]),
    "banet_eqc_workspace_bytes": (C.c_size_t, [C.c_int] * 4),
    "banet_eqc_fwd": (C.c_int, [c_float_p] * 3 + [C.c_int] * 4 + [c_float_p] * 2 + [C.c_void_p, C.c_size_t, c_stream]),
    "banet_eqc_bwd": (C.c_int, [c_float_p] * 5 + [C.c_int] * 5 + [c_float_p] * 3 + [c_stream]),
    "banet_compute_coordinates": (C.c_int, [c_float_p, c_float_p, C.c_int, C.c_int, C.c_int, c_float_p, c_stream]),
    "banet_grad_fixed_concat": (C.c_int, [c_float_p] + [C.c_int] * 5 + [c_float_p, c_stream]),
    "banet_resample": (C.c_int, [c_float_p, c_float_p, C.c_float] + [C.c_int] * 5 + [c_float_p, c_stream]),
    "banet_interpolate2d": (C.c_int, [c_float_p, c_float_p, C.c_float] + [C.c_int] * 5 + [c_float_p, c_float_p, c_stream]),
    "banet_lm_build_workspace_bytes": (C.c_size_t, [C.POINTER(BanetLevel), C.c_int]),
    "banet_lm_build": (C.c_int, [C.POINTER(BanetLevel)] + [c_float_p] * 3 + [C.c_int] + [c_float_p] * 4
                       + [C.c_void_p, C.c_size_t, c_stream]),
    "banet_mlp_param_count": (C.c_size_t, [C.c_int]),
    "banet_lm_lambda": (C.c_int, [c_float_p, C.c_int, C.c_int, C.c_int, c_float_p, C.c_float, c_float_p, c_stream]),
    "banet_lm_solve_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "banet_lm_solve_update": (C.c_int, [c_float_p] * 3 + [C.c_int, C.c_int, C.POINTER(BanetSolveOpts)] + [c_float_p] * 3
                              + [c_float_p] * 4 + [C.c_void_p] + [C.c_void_p, C.c_size_t, c_stream]),
    "banet_lm_run_workspace_bytes": (C.c_size_t, [C.POINTER(BanetLevel), C.c_int, C.c_int]),
    "banet_lm_run": (C.c_int, [C.POINTER(BanetLevel), C.c_int, C.c_int, C.POINTER(C.c_void_p), C.c_float, C.c_float,
                               C.POINTER(BanetSolveOpts), C.c_int] + [c_float_p] * 3 + [C.c_void_p]
                     + [C.c_void_p, C.c_size_t, c_stream]),
    "banet_lm_window_run_workspace_bytes": (C.c_size_t, [C.POINTER(BanetLevel), C.c_int, C.c_int]),
    "banet_lm_window_run": (C.c_int, [C.POINTER(BanetLevel), C.c_int, C.c_int, C.POINTER(C.c_void_p), C.c_float, C.c_float,
                                      C.POINTER(BanetSolveOpts), C.c_int] + [c_float_p] * 3 + [C.c_void_p]
                            + [C.c_void_p, C.c_size_t, c_stream]),
    "banet_lm_window_solve_update_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "banet_lm_window_solve_update": (C.c_int, [c_float_p] * 3 + [C.c_int, C.c_int, C.POINTER(BanetSolveOpts)] + [c_float_p] * 3
                                     + [c_float_p] * 4 + [C.c_void_p] + [C.c_void_p, C.c_size_t, c_stream]),
    "banet_lm_window_solve_update_bwd_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int]),
    "banet_lm_window_solve_update_bwd": (C.c_int, [c_float_p] * 4 + [C.c_int, C.c_int, C.POINTER(BanetSolveOpts)] + [c_float_p] * 5
                                         + [c_float_p] * 6 + [C.c_void_p, C.c_size_t, c_stream]),
    "banet_lm_window_batch_run_workspace_bytes": (C.c_size_t, [C.POINTER(BanetLevel), C.c_int, C.c_int, C.c_int]),
    "banet_lm_window_batch_run": (C.c_int, [C.POINTER(BanetLevel), C.c_int, C.c_int, C.c_int, C.POINTER(C.c_void_p), C.c_float, C.c_float,
                                            C.POINTER(BanetSolveOpts), C.c_int] + [c_float_p] * 3 + [C.c_void_p]
                                  + [C.c_void_p, C.c_size_t, c_stream]),
    "banet_lm_window_batch_solve_update_workspace_bytes": (C.c_size_t, [C.c_int] * 3),
    "banet_lm_window_batch_solve_update": (C.c_int, [c_float_p] * 3 + [C.c_int] * 3 + [C.POINTER(BanetSolveOpts)] + [c_float_p] * 3
                                           + [c_float_p] * 4 + [C.c_void_p] + [C.c_void_p, C.c_size_t, c_stream]),
    "banet_lm_window_batch_solve_update_bwd_workspace_bytes": (C.c_size_t, [C.c_int] * 3),
    "banet_lm_window_batch_solve_update_bwd": (C.c_int, [c_float_p] * 4 + [C.c_int] * 3 + [C.POINTER(BanetSolveOpts)] + [c_float_p] * 5
                                               + [c_float_p] * 6 + [C.c_void_p, C.c_size_t, c_stream]),
    "banet_depth_compose": (C.c_int, [c_float_p] * 3 + [C.c_int] * 3 + [c_float_p, c_stream]),
    "banet_lm_step": (C.c_int, [c_float_p] * 3 + [C.c_int] * 4 + [c_float_p, C.c_float, c_float_p, C.POINTER(BanetSolveOpts)] + [c_float_p] * 3
                      + [c_float_p] * 3 + [c_float_p, c_float_p, C.c_void_p, c_stream]),
    "banet_lm_track_legacy_workspace_bytes": (C.c_size_t, [C.POINTER(BanetLevel), C.c_int]),
    "banet_lm_track_legacy": (C.c_int, [C.POINTER(BanetLevel), C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_void_p), C.POINTER(BanetLegacyOpts)]
                              + [c_float_p] * 2 + [C.c_void_p, c_float_p, C.c_void_p] + [C.c_void_p, C.c_size_t, c_stream]),
    "banet_lm_build_bwd": (C.c_int, [C.POINTER(BanetLevel)] + [c_float_p] * 6 + [C.c_int] + [c_float_p] * 7 + [c_stream]),
    "banet_lm_solve_update_bwd": (C.c_int, [c_float_p] * 4 + [C.c_int, C.c_int, C.POINTER(BanetSolveOpts)] + [c_float_p] * 5 + [c_float_p] * 6 + [c_stream]),
    "banet_grad_fixed_concat_bwd": (C.c_int, [c_float_p] + [C.c_int] * 5 + [c_float_p, c_stream]),
    "banet_resample_bwd": (C.c_int, [c_float_p, c_float_p, C.c_float] + [C.c_int] * 5 + [c_float_p, c_stream]),
    "banet_depth_compose_bwd": (C.c_int, [c_float_p] * 3 + [C.c_int] * 3 + [c_float_p, c_float_p, c_stream]),
    "banet_tc_selftest": (C.c_int, [c_float_p] * 3 + [C.c_int, C.c_int, C.c_int, c_stream]),
}

_lib: Optional[C.CDLL] = None


def load() -> C.CDLL:
    """Load the library and bind every declared symbol.  Raises if it is absent (no CPU fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise BanetError(f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                         f"(or `make -C banet_b200/csrc`). banet_b200 has no CPU fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if a declared symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc: int, what: str) -> None:
    if rc != BANET_OK:
        msg = load().banet_last_error().decode("utf-8", "replace")
        raise BanetError(f"{what} failed (code {rc}): {msg}")


def set_tuning(tc_generation: int = 0, tc7_force_direct: bool = False, tc7_band_rows: int = 4, tc6_band_rows: int = 0,
               tc6_l2_hints: int = 0, tc6_tap_prefetch: int = 0) -> None:
    """Diagnostic knobs (process-wide); call with no arguments to restore the production defaults."""
    t = BanetTuning(int(tc_generation), int(tc7_force_direct), int(tc7_band_rows), int(tc6_band_rows), int(tc6_l2_hints), int(tc6_tap_prefetch))
    check(load().banet_set_tuning(C.byref(t)), "banet_set_tuning")


def require_device() -> None:
    """Raise unless the current CUDA device is a compute-capability-9.0 part (H100)."""
    check(load().banet_device_check(), "banet_device_check")
