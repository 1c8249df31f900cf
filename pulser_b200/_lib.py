"""ctypes binding of libpulser_b200.so (include/pulser_b200.h).

Loading never falls back to anything else: if the shared library is missing
the import raises, and if there is no CUDA device ``Plan`` creation raises
(`PB200_ERR_CUDA`).  There is no CPU implementation of the hot path.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libpulser_b200.so")

PB200_MAX_DRIVES = 3


class DriveDesc(C.Structure):
    _fields_ = [
        ("state_to", C.c_int32),
        ("state_from", C.c_int32),
        ("uniform", C.c_int32),
        ("reserved", C.c_int32),
    ]


class PlanDesc(C.Structure):
    _fields_ = [
        ("n_qudits", C.c_int32),
        ("dim", C.c_int32),
        ("n_times", C.c_int32),
        ("interp_order", C.c_int32),
        ("n_drives", C.c_int32),
        ("rydberg_state", C.c_int32),
        ("n_traj", C.c_int32),
        ("device", C.c_int32),
        ("sampling_times", C.POINTER(C.c_double)),
        ("drives", DriveDesc * PB200_MAX_DRIVES),
    ]


class RunOpts(C.Structure):
    _fields_ = [
        ("max_step_samples", C.c_int32),
        ("refine_window", C.c_int32),
        ("cheb_tol", C.c_double),
        ("rough_tol", C.c_double),
        ("magnus_order", C.c_int32),
        ("check_every", C.c_int32),
        ("tol", C.c_double),
        ("extrapolate", C.c_int32),
        ("integrator", C.c_int32),
    ]


class RunStats(C.Structure):
    _fields_ = [
        ("n_steps", C.c_int64),
        ("n_exponentials", C.c_int64),
        ("n_applies", C.c_int64),
        ("n_launches", C.c_int64),
        ("gpu_ms", C.c_double),
        ("max_rho", C.c_double),
        ("n_checks", C.c_int64),
        ("err_estimate", C.c_double),
        ("mean_step_samples", C.c_double),
        ("integrator", C.c_int64),
        ("n_rejected", C.c_int64),
    ]


class OpTermsDesc(C.Structure):
    """``pb200_op_terms``: an operator as monomial terms (packed by ``pulser_b200.opterms.OpTerms.c_desc``)."""

    _fields_ = [
        ("n_terms", C.c_int32),
        ("coeff", C.POINTER(C.c_double)),
        ("site_start", C.POINTER(C.c_int32)),
        ("site", C.POINTER(C.c_int32)),
        ("shift", C.POINTER(C.c_int32)),
        ("weight", C.POINTER(C.c_double)),
    ]


class LibraryMissing(ImportError):
    pass


def _load() -> C.CDLL:
    if not os.path.exists(LIB_PATH):
        raise LibraryMissing(
            f"{LIB_PATH} not found: build it with "
            "`python -m pulser_b200.build` (nvcc, sm_90a). "
            "pulser_b200 has no CPU fallback."
        )
    lib = C.CDLL(LIB_PATH)
    dp = C.POINTER(C.c_double)
    vp = C.c_void_p
    sig = {
        "pb200_version": (C.c_int, []),
        "pb200_last_error": (C.c_char_p, []),
        "pb200_device_count": (C.c_int, []),
        "pb200_plan_create": (C.c_int, [C.POINTER(vp), C.POINTER(PlanDesc)]),
        "pb200_plan_destroy": (C.c_int, [vp]),
        "pb200_plan_set_stream": (C.c_int, [vp, vp]),
        "pb200_plan_set_interaction": (
            C.c_int, [vp, C.c_int32, C.c_int32, dp, C.POINTER(C.c_uint8), C.c_int32]),
        "pb200_plan_set_xy": (
            C.c_int, [vp, C.c_int32, C.c_int32, dp, C.POINTER(C.c_uint8), C.c_int32, C.c_int32, C.c_int32]),
        "pb200_plan_set_slm_mask": (C.c_int, [vp, C.POINTER(C.c_uint8), dp]),
        "pb200_plan_set_drive": (C.c_int, [vp, C.c_int32, C.c_int32, C.c_int32, dp, dp]),
        "pb200_plan_set_dissipator": (C.c_int, [vp, C.c_int32, dp]),
        "pb200_plan_set_collapse": (C.c_int, [vp, C.c_int32, dp, C.c_uint64]),
        "pb200_plan_jump_counts": (C.c_int, [vp, C.POINTER(C.c_int64)]),
        "pb200_state_set": (C.c_int, [vp, C.c_int32, C.c_int32, dp, C.c_int64, C.c_int32]),
        "pb200_state_get": (C.c_int, [vp, C.c_int32, C.c_int32, dp]),
        "pb200_state_probabilities": (C.c_int, [vp, C.c_int32, C.c_int32, dp]),
        "pb200_state_norm2": (C.c_int, [vp, C.c_int32, C.c_int32, dp]),
        "pb200_state_occupation": (C.c_int, [vp, C.c_int32, C.c_int32, C.c_int32, dp]),
        "pb200_state_correlation": (C.c_int, [vp, C.c_int32, C.c_int32, C.c_int32, dp]),
        "pb200_state_energy": (C.c_int, [vp, C.c_double, dp, dp]),
        "pb200_state_overlap": (C.c_int, [vp, C.c_int32, C.c_int32, dp, dp]),
        "pb200_state_expect": (C.c_int, [vp, C.c_int32, C.c_int32, C.POINTER(OpTermsDesc), dp]),
        "pb200_state_sample": (
            C.c_int, [vp, C.c_int32, C.c_int32, dp, C.c_int32, C.POINTER(C.c_int64)]),
        "pb200_state_copy": (C.c_int, [vp, C.c_int32, vp, C.c_int32]),
        "pb200_state_device_ptr": (C.c_int, [vp, C.POINTER(vp)]),
        "pb200_density_trace": (C.c_int, [vp, C.c_int32, C.c_int32, dp]),
        "pb200_density_occupation": (C.c_int, [vp, C.c_int32, C.c_int32, C.c_int32, dp]),
        "pb200_density_correlation": (C.c_int, [vp, C.c_int32, C.c_int32, C.c_int32, dp]),
        "pb200_density_expect": (C.c_int, [vp, C.c_int32, C.c_int32, C.POINTER(OpTermsDesc), dp]),
        "pb200_density_energy": (C.c_int, [vp, vp, C.c_double, C.c_int32, C.c_int32, dp, dp]),
        "pb200_density_overlap": (C.c_int, [vp, C.c_int32, C.c_int32, dp, dp]),
        "pb200_density_sample": (
            C.c_int, [vp, C.c_int32, C.c_int32, dp, C.c_int32, C.POINTER(C.c_int64)]),
        "pb200_propagate": (
            C.c_int, [vp, C.c_double, C.c_double, C.POINTER(RunOpts), C.POINTER(RunStats)]),
        "pb200_apply_h": (C.c_int, [vp, C.c_int32, C.c_double, dp, dp]),
        "pb200_coefficients_at": (
            C.c_int, [vp, C.c_int32, C.c_int32, C.c_int32, C.c_double, dp]),
        "pb200_bench_apply": (
            C.c_int, [vp, C.c_double, C.c_int32, dp, C.POINTER(C.c_int64)]),
        "pb200_plan_create_shard": (C.c_int, [C.POINTER(vp), C.POINTER(PlanDesc), C.c_int32, C.c_int32]),
        "pb200_shards_link": (C.c_int, [C.POINTER(vp), C.c_int32]),
        "pb200_shards_propagate": (
            C.c_int, [C.POINTER(vp), C.c_int32, C.c_double, C.c_double, C.POINTER(RunOpts), C.POINTER(RunStats)]),
        "pb200_shards_apply_h": (C.c_int, [C.POINTER(vp), C.c_int32, C.c_double, dp, dp]),
        "pb200_shards_energy": (C.c_int, [C.POINTER(vp), C.c_int32, C.c_double, dp, dp]),
        "pb200_shards_expect": (C.c_int, [C.POINTER(vp), C.c_int32, C.POINTER(OpTermsDesc), dp]),
        "pb200_host_interpolate": (
            C.c_int, [dp, dp, C.c_int32, C.c_int32, dp, C.c_int32, dp]),
        "pb200_host_moments": (
            C.c_int, [dp, dp, C.c_int32, C.c_int32, C.c_double, C.c_double, dp]),
        "pb200_host_chebyshev": (
            C.c_int, [C.c_double, C.c_double, dp, C.c_int32, C.POINTER(C.c_int32)]),
        "pb200_host_taylor_fit": (
            C.c_int, [dp, dp, C.c_int32, C.c_int32, C.c_double, C.c_double, C.c_int32, dp, dp]),
        "pb200_host_taylor_separable": (
            C.c_int, [dp, dp, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_int32), dp, dp, dp]),
        "pb200_host_taylor_shapes": (
            C.c_int, [dp, dp, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_int32), dp, dp, dp]),
        "pb200_host_taylor_order": (
            C.c_int, [C.c_double, dp, C.c_int32, C.c_double, C.POINTER(C.c_int32), dp]),
        "pb200_host_taylor_lowprec": (
            C.c_int, [C.c_double, dp, C.c_int32, C.c_int32, C.c_int32, C.c_double, C.POINTER(C.c_int32), dp]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is missing
        fn.restype = res
        fn.argtypes = args
    return lib


EXPORTED_SYMBOLS = [
    "pb200_version", "pb200_last_error", "pb200_device_count",
    "pb200_plan_create", "pb200_plan_destroy", "pb200_plan_set_stream",
    "pb200_plan_set_interaction", "pb200_plan_set_xy", "pb200_plan_set_slm_mask", "pb200_plan_set_drive", "pb200_plan_set_dissipator", "pb200_plan_set_collapse",
    "pb200_plan_jump_counts", "pb200_state_set",
    "pb200_state_get", "pb200_state_probabilities", "pb200_state_norm2",
    "pb200_state_occupation", "pb200_state_correlation", "pb200_state_energy", "pb200_state_overlap", "pb200_state_expect", "pb200_state_sample", "pb200_state_copy", "pb200_state_device_ptr", "pb200_propagate", "pb200_apply_h",
    "pb200_coefficients_at", "pb200_bench_apply", "pb200_host_interpolate",
    "pb200_host_moments", "pb200_host_chebyshev", "pb200_host_taylor_fit", "pb200_host_taylor_order", "pb200_host_taylor_lowprec",
    "pb200_host_taylor_separable",
    "pb200_host_taylor_shapes",
    "pb200_plan_create_shard", "pb200_shards_link", "pb200_shards_propagate", "pb200_shards_apply_h", "pb200_shards_energy",
    "pb200_shards_expect",
    "pb200_density_trace", "pb200_density_occupation", "pb200_density_correlation", "pb200_density_expect",
    "pb200_density_energy", "pb200_density_overlap", "pb200_density_sample",
]

lib = _load()


class PB200Error(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"pulser_b200 error {code}: {msg}")
        self.code = code


def check(code: int) -> None:
    if code != 0:
        raise PB200Error(code, lib.pb200_last_error().decode("utf-8", "replace"))
