"""ctypes binding of include/sgmse_b200.h (the C-ABI drop-in boundary).

There is deliberately no fallback: if the shared library is missing it is built in-tree with nvcc
(``sgmse_b200.build``); if that fails, importing raises.  No torch type crosses this boundary -
callers pass ``tensor.data_ptr()`` and ``torch.cuda.current_stream().cuda_stream``.
"""
from __future__ import annotations

import ctypes as C
import os

from . import build as _build


class Config(C.Structure):
    _fields_ = [
        ("backbone", C.c_int), ("nf", C.c_int), ("num_levels", C.c_int), ("ch_mult", C.c_int * 8),
        ("num_res_blocks", C.c_int), ("num_attn_resolutions", C.c_int), ("attn_resolutions", C.c_int * 8),
        ("image_size", C.c_int), ("progressive_output_skip", C.c_int), ("progressive_input_skip", C.c_int),
        ("scale_by_sigma", C.c_int),
        ("theta", C.c_float), ("sigma_min", C.c_float), ("sigma_max", C.c_float), ("t_eps", C.c_float),
        ("n_fft", C.c_int), ("hop_length", C.c_int), ("sqrt_window", C.c_int),
        ("spec_factor", C.c_float), ("spec_abs_exponent", C.c_float), ("sample_rate", C.c_int),
        ("mode", C.c_int), ("max_batch", C.c_int), ("use_graphs", C.c_int),
        ("sde_kind", C.c_int), ("sb_k", C.c_float), ("sb_c", C.c_float), ("sb_eps", C.c_float),
        ("loss_type", C.c_int), ("network_scaling", C.c_int), ("c_in", C.c_int), ("c_out", C.c_int), ("c_skip", C.c_int),
        ("sigma_data", C.c_float), ("transform_type", C.c_int), ("not_centered", C.c_int),
    ]


class Sampler(C.Structure):
    _fields_ = [
        ("N", C.c_int), ("predictor", C.c_int), ("corrector", C.c_int), ("corrector_steps", C.c_int),
        ("snr", C.c_float), ("denoise", C.c_int), ("probability_flow", C.c_int),
        ("seed", C.c_ulonglong), ("utt_offset", C.c_int), ("pad_mode", C.c_int),
        ("kind", C.c_int), ("sb_eps", C.c_float), ("sb_n_steps", C.c_int),
    ]


class Ode(C.Structure):
    _fields_ = [("rtol", C.c_double), ("atol", C.c_double), ("eps", C.c_double), ("max_attempts", C.c_int),
                ("seed", C.c_ulonglong), ("utt_offset", C.c_int)]


# right-hand side of sgmse_b200_rk45_host: rhs(t, y, dydt, n, user)
ODE_RHS = C.CFUNCTYPE(None, C.c_double, C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_longlong, C.c_void_p)
# right-hand side of sgmse_b200_rk45_host_groups: rhs(count, systems, t, y, dydt, n, user)
ODE_RHS_GROUPS = C.CFUNCTYPE(None, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_double), C.POINTER(C.POINTER(C.c_double)),
                             C.POINTER(C.POINTER(C.c_double)), C.POINTER(C.c_longlong), C.c_void_p)


# every symbol include/sgmse_b200.h declares: name -> (restype, argtypes)
_P = C.c_void_p
SYMBOLS = {
    "sgmse_b200_last_error": (C.c_char_p, []),
    "sgmse_b200_version": (C.c_char_p, []),
    "sgmse_b200_create": (C.c_int, [C.POINTER(Config), C.POINTER(_P)]),
    "sgmse_b200_destroy": (None, [_P]),
    "sgmse_b200_manifest_count": (C.c_int, [_P]),
    "sgmse_b200_manifest_entry": (C.c_int, [_P, C.c_int, C.c_char_p, C.c_int, C.POINTER(C.c_longlong)]),
    "sgmse_b200_weights_numel": (C.c_longlong, [_P]),
    "sgmse_b200_load_weights": (C.c_int, [_P, _P, C.c_longlong]),
    "sgmse_b200_load_weights_device": (C.c_int, [_P, _P, C.c_longlong, _P]),
    "sgmse_b200_dnn_forward": (C.c_int, [_P, _P, _P, _P, C.c_int, C.c_int, C.c_int, _P]),
    "sgmse_b200_score": (C.c_int, [_P, _P, _P, _P, _P, C.c_int, C.c_int, C.c_int, _P]),
    "sgmse_b200_pc_sample": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, C.POINTER(Sampler), _P, _P,
                                       C.POINTER(C.c_int), _P]),
    "sgmse_b200_noise_draws": (C.c_int, [C.POINTER(Sampler)]),
    "sgmse_b200_model_forward": (C.c_int, [_P, _P, _P, _P, _P, C.c_int, C.c_int, C.c_int, _P]),
    "sgmse_b200_sampler_schedule": (C.c_int, [_P, C.POINTER(Sampler), _P, _P, _P, C.c_int, C.POINTER(C.c_int)]),
    "sgmse_b200_ode_sample": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, C.POINTER(Ode), _P, _P, C.POINTER(C.c_int),
                                        C.POINTER(C.c_int * 4), _P]),
    "sgmse_b200_rk45_host": (C.c_int, [ODE_RHS, _P, C.c_double, C.c_double, _P, C.c_longlong, C.c_double, C.c_double,
                                       C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int * 4)]),
    "sgmse_b200_ode_sample_groups": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(Ode), _P, _P, _P, _P,
                                               _P, _P]),
    "sgmse_b200_rk45_host_groups": (C.c_int, [ODE_RHS_GROUPS, _P, C.c_int, C.c_int, _P, C.c_double, C.c_double, _P,
                                              C.c_double, C.c_double, C.c_int, _P, _P, _P]),
    "sgmse_b200_padded_frames": (C.c_int, [_P, C.c_int]),
    "sgmse_b200_analysis": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, _P, _P, _P]),
    "sgmse_b200_synthesis": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, C.c_int, _P, _P]),
    "sgmse_b200_enhance": (C.c_int, [_P, _P, C.c_int, C.c_int, C.POINTER(Sampler), _P, _P, C.c_int, _P]),
    "sgmse_b200_enhance_ode": (C.c_int, [_P, _P, C.c_int, C.c_int, C.POINTER(Ode), C.c_int, _P, _P, C.c_int, _P, _P]),
    "sgmse_b200_get_tap": (C.c_int, [_P, C.c_char_p, _P, C.c_longlong, C.POINTER(C.c_int * 4)]),
    "sgmse_b200_workspace_bytes": (C.c_longlong, [_P, C.c_int, C.c_int, C.c_int]),
    "sgmse_b200_workspace_plan": (C.c_longlong, [_P, C.c_int, C.c_int, C.c_int, _P, C.c_longlong,
                                                 C.POINTER(C.c_longlong), C.POINTER(C.c_int)]),
    "sgmse_b200_set_option": (C.c_int, [_P, C.c_char_p, C.c_longlong]),
    "sgmse_b200_get_counter": (C.c_longlong, [_P, C.c_char_p]),
}

_lib = None


def load() -> C.CDLL:
    """Load (building if necessary) libsgmse_b200.so.  Raises if the native library cannot be had."""
    global _lib
    if _lib is not None:
        return _lib
    pdl = os.environ.get("SGMSE_B200_PDL", "0") not in ("", "0")     # A/B twin with programmatic dependent launch compiled in
    path = _build.lib_path(pdl)
    if not os.path.exists(path) or os.environ.get("SGMSE_B200_REBUILD"):
        path = _build.build(pdl=pdl)
    lib = C.CDLL(path)
    for name, (res, args) in SYMBOLS.items():
        fn = getattr(lib, name)          # AttributeError if the library does not export it
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(code: int):
    if code != 0:
        msg = load().sgmse_b200_last_error()
        raise RuntimeError(f"sgmse_b200: {msg.decode() if msg else 'error'} (code {code})")
