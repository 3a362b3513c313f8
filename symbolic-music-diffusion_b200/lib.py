"""ctypes binding of libsmd.so (include/smd.h).  Fails loudly when the CUDA library is missing: there is no
CPU fallback anywhere in the product path."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libsmd.so")


class SmdError(RuntimeError):
    pass


class SmdConfig(C.Structure):
    _fields_ = [("arch", C.c_int), ("num_layers", C.c_int), ("num_heads", C.c_int),
                ("num_mlp_layers", C.c_int), ("mlp_dims", C.c_int), ("seq_len", C.c_int),
                ("channels", C.c_int), ("max_batch", C.c_int), ("cta_group", C.c_int),
                ("training", C.c_int), ("sampler_T", C.c_int), ("precision", C.c_int)]


class SmdCoverageConfig(C.Structure):
    _fields_ = [("neighbors", C.c_int), ("prd_clusters", C.c_int), ("prd_runs", C.c_int), ("ndb_bins", C.c_int),
                ("restarts", C.c_int), ("max_iter", C.c_int)]


_P = C.c_void_p
_SIGNATURES = {
    "smd_last_error": (C.c_char_p, []),
    "smd_version": (C.c_int, []),
    "smd_plan_create": (C.c_int, [C.POINTER(SmdConfig), C.POINTER(_P)]),
    "smd_plan_destroy": (None, [_P]),
    "smd_num_tensors": (C.c_int, [_P]),
    "smd_arena_floats": (C.c_longlong, [_P]),
    "smd_tensor_info": (C.c_int, [_P, C.c_int, C.c_char_p, C.c_int, C.POINTER(C.c_longlong),
                                  C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "smd_workspace_bytes": (C.c_size_t, [_P]),
    "smd_bind_workspace": (C.c_int, [_P, _P, C.c_size_t]),
    "smd_pack_weights": (C.c_int, [_P, _P, _P]),
    "smd_forward": (C.c_int, [_P, _P, _P, _P, C.c_int, C.c_int, _P, _P]),
    "smd_ddpm_loss": (C.c_int, [_P, _P, _P, _P, _P, C.c_int, _P, _P, _P]),
    "smd_ddpm_grads": (C.c_int, [_P, _P, _P, _P, _P, C.c_int, C.c_int, _P, _P, _P]),
    "smd_grads_tail_range": (C.c_int, [_P, C.POINTER(C.c_longlong), C.POINTER(C.c_longlong)]),
    "smd_wait_tail_grads": (C.c_int, [_P, _P]),
    "smd_pack_weights_after_adam": (C.c_int, [_P, _P, _P]),
    "smd_shadow_arena": (_P, [_P]),
    "smd_clip_adam": (C.c_int, [_P, _P, _P, _P, _P, _P, C.c_longlong, C.c_float, C.c_int, C.c_float, C.c_float,
                                C.c_float, C.c_float, C.c_float, _P, _P, _P]),
    "smd_ema_update": (C.c_int, [_P, _P, C.c_longlong, C.c_float, _P]),
    "smd_objective_setup": (C.c_int, [_P, C.POINTER(C.c_float), C.c_int, _P]),
    "smd_ddpm_draws": (C.c_int, [_P, C.POINTER(C.c_uint32), C.c_int, _P, _P, _P, _P]),
    "smd_ddpm_draws_sharded": (C.c_int, [_P, C.POINTER(C.c_uint32), C.c_int, C.c_int, C.c_int, C.c_int, _P, _P, _P, _P]),
    "smd_dsm_loss": (C.c_int, [_P, _P, _P, _P, _P, C.c_int, _P, _P, _P]),
    "smd_dsm_grads": (C.c_int, [_P, _P, _P, _P, _P, C.c_int, C.c_int, _P, _P, _P]),
    "smd_dsm_setup": (C.c_int, [_P, C.POINTER(C.c_float), C.c_int, _P]),
    "smd_dsm_draws": (C.c_int, [_P, C.POINTER(C.c_uint32), C.c_int, C.c_int, C.c_int, C.c_int, _P, _P, _P, _P]),
    "smd_ssm_loss": (C.c_int, [_P, _P, _P, _P, _P, _P, C.c_int, _P, _P, _P, _P]),
    "smd_ssm_grads": (C.c_int, [_P, _P, _P, _P, _P, _P, C.c_int, C.c_int, _P, _P, _P]),
    "smd_ssm_draws": (C.c_int, [_P, C.POINTER(C.c_uint32), C.c_int, C.c_int, C.c_int, C.c_int, _P, _P, _P, _P, _P]),
    "smd_langevin_step": (C.c_int, [_P, _P, _P, C.c_int, C.c_float, C.c_float, C.POINTER(C.c_uint32), _P, _P, _P,
                                    C.c_float, C.POINTER(C.c_uint32), _P, _P, _P, _P, _P]),
    "smd_sampler_setup": (C.c_int, [_P, C.POINTER(C.c_float), C.c_int, C.POINTER(C.c_uint32), _P]),
    "smd_ddpm_reverse_step": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "smd_ddpm_sample": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, _P, _P, _P, _P, C.c_int, _P]),
    "smd_threefry_normal": (C.c_int, [C.POINTER(C.c_uint32), _P, C.c_longlong, _P]),
    "smd_threefry_normal_slice": (C.c_int, [C.POINTER(C.c_uint32), _P, C.c_longlong, C.c_longlong, C.c_longlong, _P]),
    "smd_sampler_set_shard": (C.c_int, [_P, C.c_longlong, C.c_longlong]),
    "smd_threefry_uniform": (C.c_int, [C.POINTER(C.c_uint32), _P, C.c_longlong, C.c_float, C.c_float, _P]),
    "smd_threefry_uniform_slice": (C.c_int, [C.POINTER(C.c_uint32), _P, C.c_longlong, C.c_longlong, C.c_longlong,
                                             C.c_float, C.c_float, _P]),
    "smd_threefry_split": (C.c_int, [C.POINTER(C.c_uint32), C.c_int, C.POINTER(C.c_uint32)]),
    "smd_ddim_setup": (C.c_int, [_P, C.POINTER(C.c_float), C.c_int, C.POINTER(C.c_int), C.c_int, C.c_float,
                                 C.POINTER(C.c_uint32), _P]),
    "smd_ddim_sample": (C.c_int, [_P, _P, _P, C.c_int, _P, _P, _P, _P, C.c_int, _P]),
    "smd_ddim_tables": (C.c_int, [C.POINTER(C.c_float), C.c_int, C.POINTER(C.c_int), C.c_int, C.c_float,
                                  C.POINTER(C.c_uint32), C.POINTER(C.c_float), C.POINTER(C.c_uint32),
                                  C.POINTER(C.c_int)]),
    "smd_ddim_encode_setup": (C.c_int, [_P, C.POINTER(C.c_float), C.c_int, C.POINTER(C.c_int), C.c_int, _P]),
    "smd_ddim_encode": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, _P]),
    "smd_ddim_encode_tables": (C.c_int, [C.POINTER(C.c_float), C.c_int, C.POINTER(C.c_int), C.c_int,
                                         C.POINTER(C.c_float)]),
    "smd_dpm_setup": (C.c_int, [_P, C.POINTER(C.c_float), C.c_int, C.POINTER(C.c_int), C.c_int, C.c_int,
                                C.POINTER(C.c_uint32), _P]),
    "smd_dpm_sample": (C.c_int, [_P, _P, _P, C.c_int, _P, _P, _P, _P, _P, C.c_int, _P]),
    "smd_dpm_tables": (C.c_int, [C.POINTER(C.c_float), C.c_int, C.POINTER(C.c_int), C.c_int, C.c_int,
                                 C.POINTER(C.c_uint32), C.POINTER(C.c_float), C.POINTER(C.c_uint32),
                                 C.POINTER(C.c_int)]),
    "smd_langevin_setup": (C.c_int, [_P, C.POINTER(C.c_float), C.c_int, C.c_int, C.c_float, C.c_int,
                                     C.POINTER(C.c_uint32), _P]),
    "smd_langevin_sample": (C.c_int, [_P, _P, _P, C.c_int, _P, _P, C.c_int, _P, _P, C.c_int, _P]),
    "smd_langevin_tables": (C.c_int, [C.POINTER(C.c_float), C.c_int, C.c_int, C.c_float, C.c_int, C.c_int,
                                      C.POINTER(C.c_float), C.POINTER(C.c_int)]),
    "smd_gemm_bf16": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                _P, _P, C.c_int, _P, _P, _P, _P, _P, _P]),
    "smd_gemm_bf16_epi": (C.c_int, [_P, _P, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, _P, C.c_int, _P, _P, _P,
                                    _P, _P, _P, _P, _P]),
    "smd_debug_forward_save": (C.c_int, [_P, _P, _P, _P, C.c_int, _P, _P]),
    "smd_debug_buffer": (C.c_int, [_P, C.c_char_p, C.POINTER(_P), C.POINTER(C.c_size_t)]),
    "smd_launch_count": (C.c_longlong, []),
    "smd_mdn_plan_create": (C.c_int, [C.POINTER(SmdConfig), C.c_int, C.POINTER(_P)]),
    "smd_mdn_forward": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, _P, _P, _P, _P]),
    "smd_mdn_nll": (C.c_int, [_P, _P, _P, _P, C.c_int, C.c_int, C.c_int, _P, _P]),
    "smd_mdn_loss": (C.c_int, [_P, _P, _P, C.c_int, _P, _P]),
    "smd_mdn_grads": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, _P, _P, _P]),
    "smd_mdn_mixture_sample": (C.c_int, [_P, _P, _P, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_uint32), C.c_longlong,
                                         C.c_longlong, _P, _P, _P]),
    "smd_mdn_sample": (C.c_int, [_P, _P, C.POINTER(C.c_uint32), C.c_int, C.c_longlong, C.c_longlong, _P, _P, _P, _P]),
    "smd_latent_stats_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int]),
    "smd_latent_stats": (C.c_int, [_P, C.c_int, _P, C.c_int, C.c_int, C.c_float, C.c_int, C.c_float, C.c_float, _P,
                                   C.c_size_t, _P, _P, _P]),
    "smd_latent_coverage_workspace_bytes": (C.c_size_t, [C.c_int, C.c_int, C.c_int, C.POINTER(SmdCoverageConfig)]),
    "smd_latent_coverage": (C.c_int, [_P, C.c_int, _P, C.c_int, C.c_int, C.POINTER(SmdCoverageConfig), _P, _P,
                                      C.c_size_t, _P, _P, _P, _P, _P, _P]),
}

EXPORTED_SYMBOLS = tuple(_SIGNATURES)
_lib = None


def load_library(build_if_missing: bool = False) -> C.CDLL:
    """Load libsmd.so.  Raises SmdError (never falls back) if it is absent or lacks a symbol."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        if build_if_missing:
            from . import build as _build
            _build.build()
        else:
            raise SmdError(f"{LIB_PATH} not found: run `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(the CUDA library is mandatory; there is no CPU fallback)")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in _SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError as e:  # pragma: no cover
            raise SmdError(f"libsmd.so does not export {name}") from e
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc: int) -> None:
    if rc == 0:
        return
    msg = load_library().smd_last_error().decode("utf-8", "replace")
    if rc == -1:
        raise ValueError(msg)
    raise SmdError(f"libsmd error {rc}: {msg}")
