"""ctypes binding of the C ABI declared in include/b200conv.h.

The product path has no CPU fall-back: if libb200conv.so is missing or cannot be loaded this
module raises, it never substitutes another implementation.  (`load(path)` exists so that the
test-suite can bind the same ABI of the CPU *emulation* build under tests/emu — test
infrastructure only, never used by this package on its own.)
"""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libb200conv.so")


class Config(C.Structure):
    _fields_ = [
        ("n_channels", C.c_int),
        ("device", C.c_int),
        ("max_batch_blocks", C.c_int),
        ("shard_rank", C.c_int),
        ("shard_count", C.c_int),
        ("cmac_variant", C.c_int),
    ]


class ChainConfig(C.Structure):
    _fields_ = [("srate", C.c_double), ("lowcut_hz", C.c_float), ("lowcut_slope", C.c_int), ("highcut_hz", C.c_float),
                ("highcut_slope", C.c_int), ("predelay", C.c_int), ("width", C.c_float), ("drygain", C.c_float),
                ("wetgain", C.c_float), ("true_stereo", C.c_int)]


class ChainEvent(C.Structure):
    _fields_ = [("offset", C.c_size_t), ("cfg", ChainConfig)]


class IrShapeParams(C.Structure):
    _fields_ = [("autogain", C.c_int), ("reverse", C.c_int), ("trim_left", C.c_float), ("trim_right", C.c_float),
                ("gain", C.c_float), ("decay_lut", C.c_void_p), ("srate", C.c_double), ("clip", C.c_int),
                ("attack", C.c_float), ("decay", C.c_float)]


class EqBand(C.Structure):
    """b200conv_eq_band: one SVF band (mode 0..9 = LP BP HP LS HS PK BS HP6 LP6 Off)."""
    _fields_ = [("mode", C.c_int), ("freq", C.c_float), ("q", C.c_float), ("gain", C.c_float)]


class IrRecalcParams(C.Structure):
    _fields_ = [("ir_srate", C.c_double), ("srate", C.c_double), ("stretch", C.c_float), ("autogain", C.c_int),
                ("reverse", C.c_int), ("trim_left", C.c_float), ("trim_right", C.c_float), ("gain", C.c_float),
                ("n_param_eq", C.c_int), ("param_eq", C.POINTER(EqBand)), ("n_decay_eq", C.c_int),
                ("decay_eq", C.POINTER(EqBand)), ("decay_rate", C.c_float), ("clip", C.c_int), ("attack", C.c_float),
                ("decay", C.c_float)]


class StageInfo(C.Structure):
    _fields_ = [
        ("block", C.c_size_t),
        ("partitions", C.c_size_t),
        ("tap_offset", C.c_size_t),
        ("p_begin", C.c_size_t),
        ("p_end", C.c_size_t),
    ]


REDUCE_FN = C.CFUNCTYPE(C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p)
BARRIER_FN = C.CFUNCTYPE(C.c_int, C.c_void_p)

# every symbol include/b200conv.h declares: (name, restype, argtypes)
_PP = C.POINTER(C.c_void_p)
SYMBOLS = [
    ("b200conv_create", C.c_void_p, [C.POINTER(Config)]),
    ("b200conv_destroy", None, [C.c_void_p]),
    ("b200conv_last_error", C.c_char_p, [C.c_void_p]),
    ("b200conv_init_uniform", C.c_int, [C.c_void_p, C.c_size_t, _PP, C.POINTER(C.c_size_t)]),
    ("b200conv_init_twostage", C.c_int, [C.c_void_p, C.c_size_t, C.c_size_t, _PP, C.POINTER(C.c_size_t)]),
    ("b200conv_init_stages", C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t), _PP, C.POINTER(C.c_size_t)]),
    ("b200conv_process", C.c_int, [C.c_void_p, _PP, _PP, C.c_size_t]),
    ("b200conv_process_device", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int]),
    ("b200conv_clear", C.c_int, [C.c_void_p]),
    ("b200conv_reset", C.c_int, [C.c_void_p]),
    ("b200conv_set_latency", C.c_int, [C.c_void_p, C.c_size_t]),
    ("b200conv_latency", C.c_size_t, [C.c_void_p]),
    ("b200conv_latency_waits", C.c_ulonglong, [C.c_void_p]),
    ("b200conv_group_create", C.c_void_p, [C.POINTER(C.c_void_p), C.c_int]),
    ("b200conv_group_destroy", None, [C.c_void_p]),
    ("b200conv_group_last_error", C.c_char_p, [C.c_void_p]),
    ("b200conv_group_process", C.c_int, [C.c_void_p, _PP, _PP, C.c_size_t]),
    ("b200conv_group_launch_count", C.c_ulonglong, [C.c_void_p]),
    ("b200conv_chain_group_process", C.c_int, [C.c_void_p, _PP, _PP, _PP, _PP, C.c_size_t]),
    ("b200conv_group_set_member", C.c_int, [C.c_void_p, C.c_int, C.c_void_p]),
    ("b200conv_group_set_latency", C.c_int, [C.c_void_p, C.c_size_t]),
    ("b200conv_group_latency", C.c_size_t, [C.c_void_p]),
    ("b200conv_group_process_device", C.c_int, [C.c_void_p, _PP, C.POINTER(C.c_size_t), _PP, C.POINTER(C.c_size_t),
                                                 C.c_size_t, C.c_int]),
    ("b200conv_chain_group_process_device", C.c_int, [C.c_void_p, _PP, C.POINTER(C.c_size_t), _PP, _PP, _PP,
                                                       C.POINTER(C.c_size_t), C.c_size_t, C.c_int]),
    ("b200conv_group_stream", C.c_void_p, [C.c_void_p]),
    ("b200conv_num_stages", C.c_int, [C.c_void_p]),
    ("b200conv_stage", C.c_int, [C.c_void_p, C.c_int, C.POINTER(StageInfo)]),
    ("b200conv_ir_len", C.c_size_t, [C.c_void_p, C.c_int]),
    ("b200conv_launch_count", C.c_ulonglong, [C.c_void_p]),
    ("b200conv_last_sweep_variant", C.c_int, [C.c_void_p]),
    ("b200conv_set_timing", C.c_int, [C.c_void_p, C.c_int]),
    ("b200conv_last_timing", C.c_int, [C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_int)]),
    ("b200conv_stream", C.c_void_p, [C.c_void_p]),
    ("b200conv_set_option", C.c_int, [C.c_void_p, C.c_char_p, C.c_int]),
    ("b200conv_set_reduce", C.c_int, [C.c_void_p, REDUCE_FN, C.c_void_p]),
    ("b200conv_prime", C.c_int, [C.c_void_p, _PP, C.c_size_t]),
    ("b200conv_process_xfade", C.c_int, [C.c_void_p, C.c_void_p, _PP, _PP, C.c_size_t, C.c_float, C.c_float]),
    ("b200conv_set_routing", C.c_int, [C.c_void_p, C.c_int, C.POINTER(C.c_int), C.c_int, C.POINTER(C.c_float)]),
    ("b200conv_p2p_blob_size", C.c_size_t, [C.c_void_p]),
    ("b200conv_p2p_export", C.c_int, [C.c_void_p, C.c_void_p, C.c_int]),
    ("b200conv_p2p_import", C.c_int, [C.c_void_p, C.c_void_p]),
    ("b200conv_p2p_detach", C.c_int, [C.c_void_p]),
    ("b200conv_p2p_set_input_broadcast", C.c_int, [C.c_void_p, C.c_int]),
    ("b200conv_p2p_set_host_barrier", C.c_int, [C.c_void_p, BARRIER_FN, C.c_void_p]),
    ("b200conv_ir_decay_eq", C.c_int, [C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_double]),
    ("b200conv_process_sliced", C.c_int, [C.c_void_p, _PP, _PP, C.c_size_t, C.c_int, C.c_int]),
    ("b200conv_process_device_sliced", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_size_t,
                                                  C.c_int, C.c_int, C.c_int]),
    ("b200conv_register_host", C.c_int, [C.c_void_p, C.c_size_t]),
    ("b200conv_unregister_host", C.c_int, [C.c_void_p]),
    ("b200conv_chain_configure", C.c_int, [C.c_void_p, C.c_void_p]),
    ("b200conv_chain_process", C.c_int, [C.c_void_p, _PP, C.c_void_p, C.c_void_p, _PP, C.c_size_t]),
    ("b200conv_chain_process_device", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p,
                                                 C.c_size_t, C.c_size_t, C.c_int]),
    ("b200conv_chain_process_device_events", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p,
                                                        C.c_void_p, C.c_size_t, C.c_size_t, C.c_void_p, C.c_size_t,
                                                        C.c_int]),
    ("b200conv_chain_update", C.c_int, [C.c_void_p, C.c_void_p]),
    ("b200conv_chain_swap", C.c_int, [C.c_void_p, C.c_void_p, C.c_size_t]),
    ("b200conv_chain_swap_state", C.c_int, [C.c_void_p]),
    ("b200conv_ir_shape", C.c_int, [C.c_int, _PP, C.c_int, C.c_size_t, C.c_void_p, _PP, C.c_void_p]),
    ("b200conv_init_uniform_shaped", C.c_int, [C.c_void_p, C.c_size_t, _PP, C.c_size_t, C.c_void_p]),
    ("b200conv_init_twostage_shaped", C.c_int, [C.c_void_p, C.c_size_t, C.c_size_t, _PP, C.c_size_t, C.c_void_p]),
    ("b200conv_ir_recalc_len", C.c_size_t, [C.c_size_t, C.c_void_p]),
    ("b200conv_ir_recalc", C.c_int, [C.c_int, _PP, C.c_int, C.c_size_t, C.c_void_p, _PP, C.c_size_t, C.c_void_p]),
    ("b200conv_init_uniform_recalc", C.c_int, [C.c_void_p, C.c_size_t, _PP, C.c_size_t, C.c_void_p]),
    ("b200conv_init_twostage_recalc", C.c_int, [C.c_void_p, C.c_size_t, C.c_size_t, _PP, C.c_size_t, C.c_void_p]),
    ("b200conv_alloc_host", C.c_void_p, [C.c_size_t]),
    ("b200conv_free_host", None, [C.c_void_p]),
    ("b200conv_version", C.c_char_p, []),
]


def load(path: str | None = None) -> C.CDLL:
    path = path or LIB_PATH
    if not os.path.exists(path):
        raise RuntimeError(
            f"{path} not found: build the CUDA extension first (python -m reevr_b200.build); "
            "there is no CPU fall-back")
    lib = C.CDLL(path)
    for name, res, args in SYMBOLS:
        fn = getattr(lib, name)          # AttributeError if the ABI is incomplete
        fn.restype = res
        fn.argtypes = args
    return lib


_default = None


def default() -> C.CDLL:
    global _default
    if _default is None:
        _default = load()
    return _default
