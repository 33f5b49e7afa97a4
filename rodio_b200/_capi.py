"""ctypes binding of include/rodio_b200.h.

The library is built in-tree by `rodio_b200.build` (nvcc, sm_90a).  Importing this module never
falls back to anything else: a missing .so is a hard ImportError, and a missing GPU makes
`rb_context_create` fail with RB_ERR_CUDA.
"""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
# RODIO_B200_LIB: an instrumented build of the same library (tools/hot_timing.py); never a different implementation
LIB_PATH = os.environ.get("RODIO_B200_LIB") or os.path.join(HERE, "librodio_b200.so")

RB_OK = 0
RB_ERR_INVALID_ARGUMENT = 1
RB_ERR_CUDA = 2
RB_ERR_OUT_OF_MEMORY = 3
RB_ERR_UNSUPPORTED = 4
RB_ERR_UNALIGNED_FRAMES = 5
RB_ERR_RATIO_OVERFLOW = 6
RB_ERR_NOT_SUPPORTED_SEEK = 7
RB_ERR_BUFFER_TOO_SMALL = 8
RB_ERR_STATE = 9

RB_FMT_F32, RB_FMT_I16, RB_FMT_U16, RB_FMT_I8, RB_FMT_U8, RB_FMT_I32, RB_FMT_I24_IN_I32 = range(7)

(RB_FX_AMPLIFY, RB_FX_SPEED, RB_FX_LOW_PASS, RB_FX_HIGH_PASS, RB_FX_REVERB, RB_FX_AGC, RB_FX_LIMIT,
 RB_FX_SPATIAL, RB_FX_CHANNEL_VOLUME, RB_FX_UNIFORM, RB_FX_DELAY, RB_FX_DISTORTION, RB_FX_LINEAR_RAMP,
 RB_FX_TAKE_DURATION, RB_FX_SIGNAL, RB_FX_MIX, RB_FX_APPEND, RB_FX_PAUSE) = range(1, 19)
RB_MIX_START_CONSUMED = 0xFFFFFFFFFFFFFFFF
RB_SIGNAL_SINE, RB_SIGNAL_TRIANGLE, RB_SIGNAL_SQUARE, RB_SIGNAL_SAWTOOTH = range(4)

RB_MIX_EXACT_ORDER = 1 << 0
RB_NO_FUSION = 1 << 1
RB_BIQUAD_TIME_PARALLEL = 1 << 2
RB_KEEP_STREAM_OUTPUTS = 1 << 3
RB_FUSED_LANES = 1 << 4
RB_FUSED_DUO = 1 << 5
RB_SESSION_HELD = (1 << 64) - 1
RB_SESSION_RESTARTS = 1


class rb_effect(C.Structure):
    _fields_ = [("kind", C.c_uint32), ("u32", C.c_uint32 * 3), ("f32", C.c_float * 12), ("ns", C.c_uint64 * 2)]


class rb_stream_desc(C.Structure):
    _fields_ = [
        ("sample_rate", C.c_uint32),
        ("channels", C.c_uint16),
        ("format", C.c_uint16),
        ("n_samples", C.c_uint64),
        ("span_len", C.c_uint32),
        ("n_effects", C.c_uint32),
        ("effects", C.POINTER(rb_effect)),
        ("mix_start", C.c_uint64),
    ]


class rb_span_mark(C.Structure):
    _fields_ = [("at", C.c_uint64), ("span_len", C.c_uint32), ("pad_", C.c_uint32)]


assert C.sizeof(rb_effect) == 80
assert C.sizeof(rb_span_mark) == 16

# every symbol include/rodio_b200.h declares: (restype, argtypes)
_u64p = C.POINTER(C.c_uint64)
_vpp = C.POINTER(C.c_void_p)
SYMBOLS = {
    "rb_status_string": (C.c_char_p, [C.c_int32]),
    "rb_last_error": (C.c_char_p, []),
    "rb_abi_version": (C.c_uint32, []),
    "rb_context_create": (C.c_int32, [C.c_int, _vpp]),
    "rb_context_destroy": (C.c_int32, [C.c_void_p]),
    "rb_context_sync": (C.c_int32, [C.c_void_p]),
    "rb_context_stream": (C.c_int32, [C.c_void_p, _vpp]),
    "rb_context_sm_count": (C.c_int32, [C.c_void_p, C.POINTER(C.c_int)]),
    "rb_batch_create": (C.c_int32, [C.c_void_p, C.c_uint16, C.c_uint32, C.POINTER(rb_stream_desc), C.c_size_t,
                                    C.c_uint32, _vpp]),
    "rb_batch_destroy": (C.c_int32, [C.c_void_p]),
    "rb_stream_plan": (C.c_int32, [C.POINTER(rb_stream_desc), C.c_uint16, C.c_uint32, _u64p, C.POINTER(C.c_uint16),
                                   C.POINTER(C.c_uint32), _u64p]),
    "rb_streams_plan": (C.c_int32, [C.POINTER(rb_stream_desc), C.c_size_t, C.c_size_t, C.c_uint16, C.c_uint32, _u64p,
                                    C.POINTER(C.c_uint16), C.POINTER(C.c_uint32), _u64p]),
    "rb_batch_upload": (C.c_int32, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_uint64]),
    "rb_batch_upload_packed": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_uint64]),
    "rb_batch_input_device_ptr": (C.c_int32, [C.c_void_p, C.c_size_t, _vpp, _u64p]),
    "rb_batch_stream_out_len": (C.c_int32, [C.c_void_p, C.c_size_t, _u64p]),
    "rb_batch_mix_len": (C.c_int32, [C.c_void_p, _u64p]),
    "rb_batch_launches_per_render": (C.c_int32, [C.c_void_p, C.POINTER(C.c_uint32)]),
    "rb_batch_kernel_family": (C.c_int32, [C.c_void_p, C.POINTER(C.c_int)]),
    "rb_batch_mix_group": (C.c_int32, [C.c_void_p, C.POINTER(C.c_uint32)]),
    "rb_batch_set_master": (C.c_int32, [C.c_void_p, C.POINTER(rb_effect), C.c_uint32]),
    "rb_session_set_master": (C.c_int32, [C.c_void_p, C.POINTER(rb_effect), C.c_uint32]),
    "rb_wav_parse": (C.c_int32, [C.c_void_p, C.c_uint64, C.c_void_p]),
    "rb_wav_unpack24": (None, [C.c_void_p, C.c_uint64, C.c_void_p]),
    "rb_comm_unique_id": (C.c_int32, [C.c_void_p]),
    "rb_comm_init_rank": (C.c_int32, [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.POINTER(C.c_void_p)]),
    "rb_comm_init_all": (C.c_int32, [C.POINTER(C.c_void_p), C.c_int, C.POINTER(C.c_void_p)]),
    "rb_comm_destroy": (C.c_int32, [C.c_void_p]),
    "rb_comm_transport": (C.c_int32, [C.c_void_p, C.c_char_p, C.c_uint64]),
    "rb_batch_render_mix_allreduce": (C.c_int32, [C.POINTER(C.c_void_p), C.c_int, C.c_void_p]),
    "rb_session_create": (C.c_int32, [C.c_void_p, C.c_uint16, C.c_uint32, C.c_void_p, C.c_size_t, C.c_uint32, C.c_uint32, C.POINTER(C.c_void_p)]),
    "rb_session_create_ex": (C.c_int32, [C.c_void_p, C.c_uint16, C.c_uint32, C.c_void_p, C.c_size_t, C.c_uint32, C.c_uint32, C.c_uint32,
                                         C.POINTER(C.c_void_p)]),
    "rb_session_source_runs": (C.c_int32, [C.c_void_p, C.c_size_t, C.POINTER(C.c_uint64)]),
    "rb_session_restart_launches": (C.c_int32, [C.c_void_p, C.POINTER(C.c_uint64)]),
    "rb_session_destroy": (C.c_int32, [C.c_void_p]),
    "rb_session_push": (C.c_int32, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_uint64, C.c_int]),
    "rb_session_push_packed": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "rb_session_push_silence": (C.c_int32, [C.c_void_p, C.c_size_t, C.c_uint64]),
    "rb_session_push_spans": (C.c_int32, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_uint64, C.POINTER(rb_span_mark), C.c_uint32, C.c_int]),
    "rb_session_push_packed_spans": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(rb_span_mark)]),
    "rb_session_start": (C.c_int32, [C.c_void_p, C.c_size_t]),
    "rb_session_follow": (C.c_int32, [C.c_void_p, C.c_size_t, C.c_size_t]),
    "rb_session_skip": (C.c_int32, [C.c_void_p, C.c_size_t]),
    "rb_session_set_amplify": (C.c_int32, [C.c_void_p, C.c_size_t, C.c_float]),
    "rb_session_set_volume": (C.c_int32, [C.c_void_p, C.c_size_t, C.c_float]),
    "rb_session_available": (C.c_int32, [C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_int)]),
    "rb_session_render": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64), C.POINTER(C.c_int)]),
    "rb_session_get_state": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_uint64, C.POINTER(C.c_uint64)]),
    "rb_session_set_state": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_uint64]),
    "rb_batch_algorithmic_bytes": (C.c_int32, [C.c_void_p, _u64p]),
    "rb_batch_render_mix_device": (C.c_int32, [C.c_void_p]),
    "rb_batch_mix_device_ptr": (C.c_int32, [C.c_void_p, _vpp]),
    "rb_batch_render_mix": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_uint64, _u64p]),
    "rb_batch_read_stream": (C.c_int32, [C.c_void_p, C.c_size_t, C.c_void_p, C.c_uint64, _u64p]),
    "rb_batch_read_mix": (C.c_int32, [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint64, _u64p]),
    "rb_sample_rate_out_len": (C.c_int32, [C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint16, _u64p]),
    "rb_convert_sample_rate": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint16,
                                           C.c_void_p, C.c_uint64, _u64p]),
    "rb_channels_out_len": (C.c_int32, [C.c_uint64, C.c_uint16, C.c_uint16, _u64p]),
    "rb_convert_channels": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint16, C.c_uint16, C.c_void_p,
                                        C.c_uint64, _u64p]),
    "rb_convert_samples": (C.c_int32, [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_uint64]),
    "rb_speed_sample_rate": (C.c_uint32, [C.c_uint32, C.c_float]),
    "rb_delay_samples": (C.c_uint64, [C.c_uint64, C.c_uint32, C.c_uint16]),
    "rb_db_to_linear": (C.c_float, [C.c_float]),
    "rb_linear_to_db": (C.c_float, [C.c_float]),
    "rb_spatial_volumes": (None, [C.POINTER(C.c_float), C.POINTER(C.c_float), C.POINTER(C.c_float),
                                  C.POINTER(C.c_float)]),
}


class RodioB200Error(RuntimeError):
    def __init__(self, status: int, where: str, detail: str):
        self.status = status
        super().__init__(f"{where}: status {status} ({detail})")


_lib = None


def lib():
    """Load librodio_b200.so (hard error when it was not built — there is no fallback path)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} is missing: build it with `python -m rodio_b200.build` "
                "(rodio_b200 has no CPU fallback)")
        L = C.CDLL(LIB_PATH)
        for name, (res, args) in SYMBOLS.items():
            fn = getattr(L, name)   # AttributeError if the header and the library disagree
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def check(status: int, where: str):
    if status != RB_OK:
        L = lib()
        detail = f"{L.rb_status_string(status).decode()}: {L.rb_last_error().decode()}"
        raise RodioB200Error(status, where, detail)
