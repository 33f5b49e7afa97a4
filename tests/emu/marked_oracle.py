"""The CPU oracle with a source whose current_span_len() follows a mark table (tests/emu/marked_oracle.cpp): a decoder that reports
the packet it decoded last.  Compiled on first use into tests/emu/libmarked_oracle.so with the oracle's flags (g++ only); rebuilt
when a source it is made of is newer."""
import ctypes as C
import os
import subprocess

import numpy as np

import oracle

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
SRC = os.path.join(HERE, "marked_oracle.cpp")
LIB = os.path.join(HERE, "libmarked_oracle.so")
DEPS = [SRC, os.path.join(ROOT, "oracle", "rodio_oracle_capi.cpp"), os.path.join(ROOT, "oracle", "rodio_oracle.hpp")]
# the flags of oracle/Makefile: rustc never fuses a*b+c, neither may the restatement
CXX = ["g++", "-O3", "-march=x86-64-v3", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-pthread", "-shared"]

_lib = None


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB) or any(os.path.getmtime(d) > os.path.getmtime(LIB) for d in DEPS):
            tmp = f"{LIB}.{os.getpid()}.tmp"
            subprocess.run(CXX + [SRC, "-o", tmp], check=True, capture_output=True)
            os.replace(tmp, LIB)
        L = C.CDLL(LIB)
        u64p, fp = C.POINTER(C.c_uint64), C.POINTER(C.c_float)
        L.ro_marked_chain_uniform.restype = C.c_int
        L.ro_marked_chain_uniform.argtypes = [C.c_void_p, u64p, C.c_uint64, C.c_uint16, C.c_uint32, fp, C.c_uint64, u64p]
        L.ro_marked_mixer.restype = C.c_int
        L.ro_marked_mixer.argtypes = [C.c_void_p, C.c_uint64, u64p, u64p, C.c_uint16, C.c_uint32, fp, C.c_uint64, u64p]
        _lib = L
    return _lib


def _table(marks):
    return np.ascontiguousarray(np.asarray(list(marks), dtype=np.uint64).reshape(-1, 2)).reshape(-1)


def _u64(a):
    return a.ctypes.data_as(C.POINTER(C.c_uint64))


def chain_uniform(s: oracle.Stream, marks, mixer_channels: int, mixer_rate: int) -> np.ndarray:
    """oracle.chain_uniform with the stream's PCM a source that reports s.span_len (0 = None) before the first mark, then the
    span_len of the last mark (at, span_len) with `at` <= the samples it has yielded."""
    arr, keep = oracle._pack([s])
    t = _table(marks)
    return oracle._grow(lambda out, cap, n: lib().ro_marked_chain_uniform(C.byref(arr[0]), _u64(t), t.size // 2, mixer_channels, mixer_rate,
                                                                          oracle._fptr(out), cap, C.byref(n)), 1 << 16)


def mixer(streams, marks, channels: int, rate: int) -> np.ndarray:
    """oracle.mixer with stream i's PCM reporting by marks[i] (see chain_uniform); gaps are 0.0."""
    arr, keep = oracle._pack(streams)
    tables = [_table(m) for m in marks]
    first = np.cumsum([0] + [t.size // 2 for t in tables]).astype(np.uint64)
    t = np.ascontiguousarray(np.concatenate(tables + [np.zeros(0, np.uint64)]))
    return oracle._grow(lambda out, cap, n: lib().ro_marked_mixer(arr, len(streams), _u64(first), _u64(t), channels, rate, oracle._fptr(out), cap,
                                                                  C.byref(n)), 1 << 16)
