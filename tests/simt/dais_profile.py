"""g++ build of the DAIS evaluator (da4ml_b200/csrc/dais_replay.cuh) behind the op-code driver of
dais_profile_harness.cc -- TEST INFRASTRUCTURE ONLY: per-op statistics and dumps of the op codes on the CPU."""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
LIB = HERE / 'libdais_profile.so'
CSRC = HERE.parent.parent / 'da4ml_b200' / 'csrc'
I64_MAX, I64_MIN = (1 << 63) - 1, -(1 << 63)

_lib = None


def build() -> Path:
    srcs = [HERE / 'dais_profile_harness.cc', CSRC / 'dais_replay.cuh', CSRC / 'dais_program.cuh']
    if not LIB.exists() or LIB.stat().st_mtime < max(p.stat().st_mtime for p in srcs):
        gxx = '/usr/bin/g++' if Path('/usr/bin/g++').exists() else 'g++'
        tmp = HERE / f'.libdais_profile.{os.getpid()}.so'  # concurrent test workers: build aside, rename atomically
        subprocess.run([gxx, '-O2', '-std=c++17', '-ffp-contract=off', '-fPIC', '-shared', str(HERE / 'dais_profile_harness.cc'), '-o', str(tmp)], check=True)
        os.replace(tmp, LIB)
    return LIB


def _harness():
    global _lib
    if _lib is None:
        L = C.CDLL(str(build()))
        L.dp_last_error.restype = C.c_char_p
        L.dp_profile.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p]
        L.dp_dump.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p]
        _lib = L
    return _lib


def _prog_inputs(prog, x):
    prog = np.ascontiguousarray(prog, dtype=np.int32)
    return prog, np.ascontiguousarray(np.asarray(x, dtype=np.float64).reshape(-1, max(int(prog[2]), 1)))


def stats(prog, x) -> np.ndarray:
    """[n_ops, 3] int64 {min, max, OR} of the op codes over the rows of ``x``; failures raise RuntimeError."""
    prog, x = _prog_inputs(prog, x)
    st = np.tile(np.array([I64_MAX, I64_MIN, 0], np.int64), (int(prog[4]), 1))
    if _harness().dp_profile(prog.ctypes.data, prog.size, x.ctypes.data, x.shape[0], st.ctypes.data):
        raise RuntimeError(_harness().dp_last_error().decode())
    return st


def dump(prog, x, ops=None) -> np.ndarray:
    """[n_samples, len(ops)] int64 codes of ops ``ops`` (default: all); failures raise RuntimeError."""
    prog, x = _prog_inputs(prog, x)
    sel = np.ascontiguousarray(np.arange(int(prog[4])) if ops is None else ops, dtype=np.int32)
    out = np.zeros((x.shape[0], sel.size), np.int64)
    if _harness().dp_dump(prog.ctypes.data, prog.size, x.ctypes.data, x.shape[0], sel.ctypes.data, sel.size, out.ctypes.data):
        raise RuntimeError(_harness().dp_last_error().decode())
    return out
