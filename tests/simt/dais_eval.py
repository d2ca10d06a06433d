"""g++ build of the DAIS evaluator (da4ml_b200/csrc/dais_replay.cuh) and host checks (dais_program.cuh) behind a
sequential driver -- TEST INFRASTRUCTURE ONLY (see dais_eval_harness.cc)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
LIB = HERE / 'libdais_eval.so'
CSRC = HERE.parent.parent / 'da4ml_b200' / 'csrc'

_lib = None


def build() -> Path:
    srcs = [HERE / 'dais_eval_harness.cc', CSRC / 'dais_replay.cuh', CSRC / 'dais_program.cuh']
    if not LIB.exists() or LIB.stat().st_mtime < max(p.stat().st_mtime for p in srcs):
        gxx = '/usr/bin/g++' if Path('/usr/bin/g++').exists() else 'g++'
        tmp = LIB.with_name(f'.{LIB.name}.{os.getpid()}')  # concurrent test workers: build aside, rename atomically
        subprocess.run([gxx, '-O2', '-std=c++17', '-ffp-contract=off', '-fPIC', '-shared', str(HERE / 'dais_eval_harness.cc'), '-o', str(tmp)], check=True)
        os.replace(tmp, LIB)
    return LIB


def run(program, data) -> np.ndarray:
    """Same contract as the reference's ``run_interp``: float64 [n_samples, n_in] -> float64 [n_samples, n_out];
    failures raise RuntimeError with the message."""
    global _lib
    if _lib is None:
        L = C.CDLL(str(build()))
        L.dh_last_error.restype = C.c_char_p
        L.dh_run.argtypes = [C.POINTER(C.c_int32), C.c_int64, C.POINTER(C.c_double), C.c_int64, C.POINTER(C.c_double)]
        _lib = L
    prog = np.ascontiguousarray(program, dtype=np.int32)
    n_in, n_out = int(prog[2]), int(prog[3])
    x = np.ascontiguousarray(np.asarray(data, dtype=np.float64).reshape(-1, max(n_in, 1)))
    out = np.zeros((x.shape[0], n_out), np.float64)
    if _lib.dh_run(prog.ctypes.data_as(C.POINTER(C.c_int32)), prog.size, x.ctypes.data_as(C.POINTER(C.c_double)), x.shape[0], out.ctypes.data_as(C.POINTER(C.c_double))):
        raise RuntimeError(_lib.dh_last_error().decode())
    return out
