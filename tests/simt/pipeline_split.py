"""g++ build of the split kernels and their host code (da4ml_b200/csrc/pipeline_split.cuh) under the SIMT shim --
TEST INFRASTRUCTURE ONLY (see pipeline_split_harness.cc)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
LIB = HERE / 'libpipeline_split.so'
CSRC = HERE.parent.parent / 'da4ml_b200' / 'csrc'

_lib = None


def build() -> Path:
    srcs = [HERE / 'pipeline_split_harness.cc', HERE / 'simt.h', CSRC / 'pipeline_split.cuh', CSRC / 'pipeline_price.cuh', CSRC / 'cmvm_num.cuh', CSRC / 'cmvm_types.cuh']
    if not LIB.exists() or LIB.stat().st_mtime < max(p.stat().st_mtime for p in srcs):
        gxx = '/usr/bin/g++' if Path('/usr/bin/g++').exists() else 'g++'
        tmp = LIB.with_name(f'.{LIB.name}.{os.getpid()}')  # concurrent test workers: build aside, rename atomically
        subprocess.run([gxx, '-O2', '-std=c++17', '-ffp-contract=off', '-fPIC', '-shared', '-w', str(HERE / 'pipeline_split_harness.cc'), '-o', str(tmp)], check=True)
        os.replace(tmp, LIB)
    return LIB


def split(designs, latency_cutoff, latencies=None, retiming=True, threads=64):
    """``price_pipelined(..., keep_split=True)`` on the simulated kernels with CTAs of ``threads`` threads: a
    ``PipelinePrice`` whose ``split(d, j)`` answers (``profile['launches']``: the simulated launches)."""
    global _lib
    if _lib is None:
        L = C.CDLL(str(build()))
        L.psh_last_error.restype = C.c_char_p
        I, F, D = C.POINTER(C.c_int64), C.POINTER(C.c_float), C.POINTER(C.c_double)
        L.psh_split.argtypes = [C.c_int64, I, I, I, I, I, I, I, F, D, D, C.c_int64, C.c_int, C.c_int, C.POINTER(C.c_int32), I, I, D, D, I]
        L.psh_info.argtypes = [C.c_int64, I]
        L.psh_copy.argtypes = [C.c_int64, I, I, I, I, I, D]
        _lib = L
    from da4ml_b200._binary import PipelinePrice, _price_args, _take_splits

    pk = _price_args(designs, latency_cutoff, latencies)
    n, m = len(pk['designs']), pk['cutoffs'].size
    st = np.zeros(n * m, np.int32)
    stg, rb = np.zeros(n * m, np.int64), np.zeros(n * m, np.int64)
    lm, co = np.zeros(n * m), np.zeros(n * m)
    launches = np.zeros(1, np.int64)
    I = lambda a: a.ctypes.data_as(C.POINTER(C.c_int64))  # noqa: E731
    D = lambda a: None if a is None else a.ctypes.data_as(C.POINTER(C.c_double))  # noqa: E731
    rc = _lib.psh_split(n, *[I(pk[k]) for k in ('n_stages', 'meta', 'inp_shifts', 'out_idxs', 'out_shifts', 'out_negs', 'ops_i')],
                        pk['ops_f'].ctypes.data_as(C.POINTER(C.c_float)), D(pk['latencies']), D(pk['cutoffs']), m, int(bool(retiming)), int(threads),
                        st.ctypes.data_as(C.POINTER(C.c_int32)), I(stg), I(rb), D(lm), D(co), I(launches))  # fmt: skip
    if rc:
        raise ValueError(_lib.psh_last_error().decode())
    f = lambda a: a.ctypes.data_as(C.POINTER(C.c_double) if a.dtype == np.float64 else C.POINTER(C.c_int64))  # noqa: E731
    splits = _take_splits(pk['designs'], m, lambda t, q: _lib.psh_info(t, I(q)), lambda t, *a: _lib.psh_copy(t, *map(f, a)))
    return PipelinePrice(st.reshape(n, m), stg.reshape(n, m), rb.reshape(n, m), lm.reshape(n, m), co.reshape(n, m), pk['cutoffs'], [None] * n,
                         dict(launches=int(launches[0])), splits)  # fmt: skip
