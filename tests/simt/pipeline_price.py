"""g++ build of the pipelined-pricing kernel and its host code (da4ml_b200/csrc/pipeline_price.cuh) under the SIMT shim --
TEST INFRASTRUCTURE ONLY (see pipeline_price_harness.cc)."""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
LIB = HERE / 'libpipeline_price.so'
CSRC = HERE.parent.parent / 'da4ml_b200' / 'csrc'

_lib = None


def build() -> Path:
    srcs = [HERE / 'pipeline_price_harness.cc', HERE / 'simt.h', CSRC / 'pipeline_price.cuh', CSRC / 'cmvm_num.cuh', CSRC / 'cmvm_types.cuh']
    if not LIB.exists() or LIB.stat().st_mtime < max(p.stat().st_mtime for p in srcs):
        gxx = '/usr/bin/g++' if Path('/usr/bin/g++').exists() else 'g++'
        tmp = LIB.with_name(f'.{LIB.name}.{os.getpid()}')  # concurrent test workers: build aside, rename atomically
        subprocess.run([gxx, '-O2', '-std=c++17', '-ffp-contract=off', '-fPIC', '-shared', '-w', str(HERE / 'pipeline_price_harness.cc'), '-o', str(tmp)], check=True)
        os.replace(tmp, LIB)
    return LIB


def price(designs, latency_cutoff, latencies=None, retiming=True, threads=64) -> dict:
    """``price_pipelined`` on the simulated kernel with CTAs of ``threads`` threads: dict of the ``[n_designs,
    n_cutoffs]`` arrays, ``out_latency`` (a list per design of ``[n_cutoffs, n_out]``) and ``launches``."""
    global _lib
    if _lib is None:
        L = C.CDLL(str(build()))
        L.pph_last_error.restype = C.c_char_p
        I, F, D = C.POINTER(C.c_int64), C.POINTER(C.c_float), C.POINTER(C.c_double)
        L.pph_price.argtypes = [C.c_int64, I, I, I, I, I, I, I, F, D, D, C.c_int64, C.c_int, C.c_int, C.POINTER(C.c_int32), I, I, D, D, D, I]
        _lib = L
    from da4ml_b200._binary import _price_args

    pk = _price_args(designs, latency_cutoff, latencies)
    n, m = len(pk['designs']), pk['cutoffs'].size
    n_out = [d[-1]['shape'][1] for d in pk['designs']]
    st = np.zeros(n * m, np.int32)
    stg, rb = np.zeros(n * m, np.int64), np.zeros(n * m, np.int64)
    lm, co = np.zeros(n * m), np.zeros(n * m)
    ol = np.zeros(max(sum(n_out) * m, 1))
    launches = np.zeros(1, np.int64)
    I = lambda a: a.ctypes.data_as(C.POINTER(C.c_int64))  # noqa: E731
    D = lambda a: None if a is None else a.ctypes.data_as(C.POINTER(C.c_double))  # noqa: E731
    rc = _lib.pph_price(n, *[I(pk[k]) for k in ('n_stages', 'meta', 'inp_shifts', 'out_idxs', 'out_shifts', 'out_negs', 'ops_i')],
                        pk['ops_f'].ctypes.data_as(C.POINTER(C.c_float)), D(pk['latencies']), D(pk['cutoffs']), m, int(bool(retiming)), int(threads),
                        st.ctypes.data_as(C.POINTER(C.c_int32)), I(stg), I(rb), D(lm), D(co), D(ol), I(launches))  # fmt: skip
    if rc:
        raise ValueError(_lib.pph_last_error().decode())
    edges = np.concatenate([[0], np.cumsum(np.asarray(n_out, np.int64) * m)])
    return dict(status=st.reshape(n, m), stages=stg.reshape(n, m), reg_bits=rb.reshape(n, m), latency_max=lm.reshape(n, m), cutoff=co.reshape(n, m),
                out_latency=[ol[edges[d] : edges[d + 1]].reshape(m, n_out[d]) for d in range(n)], launches=int(launches[0]))  # fmt: skip
