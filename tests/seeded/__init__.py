"""Checkers of seeded solves -- TEST INFRASTRUCTURE ONLY.

  oracle_seeded.cc -> libcmvm_oracle_seeded.so   the CPU oracle (oracle/cmvm_oracle.cc, unmodified) with the seeded
                                                 tie-break of the greedy selection threaded through
  sim_seeded.cc    -> libsim_seeded.so           the SIMT harness of tests/simt with a seed per job

The seeded order is this project's extension, not the reference's: seed 0 is the reference's rule.  Both libraries are
built on first use, as tests/simt builds its harness."""
from __future__ import annotations

import ctypes as C
import os
import subprocess
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
ROOT = HERE.parent.parent
CXX = '/usr/bin/g++' if Path('/usr/bin/g++').exists() else 'g++'


def _build(src: Path, lib: Path, deps, flags) -> Path:
    if not lib.exists() or lib.stat().st_mtime < max(p.stat().st_mtime for p in [src, *deps]):
        tmp = lib.with_name(f'.{lib.name}.{os.getpid()}')  # concurrent test workers: build aside, rename atomically
        subprocess.run([CXX, *flags, '-fPIC', '-shared', '-w', str(src), '-o', str(tmp)], check=True)
        os.replace(tmp, lib)
    return lib


_FP, _IP = C.POINTER(C.c_float), C.POINTER(C.c_int64)
_oracle = _sim = None


def oracle_lib():
    global _oracle
    if _oracle is None:
        path = _build(HERE / 'oracle_seeded.cc', HERE / 'libcmvm_oracle_seeded.so', [ROOT / 'oracle' / 'cmvm_oracle.cc'], ['-O3', '-std=c++20', '-fopenmp'])
        L = C.CDLL(str(path))
        L.orc_last_error.restype = C.c_char_p
        L.orc_tb_mask.restype = C.c_uint64
        L.orc_tb_mask.argtypes = [C.c_uint64]
        L.orc_solve_seeded.restype = C.c_void_p
        L.orc_solve_seeded.argtypes = [_FP, C.c_int64, C.c_int64, C.c_char_p, C.c_char_p, C.c_int, C.c_int, _FP, _FP, C.c_int, C.c_int, C.c_int, C.c_uint64]
        L.orc_solve_single_seeded.restype = C.c_void_p
        L.orc_solve_single_seeded.argtypes = [_FP, C.c_int64, C.c_int64, C.c_char_p, _FP, _FP, C.c_int, C.c_int, C.c_uint64]
        L.orc_free.argtypes = [C.c_void_p]
        L.orc_n_stages.restype = C.c_int64
        L.orc_n_stages.argtypes = [C.c_void_p]
        L.orc_stage_n_ops.restype = C.c_int64
        L.orc_stage_n_ops.argtypes = [C.c_void_p, C.c_int64]
        L.orc_stage_meta.argtypes = [C.c_void_p, C.c_int64, _IP]
        L.orc_stage_copy.argtypes = [C.c_void_p, C.c_int64, _IP, _IP, _IP, _IP, _IP, _FP]
        _oracle = L
    return _oracle


def _stages(L, h):
    out = []
    for s in range(L.orc_n_stages(h)):
        meta = np.zeros(11, np.int64)
        L.orc_stage_meta(h, s, meta.ctypes.data_as(_IP))
        n_in, n_out, n_ops = int(meta[0]), int(meta[1]), L.orc_stage_n_ops(h, s)
        st = dict(shape=(n_in, n_out), inp_shifts=np.zeros(n_in, np.int64), out_idxs=np.zeros(n_out, np.int64), out_shifts=np.zeros(n_out, np.int64),
                  out_negs=np.zeros(n_out, np.int64), ops_i=np.zeros((n_ops, 4), np.int64), ops_f=np.zeros((n_ops, 5), np.float32),
                  counters=dict(T=int(meta[4]), sum_F=int(meta[5]), sum_R=int(meta[6]), F0=int(meta[7]), R0=int(meta[8]), D0=int(meta[9]), D_final=int(meta[10])))  # fmt: skip
        L.orc_stage_copy(h, s, *[st[k].ctypes.data_as(_IP) for k in ('inp_shifts', 'out_idxs', 'out_shifts', 'out_negs', 'ops_i')], st['ops_f'].ctypes.data_as(_FP))
        out.append(st)
    return out


def _arrays(kernel, qintervals, latencies):
    k = np.ascontiguousarray(kernel, dtype=np.float32)
    q = None if qintervals is None else np.ascontiguousarray(np.asarray(qintervals, dtype=np.float32).reshape(-1, 3))
    l = None if latencies is None else np.ascontiguousarray(np.asarray(latencies, dtype=np.float32).reshape(-1))
    return k, q, l


def _fp(a):
    return None if a is None else a.ctypes.data_as(_FP)


def _run(L, h):
    if not h:
        raise RuntimeError(L.orc_last_error().decode())
    try:
        return _stages(L, h)
    finally:
        L.orc_free(h)


def tb_mask(seed: int) -> int:
    return int(oracle_lib().orc_tb_mask(int(seed)))


def solve(kernel, method0='wmc', method1='auto', hard_dc=-1, decompose_dc=-2, qintervals=None, latencies=None, adder_size=-1, carry_size=-1,
          search_all_decompose_dc=True, seed=0):  # fmt: skip
    """The oracle's ``solve`` under the seeded tie-break (stage dicts, as oracle.port.solve)."""
    L = oracle_lib()
    k, q, l = _arrays(kernel, qintervals, latencies)
    return _run(L, L.orc_solve_seeded(_fp(k), k.shape[0], k.shape[1], method0.encode(), method1.encode(), hard_dc, decompose_dc, _fp(q), _fp(l), adder_size, carry_size,
                                      int(search_all_decompose_dc), int(seed)))  # fmt: skip


def solve_single(kernel, method='wmc', qintervals=None, latencies=None, adder_size=-1, carry_size=-1, seed=0):
    L = oracle_lib()
    k, q, l = _arrays(kernel, qintervals, latencies)
    return _run(L, L.orc_solve_single_seeded(_fp(k), k.shape[0], k.shape[1], method.encode(), _fp(q), _fp(l), adder_size, carry_size, int(seed)))[0]


def n_adders(stages) -> int:
    return int(sum(int(np.count_nonzero(np.asarray(st['ops_i'])[:, 2] >= 0)) for st in stages))


# ---- the simulated kernels ---------------------------------------------------------------------------------------------
def sim_lib():
    global _sim
    if _sim is None:
        simt_dir, csrc = ROOT / 'tests' / 'simt', ROOT / 'da4ml_b200' / 'csrc'
        deps = [simt_dir / 'sim_cmvm.cc', simt_dir / 'simt.h', *sorted(csrc.glob('*.cuh'))]
        path = _build(HERE / 'sim_seeded.cc', HERE / 'libsim_seeded.so', deps, ['-O2', '-std=c++17', '-ffp-contract=off'])
        L = C.CDLL(str(path))
        L.sim_last_error.restype = C.c_char_p
        L.sim_seed_set.argtypes = [C.POINTER(C.c_uint64), C.c_int]
        L.sim_solve_single.restype = C.c_longlong
        L.sim_solve_single.argtypes = [_FP, C.c_int, C.c_int, C.c_char_p, _FP, _FP, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int,
                                       _IP, _IP, _IP, _IP, _IP, _IP, _FP, C.c_longlong]  # fmt: skip
        PFP, PIP = C.POINTER(_FP), C.POINTER(_IP)
        L.sim_solve_many.argtypes = [C.c_int, PFP, C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_char_p, PFP, PFP, C.c_int, C.c_int, C.c_int,
                                     PIP, PIP, PIP, PIP, PIP, PIP, PFP, C.POINTER(C.c_longlong), C.POINTER(C.c_longlong)]  # fmt: skip
        L.sim_set_segment_cap.argtypes = [C.c_int]
        L.sim_set_caps.argtypes = [C.c_int, C.c_int]
        L.sim_set_own_caps.argtypes = [C.c_int, C.c_int]
        L.sim_set_list_cap.argtypes = [C.c_int]
        _sim = L
    return _sim


def _set_seeds(seeds):
    s = (C.c_uint64 * max(len(seeds), 1))(*[int(v) for v in seeds])
    sim_lib().sim_seed_set(s, len(seeds))


def sim_solve_single(kernel, method='wmc', seed=0, qintervals=None, latencies=None, adder_size=-1, carry_size=-1, ctas=2, cta_threads=64, accounting=False, list_mul=2):
    """One seeded solve_single on the simulated kernels -> (stage dict, counters[32]); a capacity status raises
    RuntimeError('... capacity status N')."""
    L = sim_lib()
    k = np.ascontiguousarray(kernel, dtype=np.float32)
    n_in, n_out = k.shape
    q = np.ascontiguousarray(np.tile(np.array([-128.0, 127.0, 1.0], np.float32), (n_in, 1)) if qintervals is None else np.asarray(qintervals, np.float32))
    l = np.zeros(n_in, np.float32) if latencies is None else np.ascontiguousarray(latencies, dtype=np.float32)
    room = n_in + int(np.count_nonzero(k)) * 34 + 8
    meta = np.zeros(32, np.int64)
    st = dict(inp_shifts=np.zeros(n_in, np.int64), out_idxs=np.zeros(n_out, np.int64), out_shifts=np.zeros(n_out, np.int64), out_negs=np.zeros(n_out, np.int64))
    ops_i = np.zeros((room, 4), np.int64)
    ops_f = np.zeros((room, 5), np.float32)
    ip = lambda a: a.ctypes.data_as(_IP)  # noqa: E731
    _set_seeds([seed])
    n = L.sim_solve_single(_fp(k), n_in, n_out, method.encode(), _fp(q), _fp(l), adder_size, carry_size, ctas, cta_threads, int(accounting), list_mul, ip(meta),
                           ip(st['inp_shifts']), ip(st['out_idxs']), ip(st['out_shifts']), ip(st['out_negs']), ip(ops_i), _fp(ops_f), room)  # fmt: skip
    if n == -100:
        raise RuntimeError(L.sim_last_error().decode())
    if n < 0:
        raise RuntimeError(f'simulated kernel reported capacity status {-n}')
    st['ops_i'] = ops_i[:n].copy()
    st['ops_f'] = ops_f[:n].copy()
    return st, meta


def sim_solve_many(kernels, seeds, method='wmc', ctas=2, groups=1, cta_threads=64):
    """Seeded solve_single jobs (job i under seeds[i], default options otherwise) in ONE simulated launch."""
    L = sim_lib()
    ks = [np.ascontiguousarray(k, dtype=np.float32) for k in kernels]
    n = len(ks)
    qs = [np.ascontiguousarray(np.tile(np.array([-128.0, 127.0, 1.0], np.float32), (k.shape[0], 1))) for k in ks]
    ls = [np.zeros(k.shape[0], np.float32) for k in ks]
    rooms = [k.shape[0] + int(np.count_nonzero(k)) * 34 + 8 for k in ks]
    metas = [np.zeros(32, np.int64) for _ in ks]
    sts = [dict(inp_shifts=np.zeros(k.shape[0], np.int64), out_idxs=np.zeros(k.shape[1], np.int64), out_shifts=np.zeros(k.shape[1], np.int64),
                out_negs=np.zeros(k.shape[1], np.int64)) for k in ks]  # fmt: skip
    ops_i = [np.zeros((r, 4), np.int64) for r in rooms]
    ops_f = [np.zeros((r, 5), np.float32) for r in rooms]
    fa = lambda arrs: (_FP * n)(*[a.ctypes.data_as(_FP) for a in arrs])  # noqa: E731
    ia = lambda arrs: (_IP * n)(*[a.ctypes.data_as(_IP) for a in arrs])  # noqa: E731
    n_ops = (C.c_longlong * n)()
    _set_seeds(seeds)
    rc = L.sim_solve_many(n, fa(ks), (C.c_int * n)(*[k.shape[0] for k in ks]), (C.c_int * n)(*[k.shape[1] for k in ks]), method.encode(), fa(qs), fa(ls), ctas, groups,
                          cta_threads, ia(metas), ia([s['inp_shifts'] for s in sts]), ia([s['out_idxs'] for s in sts]), ia([s['out_shifts'] for s in sts]),
                          ia([s['out_negs'] for s in sts]), ia(ops_i), fa(ops_f), (C.c_longlong * n)(*rooms), n_ops)  # fmt: skip
    if rc != 0:
        raise RuntimeError(L.sim_last_error().decode())
    for i, st in enumerate(sts):
        if n_ops[i] < 0:
            raise RuntimeError(f'simulated kernel reported capacity status {-n_ops[i]} for job {i}')
        st['ops_i'] = ops_i[i][: n_ops[i]].copy()
        st['ops_f'] = ops_f[i][: n_ops[i]].copy()
    return sts
