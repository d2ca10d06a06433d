"""ctypes binding of libda4ml_b200_cmvm.so (C ABI: include/da4ml_b200_cmvm.h).

Mirror of the reference's ``da4ml._binary`` re-exports (``src/da4ml/_binary/__init__.py:4,19``;
nanobind module ``_binary/cmvm/bindings.cc:227-263``): ``solve, csd_decompose, int_arr_to_csd,
kernel_decompose, get_lsb_loc, iceil_log2, cost_add`` with the same signatures, defaults and exception
types.  Added on top: ``solve_batch`` (many independent problems in one launch) and ``solve_single``.

The shared library is the product's only compute path; importing this module without it raises.
"""

from __future__ import annotations

import contextlib
import copy
import ctypes as C
import time
from collections import namedtuple
from pathlib import Path

import numpy as np

from ..types import pipeline_from_arrays, stage_to_binary, stages_to_json

_LIB_PATH = Path(__file__).resolve().parent / 'libda4ml_b200_cmvm.so'
if not _LIB_PATH.exists():
    raise ImportError(
        f'{_LIB_PATH} not found: build it with `python -c "import __graft_entry__ as g; g.build()"` '
        '(nvcc, sm_90a). The CMVM solver has no CPU fallback.'
    )
_L = C.CDLL(str(_LIB_PATH))

_f32p = C.POINTER(C.c_float)
_i64p = C.POINTER(C.c_int64)
_i32p = C.POINTER(C.c_int32)
_i8p = C.POINTER(C.c_int8)
_vp = C.c_void_p

_L.da4ml_cmvm_last_error.restype = C.c_char_p
_L.da4ml_cmvm_device_info.argtypes = [_i32p]
_L.da4ml_cmvm_set_stream.argtypes = [_vp]
_L.da4ml_cmvm_plan.argtypes = [_i64p, C.c_int64, C.c_int, C.c_int, _i64p]
_L.da4ml_cmvm_set_group_size.argtypes = [C.c_int]
_L.da4ml_cmvm_set_accounting.argtypes = [C.c_int]
_L.da4ml_cmvm_set_job_sharing.argtypes = [C.c_int]
_L.da4ml_cmvm_set_capacity_override.argtypes = [_i64p]
_L.da4ml_cmvm_solve.argtypes = [_f32p, C.c_int64, C.c_int64, C.c_char_p, C.c_char_p, C.c_int, C.c_int, _f32p, _f32p, C.c_int, C.c_int, C.c_int, C.POINTER(_vp)]
_L.da4ml_cmvm_solve_batch.argtypes = [C.c_int64, C.POINTER(_f32p), _i64p, _i64p, C.c_char_p, C.c_char_p, C.c_int, C.c_int, C.POINTER(_f32p), C.POINTER(_f32p), C.c_int, C.c_int, C.c_int, C.POINTER(_vp)]
_L.da4ml_cmvm_solve_batch_device.argtypes = [C.c_int64, C.POINTER(_vp), _i64p, _i64p, C.c_char_p, C.c_char_p, C.c_int, C.c_int, C.POINTER(_f32p), C.POINTER(_f32p), C.c_int, C.c_int, C.c_int, C.POINTER(_vp)]
_L.da4ml_cmvm_solve_single.argtypes = [_f32p, C.c_int64, C.c_int64, C.c_char_p, _f32p, _f32p, C.c_int, C.c_int, _i32p, C.c_int64, C.POINTER(_vp)]
_L.da4ml_cmvm_solve_seeded.argtypes = [_f32p, C.c_int64, C.c_int64, C.c_char_p, C.c_char_p, C.c_int, C.c_int, _f32p, _f32p, C.c_int, C.c_int, C.c_int, C.c_uint64, C.POINTER(_vp)]
_L.da4ml_cmvm_solve_single_seeded.argtypes = [_f32p, C.c_int64, C.c_int64, C.c_char_p, _f32p, _f32p, C.c_int, C.c_int, _i32p, C.c_int64, C.c_uint64, C.POINTER(_vp)]
_L.da4ml_cmvm_solve_sweep.argtypes = [_f32p, C.c_int64, C.c_int64, _f32p, _f32p, C.c_int, C.c_int, C.c_int64, C.POINTER(C.c_char_p), C.POINTER(C.c_char_p), _i32p, _i32p, _i32p, C.c_int, C.POINTER(_vp)]
_L.da4ml_cmvm_solve_sweep_batch.argtypes = [C.c_int64, C.POINTER(_f32p), _i64p, _i64p, C.POINTER(_f32p), C.POINTER(_f32p), C.c_int, C.c_int, C.c_int64, C.POINTER(C.c_char_p),
                                            C.POINTER(C.c_char_p), _i32p, _i32p, _i32p, C.c_int, C.POINTER(_vp)]
_L.da4ml_cmvm_solve_sweep_batch_seeded.argtypes = [C.c_int64, C.POINTER(_f32p), _i64p, _i64p, C.POINTER(_f32p), C.POINTER(_f32p), C.c_int, C.c_int, C.c_int64,
                                                   C.POINTER(C.c_char_p), C.POINTER(C.c_char_p), _i32p, _i32p, _i32p, C.POINTER(C.c_uint64), C.c_int, C.POINTER(_vp)]
_L.da4ml_sweep_counts.argtypes = [_vp, _i64p]
_L.da4ml_sweep_profile.argtypes = [_vp, C.POINTER(C.c_double)]
_L.da4ml_sweep_summary.argtypes = [_vp, _i64p, _f32p]
_L.da4ml_sweep_pipeline.argtypes = [_vp, C.c_int64, C.POINTER(_vp)]
_L.da4ml_sweep_free.argtypes = [_vp]
_L.da4ml_sweep_free.restype = None
_L.da4ml_sweep_front.argtypes = [_f32p, _f32p, C.c_int64, _i8p]
_L.da4ml_pipeline_free.argtypes = [_vp]
_L.da4ml_pipeline_n_stages.restype = C.c_int64
_L.da4ml_pipeline_n_stages.argtypes = [_vp]
_L.da4ml_pipeline_stage_meta.argtypes = [_vp, C.c_int64, _i64p]
_L.da4ml_pipeline_stage_copy.argtypes = [_vp, C.c_int64, _i64p, _i64p, _i64p, _i64p, _i64p, _f32p]
_L.da4ml_pipeline_stage_counters.argtypes = [_vp, C.c_int64, _i64p]
_L.da4ml_pipeline_stage_milestones.argtypes = [_vp, C.c_int64, _i64p]
_L.da4ml_pipeline_device_ms.restype = C.c_double
_L.da4ml_pipeline_device_ms.argtypes = [_vp]
_L.da4ml_pipeline_launches.restype = C.c_int64
_L.da4ml_pipeline_launches.argtypes = [_vp]
_L.da4ml_pipeline_profile.argtypes = [_vp, C.POINTER(C.c_double)]
_L.da4ml_cmvm_csd_decompose.argtypes = [_f32p, C.c_int64, C.c_int64, C.c_int, _i8p, _i8p, _i8p, _i64p]
_L.da4ml_cmvm_int_arr_to_csd.argtypes = [_i32p, C.c_int64, _i8p, _i64p]
_L.da4ml_cmvm_kernel_decompose.argtypes = [_f32p, C.c_int64, C.c_int64, C.c_int, _f32p, _f32p]
_L.da4ml_dais_run.argtypes = [_i32p, C.c_int64, C.POINTER(C.c_double), C.c_int64, C.POINTER(C.c_double)]
_L.da4ml_dais_program_load.argtypes = [_i32p, C.c_int64, C.POINTER(_vp)]
_L.da4ml_dais_program_info.argtypes = [_vp, _i64p]
_L.da4ml_dais_program_run.argtypes = [_vp, _vp, C.c_int64, _vp, C.c_int]
_L.da4ml_dais_program_run_stream.argtypes = [_vp, _vp, C.c_int64, _vp, C.c_int, _vp]
_L.da4ml_dais_program_profile.argtypes = [_vp, _vp, C.c_int64, C.c_int, _vp, _vp]
_L.da4ml_dais_program_dump.argtypes = [_vp, _vp, C.c_int64, _vp, C.c_int64, _vp, C.c_int, _vp]
_L.da4ml_dais_program_free.argtypes = [_vp]
_L.da4ml_dais_program_free.restype = None
_L.da4ml_cmvm_get_lsb_loc.argtypes = [C.c_float]
_L.da4ml_cmvm_iceil_log2.argtypes = [C.c_float]
_L.da4ml_cmvm_cost_add.argtypes = [_f32p, _f32p, C.c_int64, C.c_int, C.c_int, C.c_int, _f32p]
_f64p = C.POINTER(C.c_double)
_L.da4ml_pipeline_price.argtypes = [C.c_int64, _i64p, _i64p, _i64p, _i64p, _i64p, _i64p, _i64p, _f32p, _f64p, _f64p, C.c_int64, C.c_int, _i32p, _i64p, _i64p, _f64p,
                                    _f64p, _f64p, _f64p]  # fmt: skip
_L.da4ml_pipeline_split.argtypes = [*_L.da4ml_pipeline_price.argtypes, C.POINTER(_vp)]
_L.da4ml_split_info.argtypes = [_vp, C.c_int64, _i64p]
_L.da4ml_split_copy.argtypes = [_vp, C.c_int64, _i64p, _i64p, _i64p, _i64p, _i64p, _f64p]
_L.da4ml_split_free.argtypes = [_vp]
_L.da4ml_split_free.restype = None

EXPORTED_SYMBOLS = [
    'da4ml_cmvm_last_error', 'da4ml_cmvm_device_info', 'da4ml_cmvm_set_stream', 'da4ml_cmvm_set_group_size',
    'da4ml_cmvm_set_accounting', 'da4ml_cmvm_set_job_sharing', 'da4ml_pipeline_profile', 'da4ml_cmvm_release', 'da4ml_cmvm_plan',
    'da4ml_cmvm_solve', 'da4ml_cmvm_solve_batch', 'da4ml_cmvm_solve_batch_device', 'da4ml_cmvm_solve_single', 'da4ml_pipeline_free',
    'da4ml_pipeline_n_stages', 'da4ml_pipeline_stage_meta', 'da4ml_pipeline_stage_copy',
    'da4ml_pipeline_stage_counters', 'da4ml_pipeline_stage_milestones', 'da4ml_pipeline_device_ms', 'da4ml_pipeline_launches',
    'da4ml_cmvm_csd_decompose', 'da4ml_cmvm_int_arr_to_csd', 'da4ml_cmvm_kernel_decompose',
    'da4ml_cmvm_get_lsb_loc', 'da4ml_cmvm_iceil_log2', 'da4ml_cmvm_cost_add', 'da4ml_dais_run',
    'da4ml_dais_program_load', 'da4ml_dais_program_info', 'da4ml_dais_program_run', 'da4ml_dais_program_run_stream',
    'da4ml_dais_program_free', 'da4ml_dais_program_profile', 'da4ml_dais_program_dump', 'da4ml_cmvm_solve_sweep', 'da4ml_cmvm_solve_sweep_batch', 'da4ml_sweep_counts',
    'da4ml_sweep_profile', 'da4ml_sweep_summary', 'da4ml_sweep_pipeline', 'da4ml_sweep_free', 'da4ml_sweep_front',
    'da4ml_cmvm_solve_seeded', 'da4ml_cmvm_solve_single_seeded', 'da4ml_cmvm_solve_sweep_batch_seeded', 'da4ml_pipeline_price',
    'da4ml_pipeline_split', 'da4ml_split_info', 'da4ml_split_copy', 'da4ml_split_free', 'da4ml_cmvm_set_capacity_override',
]  # fmt: skip

COUNTER_NAMES = ['status', 'n_ops', 'T', 'sum_F', 'sum_R', 'F0', 'R0', 'D_final', 'F_max', 'compactions', 'D0', 'n_bits', 'group_ctas',
                 'rescanned', 'list_max', 'smem_list_cap']


def lib_path() -> Path:
    return _LIB_PATH


def _check(rc: int):
    if rc == 0:
        return
    msg = _L.da4ml_cmvm_last_error().decode()
    if rc == 1:
        raise ValueError(msg)  # nanobind maps std::invalid_argument -> ValueError
    raise RuntimeError(msg)  # std::runtime_error -> RuntimeError (e.g. "Unknown method: ...")


def device_info() -> dict:
    out = (C.c_int32 * 5)()
    _L.da4ml_cmvm_device_info(out)
    return dict(abi_version=out[0], cuda_devices=out[1], sm_count=out[2], cc=(out[3], out[4]))


PLAN_FIELDS = ['ctas_per_problem', 'concurrent_groups', 'columns_per_cta', 'list_rows_smem', 'log2_chunk', 'chunk_slots',
               'segment_entries_per_cta', 'log2_pair_counters', 'shared_bytes', 'shared_budget', 'narrow_rows', 'spill_rows']


def plan(jobs, co_resident_ctas: int = 132, group_override: int = 0) -> dict:
    """Launch geometry the solver would pick for ``jobs`` (no device needed).  Each job is a dict with ``n_in, n_out,
    nbits, digits`` (CSD digits of the matrix) and optionally ``dcol_max`` (digits of the densest column, default
    digits / n_out), ``col_cap`` (bound on rows per column list, default n_in + dcol_max), ``f_mul, list_mul``
    (retry multipliers, default 1, 2)."""
    rows = np.zeros((len(jobs), 8), np.int64)
    for r, j in zip(rows, jobs):
        dcol = int(j.get('dcol_max', -(-int(j['digits']) // int(j['n_out']))))
        r[:] = [j['n_in'], j['n_out'], j['nbits'], j['digits'], dcol, j.get('col_cap', int(j['n_in']) + dcol), j.get('f_mul', 1), j.get('list_mul', 2)]
    out = np.zeros(12, np.int64)
    _check(_L.da4ml_cmvm_plan(_ip(rows), len(jobs), int(co_resident_ctas), int(group_override), _ip(out)))
    return dict(zip(PLAN_FIELDS, (int(v) for v in out)))


def set_stream(cuda_stream: int | None):
    """Run every later call on this CUDA stream (``torch.cuda.current_stream().cuda_stream``)."""
    _L.da4ml_cmvm_set_stream(_vp(cuda_stream or 0))


def set_group_size(n: int):
    _L.da4ml_cmvm_set_group_size(int(n))


def release():
    """Free the device / pinned work buffers cached between calls."""
    _check(_L.da4ml_cmvm_release())


def set_job_sharing(on: bool):
    """Solve byte-identical solve_single jobs of one call once (default on; results are the same either way)."""
    _L.da4ml_cmvm_set_job_sharing(int(bool(on)))


def set_accounting(on: bool):
    """Exact work counters (sum over iterations of the live histogram size); slower, identical results."""
    _L.da4ml_cmvm_set_accounting(int(bool(on)))


CAPACITY_KNOBS = ['segment_entries', 'list_rows', 'spill_rows', 'hash_log', 'wide_rows', 'expr_cap', 'cell_pool', 'poison']


@contextlib.contextmanager
def capacity_override(**caps):
    """Test-only: squeeze the solve kernel's capacities inside the ``with`` block, so that small problems reach its spill,
    multi-pass, compaction, overflow and retry paths (``da4ml_cmvm_set_capacity_override``).  Knobs (``CAPACITY_KNOBS``,
    omitted = the planner's): ``segment_entries`` histogram entries per CTA, ``list_rows`` shared-memory rows per owner
    list (0: every row spills), ``spill_rows``, ``hash_log`` (8..13), ``wide_rows`` (bool), ``expr_cap`` expression ids
    beyond the inputs, ``cell_pool`` cells per CTA, ``poison`` (bool: 0xA5 in every buffer the driver does not clear).
    A knob only lowers the planner's value and grows with its retries; results must not change.  Every knob is reset on
    exit."""
    bad = set(caps) - set(CAPACITY_KNOBS)
    if bad:
        raise TypeError(f'unknown capacity knobs {sorted(bad)}; known: {CAPACITY_KNOBS}')
    v = np.full(len(CAPACITY_KNOBS), -1, np.int64)
    for k, x in caps.items():
        if x is not None:
            v[CAPACITY_KNOBS.index(k)] = (1 if x else -1) if k in ('wide_rows', 'poison') else int(x)
    _check(_L.da4ml_cmvm_set_capacity_override(_ip(v)))
    try:
        yield
    finally:
        _L.da4ml_cmvm_set_capacity_override(None)


def _fp(a):
    return a.ctypes.data_as(_f32p) if a is not None else None


def _ip(a):
    return a.ctypes.data_as(_i64p)


def _kernel_arg(kernel) -> np.ndarray:
    # the reference binds `kernel` as noconvert float ndarray (bindings.cc:238): no silent dtype casts
    if not isinstance(kernel, np.ndarray) or kernel.dtype != np.float32:
        raise TypeError('kernel must be a numpy float32 ndarray')
    if kernel.ndim != 2:
        raise RuntimeError('csd_decompose only supports 2D arrays.')
    return np.ascontiguousarray(kernel)


def _qint_arg(qintervals, n_in):
    # an empty sequence means "defaults", as in the reference (bindings.cc extract_qintervals -> api.cc:161-174)
    if qintervals is None or len(qintervals) == 0:
        return None
    q = np.ascontiguousarray(np.asarray([tuple(map(float, qi)) for qi in qintervals], dtype=np.float32).reshape(-1, 3))
    if q.shape[0] != n_in:
        raise ValueError(f'expected {n_in} qintervals, got {q.shape[0]}')
    return q


def _seed_arg(seed) -> int:
    # a tie-break seed is an unsigned 64-bit integer (see solve); checked before any device call
    if isinstance(seed, bool) or not isinstance(seed, (int, np.integer)):
        raise TypeError(f'seed must be an integer, got {type(seed).__name__}')
    s = int(seed)
    if not 0 <= s < 2**64:
        raise ValueError(f'seed must be in [0, 2**64), got {s}')
    return s


def tb_mask(seed) -> int:
    """The tie-break mask of ``seed``: 0 for seed 0, else ``splitmix64(seed) & (2**36 - 1)`` (the id0, sub and shift bits
    of the packed pair key).  Host restatement of the kernel's ``tb_mask`` (cmvm_num.cuh), for tests and tools."""
    s = _seed_arg(seed)
    if s == 0:
        return 0
    m = (1 << 64) - 1
    x = (s + 0x9E3779B97F4A7C15) & m
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & m
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & m
    return (x ^ (x >> 31)) & ((1 << 36) - 1)


def _lat_arg(latencies, n_in):
    if latencies is None or len(latencies) == 0:
        return None
    l = np.ascontiguousarray(np.asarray(list(latencies), dtype=np.float32).reshape(-1))
    if l.shape[0] != n_in:
        raise ValueError(f'expected {n_in} latencies, got {l.shape[0]}')
    return l


class RawPipeline:
    """Flat-array view of one solver result (what the C ABI hands back)."""

    def __init__(self, handle=None):
        self.stages = []
        self.counters = []
        self.device_ms = 0.0
        self.launches = 0
        self.profile = {}
        if handle is None:
            return
        try:
            for s in range(_L.da4ml_pipeline_n_stages(handle)):
                meta = np.zeros(5, np.int64)
                _check(_L.da4ml_pipeline_stage_meta(handle, s, _ip(meta)))
                n_in, n_out, n_ops = int(meta[0]), int(meta[1]), int(meta[2])
                st = dict(
                    shape=(n_in, n_out),
                    inp_shifts=np.zeros(n_in, np.int64),
                    out_idxs=np.zeros(n_out, np.int64),
                    out_shifts=np.zeros(n_out, np.int64),
                    out_negs=np.zeros(n_out, np.int64),
                    ops_i=np.zeros((n_ops, 4), np.int64),
                    ops_f=np.zeros((n_ops, 5), np.float32),
                    carry_size=int(meta[3]),
                    adder_size=int(meta[4]),
                )
                _check(_L.da4ml_pipeline_stage_copy(handle, s, _ip(st['inp_shifts']), _ip(st['out_idxs']), _ip(st['out_shifts']), _ip(st['out_negs']), _ip(st['ops_i']), _fp(st['ops_f'])))
                cnt = np.zeros(32, np.int64)
                _check(_L.da4ml_pipeline_stage_counters(handle, s, _ip(cnt)))
                self.stages.append(st)
                cd = dict(zip(COUNTER_NAMES, (int(v) for v in cnt)))
                cd['phase_cycles'] = [int(v) for v in cnt[16:24]]
                cd['phase_cycles_max'] = [int(v) for v in cnt[24:32]]
                ms = np.zeros(70, np.int64)
                _check(_L.da4ml_pipeline_stage_milestones(handle, s, _ip(ms)))
                cd['milestones'] = {250 << k: [int(v) for v in ms[10 * k : 10 * k + 10]] for k in range(7) if ms[10 * k + 9] > 0}
                self.counters.append(cd)
            self.device_ms = float(_L.da4ml_pipeline_device_ms(handle))
            self.launches = int(_L.da4ml_pipeline_launches(handle))
            prof = (C.c_double * 8)()
            _L.da4ml_pipeline_profile(handle, prof)
            self.profile = dict(device_ms=prof[0], launches=int(prof[1]), solve_kernel_ms=prof[2], solve_kernel_launches=int(prof[3]), algo_bytes=prof[4], jobs_total=int(prof[5]), jobs_run=int(prof[6]), solve_retries=int(prof[7]))
        finally:
            _L.da4ml_pipeline_free(handle)

    @property
    def n_adders(self) -> int:
        return int(sum(int(np.count_nonzero(st['ops_i'][:, 2] >= 0)) for st in self.stages))

    @classmethod
    def from_stages(cls, stages):
        """Wrap per-stage flat arrays that did not come from a solver handle (fixtures, results received from
        another rank)."""
        r = cls()
        r.stages = list(stages)
        return r

    def _no_lookups(self, what: str):
        if any((np.asarray(st['ops_i']).reshape(-1, 4)[:, 2] == 8).any() for st in self.stages):
            raise ValueError(f'{what}: this design has opcode 8 lookups, and the Pipeline containers of this package hold no lookup tables '
                             '(to_binary writes them)')

    def to_pipeline(self, types_module=None):
        self._no_lookups('to_pipeline')
        return pipeline_from_arrays(self.stages, types_module)

    # ---- serialisation straight from the flat arrays (SURVEY 8f N3): no per-op Python objects
    def to_binary(self, version: int = 0) -> list:
        """One DAIS int32 program per stage (reference ``CombLogic.to_binary``, types.py:500-541)."""
        return [stage_to_binary(st, version) for st in self.stages]

    def save_binary(self, path, version: int = 0):
        """Write stage ``i`` to ``<path>.<i>`` (a single-stage result goes to ``path`` itself), the layout
        ``CombLogic.save_binary`` uses per stage."""
        progs = self.to_binary(version)
        if len(progs) == 1:
            progs[0].tofile(path)
        else:
            for i, b in enumerate(progs):
                b.tofile(f'{path}.{i}')

    def to_json(self) -> str:
        """The text ``Pipeline.save`` writes (reference types.py:678-693)."""
        self._no_lookups('to_json')
        return stages_to_json(self.stages)

    def save(self, path):
        with open(path, 'w') as f:
            f.write(self.to_json())

    def predict_stage(self, i: int, data, n_threads: int = 0):
        """Bit-exact replay of stage ``i`` on a batch of inputs through the GPU DAIS interpreter (reference
        ``CombLogic.predict``, types.py:549-581).  Stages are replayed one at a time: the reference hands stage 1 the
        *unshifted* intervals of stage 0's output ops (api.cc:101-110), so feeding stage 0's outputs into stage 1 under
        fixed-point semantics would wrap -- the reference's ``Pipeline`` has no ``predict`` either."""
        return dais_interp_run(stage_to_binary(self.stages[i]), data, n_threads)

    def stage_kernel(self, i: int):
        """Constant matrix of stage ``i`` (reference ``CombLogic.kernel``, types.py:373-378), recovered on the GPU: input
        ``j`` is probed with one quantum of its declared interval (always representable and in range, unlike 1.0) and
        the response is divided by it -- exact, every factor is a power of two."""
        st = self.stages[i]
        n_in = int(st['shape'][0])
        oi = np.asarray(st['ops_i']).reshape(-1, 4)
        q = np.asarray(st['ops_f'], dtype=np.float32).reshape(-1, 5)[oi[:, 2] == -1][:, :3].astype(np.float64)
        probe = np.where(q[:, 1] >= q[:, 2], q[:, 2], np.where(q[:, 0] <= -q[:, 2], -q[:, 2], 0.0))
        out = self.predict_stage(i, np.diag(probe))
        with np.errstate(divide='ignore', invalid='ignore'):
            k = np.where(probe[:, None] != 0, out / probe[:, None], 0.0)
        assert k.shape[0] == n_in
        return k.astype(np.float32)

    @property
    def kernel(self):
        """The constant matrix this cascade implements = product of the stage kernels (reference ``Pipeline.kernel``,
        types.py:627-629), computed from GPU replays instead of the interpreted float replay."""
        k = self.stage_kernel(0)
        for i in range(1, len(self.stages)):
            k = k @ self.stage_kernel(i)
        return k


def solve_raw(kernel, method0='wmc', method1='auto', hard_dc=-1, decompose_dc=-2, qintervals=None, latencies=None,
              adder_size=-1, carry_size=-1, search_all_decompose_dc=True, seed=0) -> RawPipeline:
    k = _kernel_arg(kernel)
    q = _qint_arg(qintervals, k.shape[0])
    l = _lat_arg(latencies, k.shape[0])
    s = _seed_arg(seed)
    h = _vp()
    _check(_L.da4ml_cmvm_solve_seeded(_fp(k), k.shape[0], k.shape[1], method0.encode(), method1.encode(), hard_dc, decompose_dc, _fp(q), _fp(l), adder_size, carry_size,
                                      int(bool(search_all_decompose_dc)), s, C.byref(h)))  # fmt: skip
    return RawPipeline(h)


def solve(kernel, method0='wmc', method1='auto', hard_dc=-1, decompose_dc=-2, qintervals=None, latencies=None,
          adder_size=-1, carry_size=-1, search_all_decompose_dc=True, seed=0):
    """``da4ml._binary.cmvm_bin.solve`` (bindings.cc:235-248): returns a ``Pipeline`` of two ``CombLogic`` stages.

    ``seed`` (this library's extension, an integer in [0, 2**64)) picks the tie-break order of the greedy pair selection:
    among pairs of equal score the one whose packed key XOR ``tb_mask(seed)`` is largest.  Seed 0 is the reference's
    order, so ``seed=0`` gives the reference's result; another seed is an equally valid greedy run whose graph may cost
    more or less.  ``solve_best_of`` keeps the cheapest of many seeds."""
    return solve_raw(kernel, method0, method1, hard_dc, decompose_dc, qintervals, latencies, adder_size, carry_size, search_all_decompose_dc, seed).to_pipeline()


def solve_batch_raw(kernels, method0='wmc', method1='auto', hard_dc=-1, decompose_dc=-2, qintervals=None, latencies=None,
                    adder_size=-1, carry_size=-1, search_all_decompose_dc=True) -> list[RawPipeline]:
    ks = [_kernel_arg(k) for k in kernels]
    n = len(ks)
    if n == 0:
        return []
    qs = [_qint_arg(qintervals[i], ks[i].shape[0]) if qintervals is not None else None for i in range(n)]
    ls = [_lat_arg(latencies[i], ks[i].shape[0]) if latencies is not None else None for i in range(n)]
    kp = (_f32p * n)(*[_fp(k) for k in ks])
    qp = (_f32p * n)(*[_fp(q) for q in qs])
    lp = (_f32p * n)(*[_fp(l) for l in ls])
    n_in = np.asarray([k.shape[0] for k in ks], np.int64)
    n_out = np.asarray([k.shape[1] for k in ks], np.int64)
    hs = (_vp * n)()
    _check(_L.da4ml_cmvm_solve_batch(n, kp, _ip(n_in), _ip(n_out), method0.encode(), method1.encode(), hard_dc, decompose_dc, qp, lp, adder_size, carry_size, int(bool(search_all_decompose_dc)), hs))
    return [RawPipeline(_vp(h)) for h in hs]


def solve_batch_device_raw(dev_ptrs, shapes, method0='wmc', method1='auto', hard_dc=-1, decompose_dc=-2, adder_size=-1,
                           carry_size=-1, search_all_decompose_dc=True) -> list[RawPipeline]:
    """Batch solve of matrices already resident in device memory: ``dev_ptrs[i]`` is the address of a dense
    float32 ``shapes[i] = (n_in, n_out)`` array on the current CUDA device (e.g. ``tensor.data_ptr()``)."""
    n = len(dev_ptrs)
    kp = (_vp * n)(*[_vp(int(p)) for p in dev_ptrs])
    n_in = np.asarray([s[0] for s in shapes], np.int64)
    n_out = np.asarray([s[1] for s in shapes], np.int64)
    hs = (_vp * n)()
    _check(_L.da4ml_cmvm_solve_batch_device(n, kp, _ip(n_in), _ip(n_out), method0.encode(), method1.encode(), hard_dc, decompose_dc, None, None, adder_size, carry_size, int(bool(search_all_decompose_dc)), hs))
    return [RawPipeline(_vp(h)) for h in hs]


def solve_batch(kernels, **kw):
    """Solve many independent constant matrices in one GPU pass; list of ``Pipeline``."""
    return [r.to_pipeline() for r in solve_batch_raw(kernels, **kw)]


def solve_single_raw(kernel, method='wmc', qintervals=None, latencies=None, adder_size=-1, carry_size=-1, trace_cap=0, seed=0):
    """One CSE stage (reference ``solve_single``, cmvm_core.cc:227).  Returns (RawPipeline, trace[n,5] or None).
    ``seed``: the tie-break order of ``solve``."""
    k = _kernel_arg(kernel)
    q = _qint_arg(qintervals, k.shape[0])
    l = _lat_arg(latencies, k.shape[0])
    s = _seed_arg(seed)
    tr = np.zeros((max(trace_cap, 1), 5), np.int32)
    h = _vp()
    _check(_L.da4ml_cmvm_solve_single_seeded(_fp(k), k.shape[0], k.shape[1], method.encode(), _fp(q), _fp(l), adder_size, carry_size,
                                             tr.ctypes.data_as(_i32p) if trace_cap > 0 else None, trace_cap, s, C.byref(h)))  # fmt: skip
    raw = RawPipeline(h)
    return raw, (tr[: min(trace_cap, raw.counters[0]['T'])] if trace_cap > 0 else None)


METHODS = ['mc', 'mc-dc', 'mc-pdc', 'wmc', 'wmc-dc', 'wmc-pdc', 'dummy']  # the library's method codes
SWEEP_SET_DEFAULTS = dict(method0='wmc', method1='auto', hard_dc=-1, decompose_dc=-2, search_all_decompose_dc=True, seed=0)  # as solve()
_SWEEP_INT_FIELDS = ['set', 'hard_dc', 'decompose_dc_start', 'method0', 'method1', 'decompose_dc', 'n_adders', 'n_ops0', 'n_ops1', 'winner', 'front', 'kept']
_SWEEP_FLOAT_FIELDS = ['cost', 'latency_min', 'latency_max']


def sweep_front(cost, latency_max) -> np.ndarray:
    """Indices of the candidates no other candidate dominates on ``(cost, latency_max)`` (<= on both, < on one); of
    exactly equal points only the first.  The rule ``solve_sweep`` applies, on the host (no device needed)."""
    c = np.ascontiguousarray(cost, dtype=np.float32).ravel()
    l = np.ascontiguousarray(latency_max, dtype=np.float32).ravel()
    if c.shape != l.shape:
        raise ValueError(f'cost and latency_max differ in length ({c.size} != {l.size})')
    f = np.zeros(c.size, np.int8)
    _check(_L.da4ml_sweep_front(_fp(c), _fp(l), c.size, f.ctypes.data_as(_i8p)))
    return np.flatnonzero(f)


class SweepResult:
    """One matrix solved under many option sets (``solve_sweep``).

    ``candidates`` holds one numpy array per field, one entry per candidate (set order, then ``decompose_dc`` order):
    ``set``, ``hard_dc`` and ``decompose_dc_start`` (the H and d its ``_solve`` started with), ``method0`` / ``method1``
    (after the ``method1='auto'`` and ``hard_dc=0`` rules and any forced ``wmc-dc`` retry), the final ``decompose_dc``,
    ``cost`` (float32, summed over both stages in op order, the value the argmin uses), ``n_adders``, ``latency_min`` /
    ``latency_max`` (``Pipeline.latency``), ``n_ops0`` / ``n_ops1``, and the flags ``winner``, ``front``, ``kept`` (op
    tables available through ``raw`` / ``pipeline``).  ``front`` and ``winners`` are index arrays; ``winners[s]`` is set
    ``s``'s result, what ``solve(kernel, **option_sets[s])`` returns.

    A result pickles (``torch.distributed`` gathers, multiprocessing, files): the copy holds the candidate arrays and the
    op tables of the kept candidates, and no library handle, and answers every method as the original does."""

    def __init__(self, handle, kernel, option_sets, qintervals, latencies, adder_size, carry_size):
        self._h = handle
        self._kept = None  # {candidate: RawPipeline} once detached from the library by pickling
        self.kernel, self.option_sets = kernel, option_sets
        self._call = dict(qintervals=qintervals, latencies=latencies, adder_size=adder_size, carry_size=carry_size)
        cnt = np.zeros(4, np.int64)
        _check(_L.da4ml_sweep_counts(handle, _ip(cnt)))
        self.n_sets, n, self.n_kept, self.n_solved = (int(v) for v in cnt)
        ints = np.zeros((n, len(_SWEEP_INT_FIELDS)), np.int64)
        floats = np.zeros((n, len(_SWEEP_FLOAT_FIELDS)), np.float32)
        _check(_L.da4ml_sweep_summary(handle, _ip(ints), _fp(floats)))
        cand = {k: ints[:, i].copy() for i, k in enumerate(_SWEEP_INT_FIELDS)}
        for k in ('method0', 'method1'):
            cand[k] = np.asarray(METHODS, dtype=object)[cand[k]].astype(str)
        for k in ('winner', 'front', 'kept'):
            cand[k] = cand[k].astype(bool)
        cand.update({k: floats[:, i].copy() for i, k in enumerate(_SWEEP_FLOAT_FIELDS)})
        self.candidates = cand
        self.front = np.flatnonzero(cand['front'])
        self.winners = np.asarray([int(np.flatnonzero(cand['winner'] & (cand['set'] == s))[0]) for s in range(self.n_sets)], np.int64)
        prof = (C.c_double * 8)()
        _check(_L.da4ml_sweep_profile(handle, prof))
        self.profile = dict(device_ms=prof[0], launches=int(prof[1]), solve_kernel_ms=prof[2], solve_kernel_launches=int(prof[3]), algo_bytes=prof[4],
                            jobs_total=int(prof[5]), jobs_run=int(prof[6]), solve_retries=int(prof[7]), candidates=n, candidates_solved=self.n_solved, candidates_kept=self.n_kept)

    def __len__(self):
        return len(self.candidates['set'])

    def __del__(self):
        h, self._h = getattr(self, '_h', None), None
        if h:
            _L.da4ml_sweep_free(h)

    def __getstate__(self):
        st = {k: v for k, v in self.__dict__.items() if k != '_h'}
        if self._h:
            st['_kept'] = {int(i): self.raw(i) for i in np.flatnonzero(self.candidates['kept'])}
        return st

    def __setstate__(self, st):
        self.__dict__.update(st)
        self._h = None

    def raw(self, i: int) -> RawPipeline:
        """Candidate ``i`` as a ``RawPipeline``; ``ValueError`` when its op tables were not kept."""
        if self._h:
            h = _vp()
            _check(_L.da4ml_sweep_pipeline(self._h, int(i), C.byref(h)))
            return RawPipeline(h)
        i, n = int(i), len(self)  # (a pickled copy: the library's checks and messages)
        if not 0 <= i < n:
            raise ValueError(f'sweep_pipeline: candidate {i} is out of range [0, {n})')
        if i not in self._kept:
            raise ValueError(f'sweep_pipeline: the op tables of candidate {i} were not kept (only the winners and the front are, unless the sweep was run with keep_all)')
        return copy.deepcopy(self._kept[i])

    def pipeline(self, i: int, types_module=None):
        return self.raw(i).to_pipeline(types_module)

    def reference_call(self, i: int) -> dict:
        """Keyword arguments of the ``solve(kernel, **kw)`` call whose result candidate ``i`` is.  A candidate of a set with
        a non-zero ``seed`` gets a ``seed`` keyword: that call is one of this library's ``solve``, which the reference's
        has no counterpart for."""
        c = self.candidates
        s = {**SWEEP_SET_DEFAULTS, **self.option_sets[int(c['set'][i])]}
        call = dict(method0=s['method0'], method1=s['method1'], hard_dc=int(c['hard_dc'][i]), decompose_dc=int(c['decompose_dc_start'][i]),
                    search_all_decompose_dc=False, **self._call)
        if int(s['seed']):
            call['seed'] = int(s['seed'])
        return call

    def pipelined(self, latency_cutoff, retiming: bool = True, pricer=None, keep_split: bool = False) -> 'PipelinePrice':
        """``price_pipelined`` of every candidate whose op tables were kept, under the sweep's own input latencies, in one
        call.  The arrays are aligned with ``candidates`` (``[len(self), n_cutoffs]``); a candidate that was not kept has
        status -1, ``stages`` / ``reg_bits`` -1 and NaN latencies.  Only the winners and the front are kept unless the
        sweep ran with ``keep_all=True``, which is needed to price every candidate.  ``pricer`` stands in for
        ``price_pipelined``.  ``keep_split=True``: ``split(i, j)`` gives candidate ``i``'s register stages under cutoff
        ``j``."""
        kept = np.flatnonzero(self.candidates['kept'])
        lat = self._call['latencies']
        kw = dict(keep_split=True) if keep_split else {}
        pr = (price_pipelined if pricer is None else pricer)([self.raw(int(i)) for i in kept], latency_cutoff, latencies=None if lat is None else [lat] * kept.size,
                                                             retiming=retiming, **kw)  # fmt: skip
        return pr._scatter(kept, len(self))


def _prefixed(tag, f, *args, **kw):
    try:
        return f(*args, **kw)
    except (TypeError, ValueError, RuntimeError) as e:
        raise type(e)(f'{tag}: {e}') from None


def _sweep_sets(option_sets) -> list[dict]:
    sets = [dict(s) for s in option_sets]
    for s in sets:
        bad = set(s) - set(SWEEP_SET_DEFAULTS)
        if bad:
            raise TypeError(f'unsupported keys in a sweep option set: {sorted(bad)} (adder_size / carry_size are arguments of the sweep itself)')
        if 'seed' in s:
            s['seed'] = _seed_arg(s['seed'])
    return sets


def solve_sweep_batch(kernels, option_sets, qintervals=None, latencies=None, adder_size=-1, carry_size=-1, keep_all=False) -> list[SweepResult]:
    """Solve every matrix of ``kernels`` under every option set of ``option_sets`` in one GPU pass (a model's layers,
    say): every pending ``solve_single`` of every candidate of every matrix runs in one launch per round.

    ``qintervals`` / ``latencies`` are per-matrix lists, as for ``solve_batch_raw``.  The option sets and the cost model
    (``adder_size``, ``carry_size``) are shared by all matrices, so costs of different matrices can be summed.  Result
    ``p`` is what ``solve_sweep(kernels[p], option_sets, ...)`` returns (its ``profile`` is the whole call's).  If any set
    fails on any matrix, the call raises ``solve``'s error and returns nothing."""
    named = (lambda i, f, *args: _prefixed(f'matrix {i}', f, *args)) if len(kernels) > 1 else (lambda i, f, *args: f(*args))  # (a lone matrix needs no name)
    ks = [named(i, _kernel_arg, k) for i, k in enumerate(kernels)]
    n = len(ks)
    sets = _sweep_sets(option_sets)
    for name, v in (('qintervals', qintervals), ('latencies', latencies)):
        if v is not None and len(v) != n:
            raise ValueError(f'expected {name} for {n} matrices, got {len(v)}')
    qs = [named(i, _qint_arg, qintervals[i], ks[i].shape[0]) if qintervals is not None else None for i in range(n)]
    ls = [named(i, _lat_arg, latencies[i], ks[i].shape[0]) if latencies is not None else None for i in range(n)]
    if n == 0:
        return []
    full = [{**SWEEP_SET_DEFAULTS, **s} for s in sets]
    m = len(full)
    m0 = (C.c_char_p * max(m, 1))(*[str(s['method0']).encode() for s in full])
    m1 = (C.c_char_p * max(m, 1))(*[str(s['method1']).encode() for s in full])
    hdc = np.asarray([int(s['hard_dc']) for s in full] or [0], np.int32)
    ddc = np.asarray([int(s['decompose_dc']) for s in full] or [0], np.int32)
    sa = np.asarray([int(bool(s['search_all_decompose_dc'])) for s in full] or [0], np.int32)
    sd = (C.c_uint64 * max(m, 1))(*[int(s['seed']) for s in full])
    kp = (_f32p * n)(*[_fp(k) for k in ks])
    qp = (_f32p * n)(*[_fp(q) for q in qs])
    lp = (_f32p * n)(*[_fp(l) for l in ls])
    n_in = np.asarray([k.shape[0] for k in ks], np.int64)
    n_out = np.asarray([k.shape[1] for k in ks], np.int64)
    hs = (_vp * n)()
    i32 = lambda a: a.ctypes.data_as(_i32p)  # noqa: E731
    _check(_L.da4ml_cmvm_solve_sweep_batch_seeded(n, kp, _ip(n_in), _ip(n_out), qp, lp, int(adder_size), int(carry_size), m, m0, m1, i32(hdc), i32(ddc), i32(sa), sd,
                                                  int(bool(keep_all)), hs))  # fmt: skip
    return [SweepResult(_vp(h), k, [dict(s) for s in sets], None if q is None else [tuple(map(float, r)) for r in q], None if l is None else [float(v) for v in l],
                        int(adder_size), int(carry_size)) for h, k, q, l in zip(hs, ks, qs, ls)]


def solve_sweep(kernel, option_sets, qintervals=None, latencies=None, adder_size=-1, carry_size=-1, keep_all=False) -> SweepResult:
    """Solve one matrix under every option set of ``option_sets`` in one GPU pass.

    Each option set is a dict of ``solve`` keywords (``method0, method1, hard_dc, decompose_dc,
    search_all_decompose_dc, seed``; missing keys take ``solve``'s defaults).  Sets that differ only in ``seed`` are
    distinct candidates.  The intervals, latencies and the cost model
    (``adder_size``, ``carry_size``) are shared by all sets: costs under different cost models are not comparable.
    Op tables come back for the winners and the front, or for every candidate with ``keep_all``.  The batch of one
    matrix of ``solve_sweep_batch``."""
    return solve_sweep_batch([kernel], option_sets, None if qintervals is None else [qintervals], None if latencies is None else [latencies], adder_size, carry_size,
                             keep_all)[0]


_SWEEP_CALL_KEYS = ('qintervals', 'latencies', 'adder_size', 'carry_size')  # solve() keywords that are arguments of a sweep


def solve_best_of_raw(kernel, n_seeds=16, solver=None, **solve_kwargs) -> tuple[RawPipeline, int]:
    """``solve_best_of`` as a ``RawPipeline``: ``(result, seed)``."""
    if isinstance(n_seeds, bool) or not isinstance(n_seeds, (int, np.integer)) or n_seeds < 1:
        raise ValueError(f'n_seeds must be a positive integer, got {n_seeds!r}')
    if 'seed' in solve_kwargs:
        raise TypeError('solve_best_of tries the seeds 0 .. n_seeds - 1 itself: it takes no seed keyword')
    call = {k: solve_kwargs.pop(k) for k in _SWEEP_CALL_KEYS if k in solve_kwargs}
    sets = [{**solve_kwargs, 'seed': s} for s in range(int(n_seeds))]
    sw = (solve_sweep if solver is None else solver)(kernel, sets, **call)
    winners = np.asarray(sw.winners, np.int64)
    s = int(np.argmin(np.asarray(sw.candidates['cost'], np.float32)[winners]))  # (the first minimum: ties go to the lowest seed)
    return sw.raw(int(winners[s])), s


def solve_best_of(kernel, n_seeds=16, types_module=None, solver=None, **solve_kwargs):
    """Best of ``n_seeds`` tie-break orders: ``solve(kernel, **solve_kwargs, seed=s)`` for ``s = 0 .. n_seeds - 1`` in one
    GPU pass (a ``solve_sweep`` of one option set per seed), and the cheapest result.  Returns ``(Pipeline, seed)``.

    Cost is ``SweepResult``'s float32 ``cost``; of equal costs the lowest seed wins, so the result is never costlier
    than ``solve(kernel, **solve_kwargs)`` (seed 0) and is that result when no seed does better.  The returned design is
    bit for bit what ``solve(kernel, **solve_kwargs, seed=seed)`` returns.  Every seed's greedy run is a valid run of the
    same algorithm; a seed's graph is about as likely to be worse than seed 0's as better, and the gain is in keeping the
    cheapest.  ``solver(kernel, option_sets, **kw)`` stands in for ``solve_sweep`` (same keywords and result)."""
    raw, seed = solve_best_of_raw(kernel, n_seeds, solver, **solve_kwargs)
    return raw.to_pipeline(types_module), seed


NetworkPoint = namedtuple('NetworkPoint', ['cost', 'latency', 'choice'])


class NetworkFront:
    """The cost / latency front of a chain of layers (``network_front``).  ``cost`` and ``latency`` are float32 arrays
    sorted by ascending latency; ``choice[p, k]`` is the candidate of layer ``k``'s sweep that point ``p`` uses."""

    def __init__(self, cost, latency, choice):
        self.cost, self.latency, self.choice = cost, latency, choice

    def __len__(self):
        return len(self.cost)

    def best(self, latency_budget) -> NetworkPoint:
        """The cheapest point whose latency is at most ``latency_budget`` (the first of equal ones); ``ValueError`` when
        every point is slower."""
        ok = np.flatnonzero(self.latency.astype(np.float64) <= float(latency_budget))
        if ok.size == 0:
            raise ValueError(f'no design of the network meets a latency budget of {latency_budget} (the fastest has latency {float(self.latency[0])})')
        p = int(ok[np.argmin(self.cost[ok])])
        return NetworkPoint(float(self.cost[p]), float(self.latency[p]), tuple(int(c) for c in self.choice[p]))


def network_front(sweeps) -> NetworkFront:
    """Combine the sweeps of a chain of layers (``sweeps[k]`` of layer ``k``, in order) into the network's front.

    A point takes one candidate per layer from that layer's ``front``; its cost and latency are the float32 sums, in
    layer order, of the layers' ``cost`` and ``latency_max``.  The combinations are built layer by layer, in
    lexicographic order of the per-layer choices, and pruned after each layer with the ``sweep_front`` rule (of exactly
    equal points the first is kept).  Every chosen candidate is on its layer's front, so its op tables are kept.

    Latency model: each layer is swept with its input latencies counted from its own inputs (zeros by default).  An op's
    latency is max-plus monotone in its operands' latencies, so shifting every input of a layer by t shifts each of its
    outputs by at most t; the sum of the chosen graphs' ``latency_max`` therefore bounds the chain's adder depth from
    the network inputs.  Branching networks are not covered."""
    sweeps = list(sweeps)
    if not sweeps:
        raise ValueError('network_front needs the sweep of at least one layer')
    cost = lat = choice = None
    for sw in sweeps:
        f = np.asarray(sw.front, np.int64)
        c = np.asarray(sw.candidates['cost'], np.float32)[f]
        l = np.asarray(sw.candidates['latency_max'], np.float32)[f]
        if choice is None:
            cost, lat, choice = c, l, f[:, None]
        else:  # every (point so far, front candidate) pair, in lexicographic order of the choices
            cost = (cost[:, None] + c[None, :]).ravel()
            lat = (lat[:, None] + l[None, :]).ravel()
            choice = np.concatenate([np.repeat(choice, f.size, axis=0), np.tile(f, len(choice))[:, None]], axis=1)
        keep = sweep_front(cost, lat)
        cost, lat, choice = cost[keep], lat[keep], choice[keep]
    order = np.argsort(lat, kind='stable')
    return NetworkFront(cost[order], lat[order], choice[order])


def _out_latencies(raw) -> np.ndarray:
    """Latency of each output of a result (float32, ``CombLogic.out_latency`` of its last stage): the op latency at each
    ``out_idx``, and 0.0 for a column with ``out_idx == -1`` (a constant zero)."""
    last = raw.stages[-1]
    idx = np.asarray(last['out_idxs'], np.int64)
    lat = np.asarray(last['ops_f'], np.float32).reshape(-1, 5)[:, 3]
    out = np.zeros(idx.size, np.float32)
    out[idx >= 0] = lat[idx[idx >= 0]]
    return out


class ChainFront(NetworkFront):
    """The cost / latency front of a chain of layers, each solved under the output latencies of the one before it
    (``chain_front``).  ``cost`` and ``latency`` are float32 arrays sorted by ascending latency; ``choice[p, k]`` is the
    candidate that point ``p`` takes at layer ``k``, an index into the sweep of that layer under the point's own input
    latencies.  ``best(latency_budget)`` is ``NetworkFront.best``.  ``profile`` holds the sweeps' launches, device time
    and jobs, in total and per layer (``layers[k]``: input-latency states, candidates, points kept, ...).

    ``activations``: the relu / quantizers between the layers that the front was searched with (``chain_front(...,
    activations=...)``, each as ``(kind, [n_out, 3] kif)``), or ``None``.  ``biases``: its per-layer biases (``None`` or
    ``[n_out]`` float64 each), or ``None`` when it was searched without a non-zero one.

    Only host arrays are held (each point's designs are ``RawPipeline`` copies), so a front pickles as it is."""

    activations = None  # (a front built without activations holds no attribute of its own: it pickles as before)
    biases = None  # (likewise without biases)

    def __init__(self, cost, latency, choice, raws, calls, profile, latency_cutoff=0.0, activations=None, biases=None):
        super().__init__(cost, latency, choice)
        self._raws, self._calls, self.profile = raws, calls, profile
        self.latency_cutoff = float(latency_cutoff)
        if activations is not None:
            self.activations = activations
        if biases is not None:
            self.biases = biases
        c = self.latency_cutoff
        # (to_pipeline's stage of the last output, + 1: the clock count of a chain whose network inputs arrive before c)
        self.stages = (np.floor(np.asarray(latency, np.float64) / (c + 1e-9)).astype(np.int64) + 1) if c > 0 else np.ones(len(cost), np.int64)

    def best_stages(self, n_stages) -> NetworkPoint:
        """The cheapest point with at most ``n_stages`` register stages (the first of equal ones); ``ValueError`` when
        every point needs more."""
        ok = np.flatnonzero(self.stages <= int(n_stages))
        if ok.size == 0:
            raise ValueError(f'no design of the network fits in {n_stages} stages (the fastest needs {int(self.stages.min())})')
        p = int(ok[np.argmin(self.cost[ok])])
        return NetworkPoint(float(self.cost[p]), float(self.latency[p]), tuple(int(c) for c in self.choice[p]))

    def raw(self, p: int, k: int) -> RawPipeline:
        """Layer ``k``'s design in point ``p``."""
        return copy.deepcopy(self._raws[p][k])

    def pipelines(self, p: int, types_module=None) -> list:
        """Point ``p``'s designs as one ``Pipeline`` per layer."""
        return [r.to_pipeline(types_module) for r in self._raws[p]]

    def design(self, p: int, activations=None, biases=None) -> RawPipeline:
        """Point ``p``'s designs as one chain design with ``activations`` between the layers: ``chain_design(self.pipelines(p),
        activations, biases)``, for ``price_pipelined`` (register bits, ``keep_split``).  A front searched with activations uses its
        own when none are given, and refuses others (``ValueError``): its later layers were solved for its own.  A front
        searched without them needs them.  Biases likewise: the front's own are used, and other non-zero ones are refused."""
        if biases is not None or self.biases is not None:
            n_outs = [int(r.stages[-1]['shape'][1]) for r in self._raws[p]]
            mine = self.biases or [None] * len(n_outs)
            theirs = mine if biases is None else (_biases_arg(biases, n_outs) or [None] * len(n_outs))
            if any((a is None) != (b is None) or (a is not None and not np.array_equal(a, b)) for a, b in zip(mine, theirs)):
                raise ValueError('these biases differ from the ones the front was searched with: its later layers were solved for those')
        if activations is None:
            if self.activations is None:
                raise TypeError('this front was searched without activations: design(p, activations) needs them')
            activations = [[_act_tuple(a) for a in seq] for seq in self.activations]
        elif self.activations is not None:
            acts = list(activations)
            n_outs = [int(r.stages[-1]['shape'][1]) for r in self._raws[p]]
            same = len(acts) == len(self.activations)
            for k, (act, mine) in enumerate(zip(acts, self.activations) if same else ()):
                r = _same_acts(_act_seq(k, act, n_outs[k]), mine)
                if r is False:  # (kinds, kifs or modes differ: no table comparison can make them the same)
                    same = False
                    break
                if r is None:
                    same = None
            if same is None:  # only the 'apply' functions differ: the same tables are the same activations
                mine = [[_act_tuple(a) for a in seq] for seq in self.activations]
                a, b = chain_design(self._raws[p], activations, self.biases), chain_design(self._raws[p], mine, self.biases)
                same = len(a.stages) == len(b.stages) and all(_same_tables(x.get('lookup_tables'), y.get('lookup_tables')) for x, y in zip(a.stages, b.stages))
            if not same:
                raise ValueError('these activations differ from the ones the front was searched with: its later layers were solved for those')
        return chain_design(self._raws[p], activations, self.biases)

    def reference_calls(self, p: int) -> list[dict]:
        """Per layer, the keywords of the ``solve(kernels[k], **kw)`` call that returns layer ``k``'s design in point
        ``p``: the candidate's options, the layer's ``qintervals`` and its input ``latencies`` as Python floats (for
        ``k > 0``, the output latencies of the point's design of layer ``k - 1``).  With activations, ``qintervals`` of
        ``k > 0`` are the intervals of layer ``k - 1``'s traced outputs after the activation, as the float32 values the
        layer was solved under.  A candidate of a seeded option set carries its ``seed``, as ``SweepResult.reference_call``
        does."""
        return copy.deepcopy(self._calls[p])


def _chain_layer(points, state_of, sweeps, state_lats, traced=None, state_qs=None, acted=None, cutoff=0.0):
    """Extend the points of the layers so far by the next layer and prune.  ``points`` is ``None`` at layer 0, else
    ``(cost, lat, choice, outs, raws, calls)``; ``state_of[p]`` is the index of point ``p``'s input-latency state in
    ``sweeps`` and ``state_lats`` (lists of Python floats); at layer 0 there is one state and ``state_of == [0]``.
    Parents are taken in order and each is extended by every ``front`` candidate of its state's sweep, in candidate
    order; cost is the float32 sum in layer order, latency the new design's ``latency_max``; then the ``sweep_front``
    rule.  ``outs[p]`` are the output latencies of point ``p``'s last design.  ``traced[s, i]`` (pipelined chains):
    ``(latency_max, output latencies)`` of front candidate ``i`` of state ``s`` as traced under the cutoff, which replace the
    solver's; a front candidate without an entry is dropped.

    Chains with activations: ``state_qs[s]`` are state ``s``'s qintervals for the reference calls, and ``acted`` is
    ``(group_of, table, ...)`` at every layer but the last (and at the last when it has a bias): ``group_of[p]`` is parent ``p``'s replay group (the parents of one state with the same float64
    input intervals); ``table[g, i]`` is ``None`` when candidate ``i`` under group ``g`` makes a non-zero constant (the
    pair is dropped), else ``(act_cost, zero, intervals, views, dls)``: the float32 cost of each op of the bias /
    activation stage in stage order (with a bias: each output's constant addition, then each activation's op of each
    output; 0 without one), which outputs become the constant 0, the outputs' intervals after the bias and activations,
    their ``[n, 2]`` (factor, cadd) of ``_traced_views``, and per output its latency steps in order (a lookup's increment, or a leaky
    ReLU's (condition dlat, mux dlat), applied at ``cutoff`` by ``_act_latency``).  A point's cost then continues with ``act_cost`` added in order, and
    its ``outs`` entry is ``(latencies, intervals, views)``, the latency of a constant 0 being 0."""
    fronts = [np.asarray(sw.front, np.int64) for sw in sweeps]
    if traced is not None:
        fronts = [np.asarray([i for i in f.tolist() if (s, i) in traced], np.int64) for s, f in enumerate(fronts)]
    f_cost = [np.asarray(sw.candidates['cost'], np.float32)[f] for sw, f in zip(sweeps, fronts)]
    if traced is None:
        f_lat = [np.asarray(sw.candidates['latency_max'], np.float32)[f] for sw, f in zip(sweeps, fronts)]
    else:
        f_lat = [np.asarray([traced[s, i][0] for i in f.tolist()], np.float64) for s, f in enumerate(fronts)]
    par = np.concatenate([np.full(fronts[s].size, p, np.int64) for p, s in enumerate(state_of)])
    sidx = np.concatenate([np.full(fronts[s].size, s, np.int64) for s in state_of])
    cand = np.concatenate([fronts[s] for s in state_of])
    cost = np.concatenate([f_cost[s] for s in state_of])
    lat = np.concatenate([f_lat[s] for s in state_of])
    if acted is not None:
        group_of, table = acted[:2]
        ok = np.asarray([table[group_of[p], i] is not None for p, i in zip(par.tolist(), cand.tolist())], bool).reshape(-1)
        par, sidx, cand, cost, lat = par[ok], sidx[ok], cand[ok], cost[ok], lat[ok]
    if points is not None:
        cost = points[0][par] + cost
    if acted is not None and par.size:
        act_cost = np.stack([table[group_of[p], i][0] for p, i in zip(par.tolist(), cand.tolist())])
        for j in range(act_cost.shape[1]):  # (float32, in output order: the order of the activation stage's ops)
            cost = cost + act_cost[:, j]
    keep = sweep_front(cost, lat)
    par, sidx, cand, cost, lat = par[keep], sidx[keep], cand[keep], cost[keep], lat[keep]
    choice = cand[:, None] if points is None else np.concatenate([points[2][par], cand[:, None]], axis=1)
    designs = {}  # (state, candidate) -> (RawPipeline, solve() keywords, output latencies), shared by the points using it
    raws, calls, outs = [], [], []
    for p, s, i in zip(par.tolist(), sidx.tolist(), cand.tolist()):
        if (s, i) not in designs:
            r = sweeps[s].raw(i)
            call = {**sweeps[s].reference_call(i), 'latencies': state_lats[s]}
            if state_qs is not None:
                call['qintervals'] = state_qs[s]
            designs[s, i] = (r, call, _out_latencies(r) if traced is None else traced[s, i][1])
        r, call, o = designs[s, i]
        raws.append([r] if points is None else [*points[4][p], r])
        calls.append([call] if points is None else [*points[5][p], call])
        if acted is not None:
            _, zero, vals, aux, dls = table[group_of[p], i]
            o = np.asarray(o).copy()
            for j, dl in enumerate(dls):  # lookups and leaky ReLUs, in order (_act_latency)
                for d in dl:
                    o[j] = _act_latency(float(o[j]), d, cutoff) if isinstance(d, tuple) else d + o[j]
            o = (np.where(zero, 0.0, o).astype(o.dtype), vals, aux)
        outs.append(o)
    return cost, lat, choice, outs, raws, calls


def chain_front(kernels, option_sets, qintervals=None, latencies=None, adder_size=-1, carry_size=-1, solver=None, latency_cutoff=0.0, pricer=None,
                activations=None, biases=None) -> ChainFront:
    """The cost / latency front of a chain of layers, each layer solved under the output latencies of the design chosen
    for the layer before it, as a traced model's matmuls are: every reported design is what
    ``solve(kernels[k], **front.reference_calls(p)[k])`` returns, and every reported cost and latency is the chain's own.

    ``kernels[k]`` is layer ``k``'s constant matrix (``kernels[k].shape[1] == kernels[k + 1].shape[0]``).
    ``option_sets`` and the cost model (``adder_size``, ``carry_size``) are those of ``solve_sweep`` and the same for
    every layer.  ``qintervals`` is ``None`` or one entry per layer: ``None`` (``solve``'s default) or that layer's input
    intervals, e.g. those of the quantizer in front of it; without ``activations``, intervals are not carried over from a
    layer's outputs.  ``latencies`` are layer 0's input latencies (default zeros).

    ``activations[k]`` (``len(kernels) - 1`` of them, in ``chain_design``'s format: ``('relu' | 'quantize', kif[, 'TRN'[,
    'WRAP']])``, ``('apply', fn, kif[, round_mode[, overflow_mode]])``, ``('leaky_relu', alpha)``, or a non-empty list of
    these applied in order) is
    the op between layer ``k`` and layer ``k + 1``.  With them every layer after the first is solved under
    the intervals a traced model hands it: those of the previous design's traced outputs after the activation (the
    intervals ``chain_design`` gives the activation stage's outputs).  A dead column, or a value that loses all its bits, is
    the tracer's constant 0: the interval (0, 0, 2**32) at latency 0.  Only ``qintervals[0]`` may then be given (``ValueError`` otherwise).

    Search: layer 0 is swept once, and its ``front`` candidates are the first points.  At each later layer a point's
    input-latency state is the output latencies of its last design (``Pipeline.out_latencies``; 0.0 for a constant-zero
    output), with activations together with its activated intervals; points whose states are equal as float32 (the values
    the solver sees) share one problem, and all the layer's states go into one ``solver`` call (``solve_sweep_batch``:
    one GPU pass per layer, each state with its own ``qintervals``).  Each point is extended by every ``front`` candidate
    of its state's sweep; its cost is the float32 sum of the designs' costs in layer order, and its latency the new
    design's ``latency_max``, which already contains the upstream latency.  With activations the cost is the float32 sum,
    in stage order, of the ``ops_f`` cost column of the point's chain design (``design(p)``): each layer design's cost
    followed by the cost of each op of the activation after it, in output order (relu: ``sum(kif) / 2`` per changed
    value, quantize: 0).  A (state, candidate) pair whose activation turns some output into a non-zero constant is
    dropped (``profile['layers'][k]['dropped_constant']``; ``replay_ms`` is the host time of the interval replay).  The
    points are pruned after each layer with the ``sweep_front`` rule, and the result is sorted by ascending latency.

    Latency model: with ``latency_cutoff = 0`` (the default) latency is the solver's op latency.  With ``latency_cutoff =
    c > 0`` it is the latency the tracer gives the design under ``HWConfig(adder_size, carry_size, c)``: after each
    layer's sweep every front candidate of every state is priced under that state's latencies (``price_pipelined``
    without retiming, one call per layer); a point's latency is the traced ``latency_max``, its next state the traced
    output latencies (what the traced model hands the next ``solve``), pruning uses (cost, traced latency), and a
    candidate whose status is not ok (an adder slower than ``c``) is dropped (``profile['layers'][k]['dropped']``).
    ``stages[p] = floor(latency / (c + 1e-9)) + 1`` is the clock count ``to_pipeline`` gives the chain when its network
    inputs arrive before ``c``; ``retime_pipeline`` never accepts a split with more stages, so retiming never adds a
    clock.  ``best_stages(n)`` is the cheapest point with at most ``n`` stages.  A point's register bits and register
    stages as one pipeline, with the activations between its layers, are ``price_pipelined(front.design(p,
    activations), c, keep_split=True)`` (``chain_design``).
    ``relu`` and ``quantize`` add no latency, as ``relu`` and ``wrap`` in the tracer keep their input's latency; a lookup
    (``'apply'``) adds the tracer's ``max(b_in - 6, 1)`` to its operand's latency, with no register-boundary rule, and
    the next layer's state latencies (and, with a cutoff, the traced ones) include it.  The
    front is the front of the chains explored: the solver is not monotone in its input latencies, so pruning partial
    chains on (cost, latency) is a heuristic and a pruned chain could have led to a better design.  What is reported is
    exact.

    ``biases`` (needs ``activations``; ``None``, or one per layer: ``None`` or an ``[n_out_k]`` array) are added to each
    layer's outputs before its activation, in ``chain_design``'s format; the last layer's bias is allowed.  The search
    states are then the (latencies, intervals) after bias and activation, and a point's cost is the float32 sum in stage
    order of ``design(p)``'s cost column, its bias / activation stage's ops in the order: input ops (cost 0), each
    output's constant addition, each output's activation op.  A pair whose bias makes a non-zero constant is dropped
    (``dropped_constant``), and one whose bias the tracer folds into the previous layer's (``chain_design``'s folding case)
    is dropped and counted in ``profile['layers'][k]['dropped_folded']``, and one whose bias op is not exact in the stage
    arrays (float32 intervals, ``|data| < 2**31``; ``chain_design`` refuses it) in ``dropped_inexact``.  The bias values
    themselves are checked before any device call.  ``biases=None`` and all-zero biases give the front without them.

    Limits: a layer's states all run in one call, and their op tables stay on the device until that call ends; if they do
    not fit (``DA4ML_E_CAPACITY``), or any set fails on any state, the call raises that layer's error prefixed with
    ``layer k: `` and returns nothing.  Branching networks are not covered, nor is a bias the tracer folds across an
    activation (above).  ``solver(kernels, option_sets, **kw)`` stands
    in for ``solve_sweep_batch`` (same keywords and results), ``pricer`` for ``price_pipelined``."""
    ks = [_prefixed(f'layer {k}', _kernel_arg, W) for k, W in enumerate(kernels)]
    if not ks:
        raise ValueError('chain_front needs at least one layer')
    for k in range(1, len(ks)):
        if ks[k - 1].shape[1] != ks[k].shape[0]:
            raise ValueError(f'layer {k - 1} has {ks[k - 1].shape[1]} outputs but layer {k} has {ks[k].shape[0]} inputs')
    sets = _sweep_sets(option_sets)
    if qintervals is not None and len(qintervals) != len(ks):
        raise ValueError(f'expected qintervals for {len(ks)} layers, got {len(qintervals)}')
    acts = None
    if activations is not None:
        acts = list(activations)
        if len(acts) != len(ks) - 1:
            raise ValueError(f'{len(ks)} layers need {len(ks) - 1} activations, got {len(acts)}')
        acts = [_act_seq(k, act, int(ks[k].shape[1])) for k, act in enumerate(acts)]
        for k in range(1, len(ks) if qintervals is not None else 0):
            if qintervals[k] is not None:
                raise ValueError(f"layer {k}: with activations a layer's qintervals are its traced inputs' (only layer 0's may be given)")
    bs = None
    if biases is not None:
        if acts is None:
            raise ValueError('biases need activations (an empty list for one layer): a chain with biases is solved under its traced intervals')
        bs = _biases_arg(biases, [int(W.shape[1]) for W in ks])
    qs = [None if qintervals is None else _prefixed(f'layer {k}', _qint_arg, qintervals[k], W.shape[0]) for k, W in enumerate(ks)]
    qs = [None if q is None else [tuple(map(float, r)) for r in q] for q in qs]
    l0 = _prefixed('layer 0', _lat_arg, latencies, ks[0].shape[0])
    c = float(latency_cutoff)
    if not (c >= 0 and np.isfinite(c)):
        raise ValueError(f'latency_cutoff must be a non-negative number, got {latency_cutoff!r}')
    dt = np.float64 if c > 0 else np.float32  # (traced latencies are the tracer's doubles)
    states = [np.zeros(ks[0].shape[0], dt) if l0 is None else l0.astype(dt)]
    state_qs = [qs[0]]  # (with activations: each state's qintervals, float32 values as Python floats)
    solver = solve_sweep_batch if solver is None else solver
    pricer = price_pipelined if pricer is None else pricer
    prof = dict(launches=0, device_ms=0.0, jobs_run=0, jobs_total=0, layers=[])
    points, state_of = None, np.zeros(1, np.int64)
    for k, W in enumerate(ks):
        if k > 0 and acts is None:  # one state per distinct output-latency vector, in order of first use
            index = {}
            state_of = np.asarray([index.setdefault(np.asarray(o, dt).tobytes(), len(index)) for o in points[3]], np.int64)
            states = [np.frombuffer(b, dt) for b in index]
        elif k > 0:  # one state per distinct (output latencies, float32 activated intervals), in order of first use
            index, first = {}, []
            for p, (o, v, *_) in enumerate(points[3]):
                key = np.asarray(o, dt).tobytes() + np.asarray(v, np.float32).tobytes()
                if key not in index:
                    index[key] = len(first)
                    first.append(p)
            state_of = np.asarray([index[np.asarray(o, dt).tobytes() + np.asarray(v, np.float32).tobytes()] for o, v, *_ in points[3]], np.int64)
            states = [np.asarray(points[3][p][0], dt) for p in first]
            state_qs = [[tuple(map(float, r)) for r in np.asarray(points[3][p][1], np.float32)] for p in first]
        n, lats = len(states), [[float(v) for v in s] for s in states]
        sweeps = _prefixed(f'layer {k}', solver, [W] * n, sets, qintervals=[qs[k]] * n if acts is None else state_qs, latencies=lats, adder_size=int(adder_size),
                           carry_size=int(carry_size))  # fmt: skip
        traced, priced = None, {}
        if c > 0:  # every front candidate of every state, traced under its state's latencies: one pricing call
            keys = [(s, int(i)) for s, sw in enumerate(sweeps) for i in np.asarray(sw.front, np.int64).tolist()]
            pr = _prefixed(f'layer {k}', pricer, [sweeps[s].raw(i) for s, i in keys], c, latencies=[lats[s] for s, _ in keys], retiming=False)
            traced = {key: (float(pr.latency_max[j, 0]), np.asarray(pr.out_latency(j, 0), np.float64)) for j, key in enumerate(keys) if int(pr.status[j, 0]) == 0}
            priced = dict(dropped=len(keys) - len(traced), price_launches=int(pr.profile.get('launches', 0)), price_device_ms=float(pr.profile.get('device_ms', 0.0)))
        acted, replayed = None, {}
        bias = None if bs is None else bs[k]
        if acts is not None and (k < len(ks) - 1 or bias is not None):
            t0 = time.perf_counter()
            acted = _chain_replay(points, state_of, sweeps, traced, k, acts[k] if k < len(acts) else [], bias)
            replayed = dict(replay_ms=(time.perf_counter() - t0) * 1e3, dropped_constant=acted[2]['constant'])
            if bs is not None:
                replayed.update(dropped_folded=acted[2]['folded'], dropped_inexact=acted[2]['inexact'])
        elif acts is not None:
            replayed = dict(replay_ms=0.0, dropped_constant=0, **({} if bs is None else dict(dropped_folded=0, dropped_inexact=0)))
        points = _chain_layer(points, state_of, sweeps, lats, traced, None if acts is None else state_qs, acted, c)
        if len(points[0]) == 0:
            if replayed.get('dropped_constant') or replayed.get('dropped_folded') or replayed.get('dropped_inexact'):
                raise ValueError(f'layer {k}: every front candidate is slower than the latency cutoff {c}, makes an output of bias / activation {k} a '
                                 'non-zero constant, has a bias the tracer folds or a bias op that is not exact in the stage arrays')
            raise ValueError(f'layer {k}: every front candidate has an adder slower than the latency cutoff {c}')
        p0 = sweeps[0].profile  # (the whole call's)
        layer = dict(states=n, candidates=sum(len(sw.candidates['cost']) for sw in sweeps), points=len(points[0]),
                     **{key: p0[key] for key in ('launches', 'device_ms', 'jobs_run', 'jobs_total')}, **priced, **replayed)
        prof['layers'].append(layer)
        for key in ('launches', 'device_ms', 'jobs_run', 'jobs_total'):
            prof[key] += layer[key]
        del sweeps  # (the designs are copied out: free the handles before the next layer's call)
    cost, lat, choice, _, raws, calls = points
    order = np.argsort(lat, kind='stable')
    return ChainFront(cost[order], lat[order], choice[order], [raws[p] for p in order], [calls[p] for p in order], prof, c, acts, bs)


_ZERO_QINT = (0.0, 0.0, 2.0**32)  # the tracer's constant 0: FixedVariable gives a constant the step 2**-_const_f(0) = 2**32


def _chain_replay(points, state_of, sweeps, traced, k, seq, bias=None):
    """``_chain_layer``'s ``acted`` for layer ``k`` of a chain with activations: every front candidate (that pricing
    kept) of every state, replayed through bias ``k`` and the activations ``seq`` after layer ``k`` (empty: the last
    layer's bias alone) from each distinct float64 input values of the state's parents (at layer 0, the design's own
    input intervals, as in ``chain_design``).  A table entry is ``None`` for a dropped pair; its reason goes to the
    returned counts (``constant``, ``folded``, ``inexact``)."""
    group_of, groups = [], {}  # parent -> replay group; (state, float64 intervals and views) -> group
    for p, s in enumerate(state_of.tolist()):
        key = None if points is None else np.asarray(points[3][p][1], np.float64).tobytes() + np.asarray(points[3][p][2], np.float64).tobytes()
        group_of.append(groups.setdefault((s, key), len(groups)))
    table, drops = {}, dict(constant=0, folded=0, inexact=0)
    cache = [{} for _ in seq]  # ('apply' tables by interval and kif, shared by every replay of the layer)
    for (s, key), g in groups.items():
        for i in np.asarray(sweeps[s].front, np.int64).tolist():
            if traced is not None and (s, i) not in traced:
                continue
            stages = sweeps[s].raw(i).stages
            if key is None:
                vals = _input_intervals(stages)
            else:
                q = np.frombuffer(key, np.float64)
                n = q.size // 5
                vals = [(*r[:3], r[3], bool(r[4])) for r in np.concatenate([q[: 3 * n].reshape(n, 3), q[3 * n :].reshape(n, 2)], axis=1).tolist()]
            try:
                traced_vals, biased, changed, nxt = _activated_intervals(stages, vals, k, seq, bias, cache)
            except _FoldedBias:
                table[g, i] = None
                drops['folded'] += 1
                continue
            except _InexactBias:
                table[g, i] = None
                drops['inexact'] += 1
                continue
            except _ConstantValue:
                table[g, i] = None
                drops['constant'] += 1
                continue
            # (stage order: the constant additions, then each activation's ops in value order)
            act_cost = [np.asarray([0.0 if c is None else c[3] for c in biased], np.float32)] if bias is not None else []
            act_cost = np.concatenate(act_cost + [np.asarray(_op_costs(ops), np.float32) for ops in changed]).astype(np.float32)
            dls = [tuple((a.cond[4], a.mux[4]) if isinstance(a, _Mux) else int(a[4]) for a in (ops[j] for ops in changed)
                         if a is not None and not isinstance(a, _View) and (isinstance(a, _Mux) or a[4])) for j in range(len(nxt))]
            zero = np.asarray([v[0] == v[1] for v in nxt], bool)
            vals = [_ZERO_QINT if v[0] == v[1] else v[:3] for v in nxt]
            aux = np.asarray([v[3:] for v in nxt], np.float64).reshape(-1, 2)
            table[g, i] = (act_cost, zero, np.asarray(vals, np.float64).reshape(-1, 3), aux, dls)
    return group_of, table, drops


def _op_costs(ops) -> list:
    """The cost of every op one activation records, in stage order: per value (0 for none); for a leaky ReLU every
    condition adder, then every mux."""
    if any(isinstance(a, (_Mux, _View)) for a in ops):
        return [a.cond[3] if isinstance(a, _Mux) else 0.0 for a in ops] + [a.mux[3] if isinstance(a, _Mux) else 0.0 for a in ops]
    return [0.0 if a is None else a[3] for a in ops]


def _act_latency(lat: float, dl, c: float) -> float:
    """An output's latency after one latency step of ``_chain_replay``'s ``dls``: a lookup's increment (no cutoff rule), or
    a leaky ReLU's (condition dlat, mux dlat): the condition adder under the tracer's register-boundary rule at cutoff
    ``c`` (trace/fixed_variable.py:373-379), then the mux, ``max`` of its operands plus its dlat, with no rule."""
    from math import ceil

    if not isinstance(dl, tuple):
        return dl + lat
    d, m = float(dl[0]), float(dl[1])
    cond = d + lat
    if c > 0 and ceil(cond / c) > ceil(lat / c):
        cond = ceil(lat / c) * c + d
    return max(lat, cond) + m


def _kif_prop(lo: float, hi: float, step: float) -> tuple[int, int, int]:
    """``FixedVariable.kif`` (reference trace/fixed_variable.py:418-428) of a non-constant value."""
    return int(lo < 0), int(np.ceil(np.log2(max(-lo, hi + step)))), -int(np.log2(step))


def _activate(kind: str, lo: float, hi: float, step: float, k: int, i: int, f: int):
    """What the tracer's ``relu(i, f)`` (TRN, trace/fixed_variable.py:645-686) or ``quantize(k, i, f)`` (WRAP / TRN,
    :688-779) makes of a non-constant value [lo, hi] / step: ``None`` (the value itself), or the (lo, hi, step) of the result
    (lo == hi: a constant).  Every number is a dyadic rational, exact in float64."""
    from math import ceil, floor

    if kind == 'relu':
        st = max(2.0**-f, step)
        l, h = floor(max(0.0, lo) / st) * st, floor(hi / st) * st
        if 2.0**i - st < h:
            l, h = 0.0, 2.0**i - st
        h = max(0.0, h)
        return None if (l, h, st) == (lo, hi, step) else (l, h, st)
    if k + i + f <= 0:
        return 0.0, 0.0, 1.0
    k0, i0, f0 = _kif_prop(lo, hi, step)
    if k >= k0 and i >= i0 and f >= f0:
        return None
    f = min(f, f0)
    k = min(k, k0) if i >= i0 else k
    st = 2.0**-f
    if lo < 0:
        i0 = max(i0, ceil(np.log2(-(floor(lo / st) * st))))
    i = min(i, i0 + int(k == 0 and k0 == 1))
    if i + k + f <= 0:
        return 0.0, 0.0, 1.0
    l, h = -k * 2.0**i, 2.0**i - st
    if lo >= l and hi <= h:
        l, h = floor(lo / st) * st, floor(hi / st) * st
    return l, h, st


def _traced_views(stages, vals):
    """``_traced_intervals`` with each output's factor and kind: (lo, hi, step, factor, cadd) per output, ``factor`` the
    +-2**k of the tracer's view of it (``FixedVariable._factor``: the operand with a positive factor leads an addition,
    shifts and negations scale it) and ``cadd`` whether that view is of a constant addition (``opr == 'cadd'``, which
    ``_pow2_mul``, ``__neg__`` and an addition of the constant 0 keep).  ``vals`` entries are (lo, hi, step) (factor 1, not
    a constant addition) or such 5-tuples."""
    vals = [tuple(v) if len(v) == 5 else (*v, 1.0, False) for v in vals]
    for st in stages:
        ins = [(lo * 2.0**sh, hi * 2.0**sh, s * 2.0**sh, f * 2.0**sh, c) for (lo, hi, s, f, c), sh in zip(vals, np.asarray(st['inp_shifts'], np.int64).tolist())]
        buf = []
        for id0, id1, opc, data in np.asarray(st['ops_i'], np.int64).reshape(-1, 4).tolist():
            if opc == -1:
                buf.append(ins[id0])
                continue
            a, (lo, hi, s, f, c) = buf[id0], buf[id1]
            b = (lo * 2.0**data, hi * 2.0**data, s * 2.0**data, f * 2.0**data, c)
            if opc == 1:
                b = (-b[1], -b[0], b[2], -b[3], c)
            if a[0] != a[1] and b[0] != b[1]:
                buf.append((a[0] + b[0], a[1] + b[1], min(a[2], b[2]), a[3] if a[3] > 0 or b[3] < 0 else b[3], False))
            else:
                buf.append(b if a[0] == a[1] else a)
        vals = []
        for i, sh, ng in zip(np.asarray(st['out_idxs'], np.int64).tolist(), np.asarray(st['out_shifts'], np.int64).tolist(), np.asarray(st['out_negs']).astype(bool).tolist()):
            if i < 0:
                vals.append((0.0, 0.0, 1.0, 1.0, False))
                continue
            lo, hi, s, f = (v * 2.0**sh for v in buf[i][:4])
            vals.append((-hi, -lo, s, -f, buf[i][4]) if ng else (lo, hi, s, f, buf[i][4]))
    return vals


def _traced_intervals(stages, vals):
    """The intervals (lo, hi, step) of a design's outputs as the tracer's replay (``CombLogic.__call__`` on
    ``FixedVariable``s) gives them for inputs of intervals ``vals``: sums of the operands' scaled intervals, which can be
    wider than the ones the solver records.  A dead column is the constant 0, (0, 0, 1)."""
    return [v[:3] for v in _traced_views(stages, vals)]


def _const_f(c: float) -> int:
    """``_const_f`` of the tracer (trace/fixed_variable.py:201-214): the least f in (-32, 32] with ``c * 2**f`` an integer."""
    if c == 0:
        return -32
    lo, hi = -32, 32
    while hi - lo > 1:
        mid = (hi + lo) // 2
        v = c * 2.0**mid
        if v == int(v):
            hi = mid
        else:
            lo = mid
    return hi


def _exact_sum(a: float, b: float) -> float | None:
    """``a + b`` when it is exact in float64 (the tracer adds Decimals), else ``None``."""
    s = a + b
    bb = s - a
    return s if (a - (s - bb)) + (b - bb) == 0.0 else None


def _bias_op(j: int, k: int, v, b: float):
    """What the tracer's ``v + b`` (``FixedVariable._const_add``, trace/fixed_variable.py:484-513) makes of output ``j`` of
    layer ``k``, ``v`` its (lo, hi, step, factor, cadd) and ``b`` a non-zero bias: (lo, hi, step, cost, data) of the
    constant-addition node in the value's own units, ``data`` the bias in steps of the result.  Its cost is the tracer's,
    ``ceil(log2(|b / factor| + 2**-f)) + f`` with ``f = _const_f(b / factor)``.  ``_ConstantValue`` for a constant
    result; ``_FoldedBias`` when ``v`` is itself a constant addition (the tracer folds the two); ``ValueError`` when the op
    is not exact in the stage arrays (float32 intervals, an int32 ``data``): ``_InexactBias``."""
    from fractions import Fraction
    from math import ceil, log2

    lo, hi, st, fac, cadd = v
    if lo == hi:
        raise _ConstantValue(f'bias {k}: output {j} of layer {k} is the constant {_exact_sum(lo, b)} (only the constant 0 is covered)')
    if cadd:
        raise _FoldedBias(f'bias {k}: output {j} of layer {k} passes a biased value of the layer before through unchanged, and the tracer folds '
                          'the two biases into one constant addition across the activation (not covered)')
    l, h = _exact_sum(lo, b), _exact_sum(hi, b)
    step = min(st, 2.0 ** -_const_f(b))
    data = b / step
    if l is None or h is None or any(float(np.float32(x)) != x for x in (l, h, step)) or abs(data) >= 2**31:
        raise _InexactBias(f'bias {k}: output {j} of layer {k} plus {b!r} is not exact in the stage arrays (float32 intervals, |bias / step| < 2**31)')
    d = b / fac
    f = _const_f(d)
    cost = float(ceil(log2(float(abs(Fraction(d)) + Fraction(2) ** -f))) + f)
    return l, h, step, cost, int(data)


class _ConstantValue(ValueError):
    """A value of a chain that is or becomes a constant other than 0: ``chain_design`` refuses it, ``chain_front`` drops
    the candidate."""


class _InexactBias(ValueError):
    """A bias whose constant addition is not exact in the stage arrays (float32 intervals, ``|data| < 2**31``):
    ``chain_design`` refuses it, ``chain_front`` drops the candidate."""


class _FoldedBias(ValueError):
    """A bias the tracer folds into the constant addition of the layer before (a pass-through column of a biased value
    that the activation left unchanged): ``chain_design`` refuses it, ``chain_front`` drops the candidate."""


def _input_intervals(stages) -> list:
    """The intervals (lo, hi, step) of a design's inputs (``CombLogic.inp_qint``: an input without an input op is (0, 0, 1))."""
    s0 = stages[0]
    vals = [(0.0, 0.0, 1.0)] * int(s0['shape'][0])
    for (id0, _, opc, _), q in zip(np.asarray(s0['ops_i'], np.int64).reshape(-1, 4).tolist(), np.asarray(s0['ops_f'], np.float64).reshape(-1, 5).tolist()):
        if opc == -1:
            vals[id0] = tuple(q[:3])
    return vals


def _activated_intervals(stages, vals, k: int, seq, bias=None, cache=None):
    """One step of the tracer's interval replay of a chain: layer ``k``'s design (``stages``) on inputs ``vals``
    (``_traced_views``), then bias ``k`` (``None`` or ``[n_out]`` float64, added to every output with
    ``FixedVariable._const_add``), then the activations of ``seq`` (``_act_seq`` specs, in order; empty: none, as after
    the last layer) on every output.  Returns ``(traced, biased, acts, nxt)``: ``traced[j]`` is output ``j``'s (lo, hi,
    step); ``biased[j]`` is ``None`` without a bias op, else the (lo, hi, step, cost, data) of the constant addition the
    tracer records (``_bias_op``); ``acts[a][j]`` is ``None`` when activation ``a`` of the sequence leaves value ``j``
    unchanged, else the (lo, hi, step, cost, dl, table) of the op the tracer records for it (relu: cost ``sum(kif) / 2``,
    quantize: 0, both dl 0 and table ``None``; apply: the lookup's cost, latency increment and table, ``_apply_op``;
    leaky_relu: a ``_Mux`` or a ``_View``, ``_leaky_op``), or
    (0.0, 0.0, 1.0, 0.0, 0, None) for the constant 0 (a dead column, or a format with no bits left); ``nxt[j]`` is the
    value handed on, as (lo, hi, step, factor, cadd).  ``_ConstantValue`` when a value is or becomes any other constant,
    ``_FoldedBias`` for a bias the tracer folds.  ``cache``: the tables of ``'apply'`` activations by (interval, kif), one
    dict per activation of ``seq``.  The one Python copy of these rules (the C++ copy is ``pp_prepare``'s)."""
    views = _traced_views(stages, vals)
    traced = [v[:3] for v in views]
    biased, cur = [], []
    for j, v in enumerate(views):
        b = 0.0 if bias is None else float(bias[j])
        if b != 0.0:
            r = _bias_op(j, k, v, b)
            biased.append(r)
            v = (*r[:3], v[3], True)
        else:
            biased.append(None)
        cur.append(v)
    cache = [{} for _ in seq] if cache is None else cache
    acts = []
    for a, spec in enumerate(seq):
        kind, kif = spec[:2]
        ops, nxt = [], []
        for j, v in enumerate(cur):
            lo, hi, st = v[:3]
            if kind == 'leaky_relu':
                r, w = _leaky_op(j, k, v, kif, int(stages[0]['adder_size']), int(stages[0]['carry_size']))
                ops.append(r)
                nxt.append(w)
                continue
            if kind == 'apply':
                r = _apply_op(j, k, v, kif[j], *spec[2:], cache[a])
                if r is None:
                    ops.append((0.0, 0.0, 1.0, 0.0, 0, None))
                    nxt.append((0.0, 0.0, 1.0, 1.0, False))
                else:
                    ops.append(r)
                    nxt.append((*r[:3], 1.0, False))
                continue
            if lo == hi:
                if lo != 0.0 or hi != 0.0:
                    raise _ConstantValue(f'activation {k}: output {j} of layer {k} is the constant {lo} (only the constant 0 is covered)')
                ops.append((0.0, 0.0, 1.0, 0.0, 0, None))
                nxt.append((0.0, 0.0, 1.0, 1.0, False))
                continue
            r = _activate(kind, lo, hi, st, *(int(x) for x in kif[j]))
            if r is None:
                ops.append(None)
                nxt.append(v)
            elif r[0] == r[1]:
                if r[0] != 0.0:
                    raise _ConstantValue(f'activation {k}: output {j} becomes the constant {r[0]} (only the constant 0 is covered)')
                ops.append((0.0, 0.0, 1.0, 0.0, 0, None))
                nxt.append((0.0, 0.0, 1.0, 1.0, False))
            else:
                ops.append((*r, sum(_kif_prop(*r)) / 2 if kind == 'relu' else 0.0, 0, None))
                nxt.append((*r, abs(v[3]), False))
        acts.append(ops)
        cur = nxt
    for j, v in enumerate(cur):
        if not seq and v[0] == v[1]:
            if v[0] != 0.0 or v[1] != 0.0:
                raise _ConstantValue(f'activation {k}: output {j} of layer {k} is the constant {v[0]} (only the constant 0 is covered)')
            cur[j] = (0.0, 0.0, 1.0, 1.0, False)
    return traced, biased, acts, cur


def _bias_arg(k: int, b, n: int):
    """``None`` (no bias, or an all-zero one) or the ``[n]`` float64 bias ``k`` of ``chain_design`` / ``chain_front``."""
    if b is None:
        return None
    try:
        a = np.asarray(b, np.float64)
    except (TypeError, ValueError):
        raise ValueError(f'bias {k}: expected None or {n} numbers, got {b!r}') from None
    if a.shape != (n,):
        raise ValueError(f'bias {k}: expected None or shape ({n},), got shape {a.shape}')
    if not np.isfinite(a).all():
        raise ValueError(f'bias {k}: every value must be finite')
    sc = a * 2.0**32
    if not (np.abs(sc) < 2.0**63).all() or (sc != np.round(sc)).any():
        raise ValueError(f'bias {k}: every value must be a multiple of 2**-32 (the tracer finds a constant\'s step in [2**-32, 2**32]), with |value| < 2**31')
    return a if (a != 0).any() else None


def _biases_arg(biases, n_outs):
    """Per layer ``None`` or its ``[n_out]`` bias (``_bias_arg``), or ``None`` when no layer has a non-zero one."""
    if biases is None:
        return None
    bs = list(biases)
    if len(bs) != len(n_outs):
        raise ValueError(f'{len(n_outs)} layers need {len(n_outs)} biases (None for none), got {len(bs)}')
    bs = [_bias_arg(k, b, n) for k, (b, n) in enumerate(zip(bs, n_outs))]
    return bs if any(b is not None for b in bs) else None


_APPLY_ROUND = ('TRN', 'RND')
_APPLY_OVERFLOW = ('WRAP', 'SAT', 'SAT_SYM')


def _act_arg(k: int, act, n: int):
    """(kind, [n, 3] int64 kif) of activation ``k`` of ``chain_design``; for ``'apply'``, (kind, kif, fn, round_mode,
    overflow_mode); for ``'leaky_relu'``, (kind, alpha)."""
    if isinstance(act, (tuple, list)) and len(act) and isinstance(act[0], str) and act[0] == 'leaky_relu':
        a = act[1] if len(act) == 2 else None
        ok = isinstance(a, (int, float, np.integer, np.floating)) and not isinstance(a, (bool, np.bool_))
        if ok:
            a = float(a)
            ok = bool(np.isfinite(a)) and 0.0 < a < 1.0 and np.frexp(a)[0] == 0.5
        if not ok:
            raise ValueError(f"activation {k}: ('leaky_relu', alpha) needs alpha a power of two with 0 < alpha < 1 (the tracer multiplies by any "
                             f'other with adders), got {act!r}')
        return ('leaky_relu', a)
    if not isinstance(act, (tuple, list)) or len(act) not in ((3, 4, 5) if len(act) and isinstance(act[0], str) and act[0] == 'apply' else (2, 3, 4)):
        raise ValueError(f"activation {k}: expected ('quantize' | 'relu', kif[, round_mode[, overflow_mode]]) or ('apply', fn, kif[, round_mode[, overflow_mode]]), got {act!r}")
    if isinstance(act[0], str) and act[0] == 'apply':
        kind, fn, kif, *modes = act
        if not callable(fn):
            raise ValueError(f"activation {k}: the function of 'apply' must be callable, got {fn!r}")
        rnd = str(modes[0]).upper() if len(modes) > 0 else 'TRN'
        ovf = str(modes[1]).upper() if len(modes) > 1 else 'WRAP'
        if rnd not in _APPLY_ROUND:
            raise ValueError(f"activation {k}: rounding mode {modes[0]!r} of 'apply' is not one of {', '.join(_APPLY_ROUND)}")
        if ovf not in _APPLY_OVERFLOW:
            raise ValueError(f"activation {k}: overflow mode {modes[1]!r} of 'apply' is not one of {', '.join(_APPLY_OVERFLOW)}")
    else:
        kind, kif, *modes = act
        if kind not in ('quantize', 'relu'):
            raise ValueError(f"activation {k}: {kind!r} is not 'quantize', 'relu', 'apply' or 'leaky_relu'")
        if len(modes) > 0 and str(modes[0]).upper() != 'TRN':
            raise ValueError(f'activation {k}: rounding mode {modes[0]!r} is not covered (only TRN)')
        if len(modes) > 1 and str(modes[1]).upper() != 'WRAP':
            raise ValueError(f'activation {k}: overflow mode {modes[1]!r} is not covered (only WRAP)')
    a = np.asarray(kif)
    if a.dtype == bool:
        a = a.astype(np.int64)
    if a.size == 0 or not (np.issubdtype(a.dtype, np.integer) or (np.issubdtype(a.dtype, np.floating) and np.all(np.isfinite(a)) and np.all(a == np.round(a)))):
        raise ValueError(f'activation {k}: kif must be integers')
    a = a.astype(np.int64)
    if a.shape == (3,):
        a = np.tile(a, (n, 1))
    if a.shape != (n, 3):
        raise ValueError(f'activation {k}: kif must be one (k, i, f) triple or [{n}, 3], got shape {np.asarray(kif).shape}')
    if not np.isin(a[:, 0], (0, 1)).all() or (kind == 'relu' and (a[:, 0] != 0).any()):
        raise ValueError(f"activation {k}: k must be 0 or 1" + (" (0 for 'relu': its output is unsigned)" if kind == 'relu' else ''))
    if (np.abs(a[:, 1:]) > 64).any():
        raise ValueError(f'activation {k}: i and f must be within [-64, 64]')
    return (kind, a) if kind != 'apply' else (kind, a, fn, rnd, ovf)


def _act_tuple(spec) -> tuple:
    """The ``chain_design`` activation tuple of an ``_act_arg`` spec."""
    return ('apply', spec[2], spec[1], *spec[3:]) if spec[0] == 'apply' else tuple(spec)


def _act_seq(k: int, act, n: int) -> list:
    """Activation ``k`` of ``chain_design`` / ``chain_front`` as a list of ``_act_arg`` specs, applied in order: one
    activation tuple (its first element a ``str``) or a non-empty list of them."""
    if isinstance(act, (tuple, list)) and len(act) and isinstance(act[0], str):
        return [_act_arg(k, act, n)]
    if not isinstance(act, (tuple, list)) or len(act) == 0:
        raise ValueError(f'activation {k}: expected an activation tuple or a non-empty list of them, got {act!r}')
    return [_act_arg(k, a, n) for a in act]


def _same_acts(a: list, b: list) -> bool | None:
    """Whether two ``_act_seq`` lists are the same activations: ``False`` when kinds, kifs or modes differ, ``True`` when
    they are equal and every ``'apply'`` function is the same object, ``None`` when only the functions differ (the caller
    compares the tables they give)."""
    if len(a) != len(b) or any(x[0] != y[0] or not np.array_equal(x[1], y[1]) or x[3:] != y[3:] for x, y in zip(a, b)):
        return False
    return None if any(x[0] == 'apply' and x[2] is not y[2] for x, y in zip(a, b)) else True


def fixed_quantize(x, k, i, f, overflow_mode: str = 'WRAP', round_mode: str = 'TRN') -> np.ndarray:
    """The numeric fixed-point quantizer the tracer applies to an ``apply`` table (``_quantize``): round to the step
    ``2**-f`` (TRN: floor, RND: floor of ``x + step / 2``), then bring the result into ``[-k * 2**i, 2**i - 2**-f]``
    (WRAP: modulo ``2**(k + i)``; SAT: clip; SAT_SYM: clip to ``[-k * (2**i - 2**-f), 2**i - 2**-f]``).  A format with
    ``k + i + f <= 0`` gives 0."""
    x = np.asarray(x, np.float64)
    if k + i + f <= 0:
        return np.zeros_like(x)
    st = 2.0**-f
    y = np.floor(x / st + (0.5 if round_mode == 'RND' else 0.0)) * st
    hi = 2.0**i - st
    if overflow_mode == 'WRAP':
        lo = -k * 2.0**i
        return np.mod(y - lo, 2.0 ** (i + k)) + lo
    lo = -k * 2.0**i if overflow_mode == 'SAT' else -k * hi
    return np.clip(y, lo, hi)


def _interpret_as(x, k: int, i: int, f: int):
    """``interpret_as`` of the tracer (trace/fixed_variable.py:100-110): integers read as two's complement (k, i, f)."""
    b = k + i + f
    bias = 2.0 ** (b - 1) * k
    return 2.0**-f * (np.floor(x + bias) % 2.0**b - bias)


def _lsb_locs(x: np.ndarray) -> np.ndarray:
    """``get_lsb_loc`` of every element (its float32 value): the exponent of its lowest set bit, 127 for 0."""
    b = np.asarray(x, np.float32).view(np.uint32).astype(np.int64)
    e, m = (b >> 23) & 0xFF, (b & 0x7FFFFF) + (1 << 23)
    tz = np.log2(m & -m).astype(np.int64)
    return np.where(np.asarray(x, np.float32) == 0, 127, e + tz - 150)


def _make_table(values: np.ndarray):
    """``to_spec`` of the tracer (trace/fixed_variable.py:72-79): (sha256 hex, int32 table, out_qint)."""
    import hashlib

    f_out = int(-_lsb_locs(values).min())
    ints = (values * 2.0**f_out).astype(np.int32)
    h = hashlib.sha256(ints.data)
    h.update(f'{f_out}'.encode())
    return h.hexdigest(), ints, (float(np.min(values)), float(np.max(values)), float(2.0**-f_out))


def _apply_op(j: int, k: int, v, kif, fn, rnd: str, ovf: str, cache: dict):
    """What the tracer's ``x.apply(fn).quantize(k, i, f, ovf, rnd)`` makes of value ``v`` = (lo, hi, step, factor, cadd):
    the table over the value's interval (reversed for a negative factor), each entry quantized (``fixed_quantize``), its
    ``to_spec``, then ``FixedVariable.lookup``.  Returns ``None`` for the constant 0, else (lo, hi, step, cost, dl, table)
    with the tracer's lookup cost and latency increment (trace/fixed_variable.py:331-340) and ``table`` = (sha, int32
    values, out_qint).  ``_ConstantValue`` for a non-zero constant.  ``cache`` holds the tables of one activation by
    (interval, kif), as the tracer's ``local_tables``."""
    from math import ceil

    lo, hi, st, fac = v[:4]
    a, b = (lo, hi) if fac >= 0 else (hi, lo)
    kk, ii, ff = (int(x) for x in kif)
    key = (a, b, st if lo != hi else 0.0, kk, ii, ff)
    if key not in cache:
        n = round(abs(b - a) / st) + 1 if lo != hi else 1
        x = np.linspace(a, b, n)
        y = np.asarray(fn(x), np.float64)
        if y.shape != x.shape:
            raise ValueError(f'activation {k}: the function of \'apply\' gave shape {y.shape} for an input of shape {x.shape}')
        if not np.isfinite(y).all():
            raise ValueError(f"activation {k}: the function of 'apply' gave a value that is not finite on the interval [{min(a, b)}, {max(a, b)}]")
        cache[key] = _make_table(fixed_quantize(y, kk, ii, ff, ovf, rnd))
    table = cache[key]
    o_lo, o_hi, o_st = table[2]
    if o_lo == o_hi:
        if o_lo != 0.0:
            raise _ConstantValue(f'activation {k}: output {j} becomes the constant {o_lo} (only the constant 0 is covered)')
        return None
    b_in, b_out = sum(_kif_prop(lo, hi, st)), sum(_kif_prop(o_lo, o_hi, o_st))
    cost = 2 ** max(b_in - 5, 0) * ceil(b_out / 2)
    if b_in < 5:
        cost *= b_in / 5
    return o_lo, o_hi, o_st, float(cost), max(b_in - 6, 1), table


class _Mux(tuple):
    """The two ops the tracer's ``np.maximum(x, alpha * x)`` records for one value: ``cond`` = (lo, hi, step, cost, dlat) of
    the condition adder ``x - alpha * x`` and ``mux`` = (lo, hi, step, cost, dlat) of the MSB mux of ``alpha * x`` and ``x``
    on it (the intervals those of the values the tracer hands on), ``qint`` the interval ``max_of`` hands ``msb_mux``."""

    cond = property(lambda self: self[0])
    mux = property(lambda self: self[1])
    qint = property(lambda self: self[2])


class _View(tuple):
    """A leaky ReLU the tracer answers with the view ``alpha * x`` (no op): ``shift`` = log2(alpha)."""

    shift = property(lambda self: self[0])


def _leaky_op(j: int, k: int, v, alpha: float, a_sz: int, c_sz: int):
    """What the tracer's ``np.maximum(x, alpha * x)`` (``FixedVariable.max_of``, trace/fixed_variable.py:902-920, then
    ``msb_mux`` with ``zt_sensitive=False``, :788-859) makes of value ``v`` = (lo, hi, step, factor, cadd), ``alpha`` a
    power of two in (0, 1): (op, value handed on).  ``op`` is ``None`` when it is ``x`` itself (``lo >= alpha * hi``), a
    ``_View`` when it is the view ``alpha * x`` (``hi <= alpha * lo``), the constant-0 record for 0, else a ``_Mux``.
    ``_ConstantValue`` for a non-zero constant."""
    from math import floor, log2

    lo, hi, st, fac, cadd = v
    if lo == hi:
        if lo != 0.0:
            raise _ConstantValue(f'activation {k}: output {j} of layer {k} is the constant {lo} (only the constant 0 is covered)')
        return (0.0, 0.0, 1.0, 0.0, 0, None), (0.0, 0.0, 1.0, 1.0, False)
    ax = (alpha * lo, alpha * hi, alpha * st, alpha * fac)  # (_pow2_mul: a view of the same node)
    if lo >= ax[1]:
        return None, v
    if hi <= ax[0]:
        return _View((int(log2(alpha)),)), (*ax, cadd)
    x = (lo, hi, st, fac)
    nax = (0.0 - ax[1], 0.0 - ax[0], ax[2], -ax[3])
    X, Y = (x, nax) if fac > 0 else (nax, x)  # (FixedVariable.__add__: the operand with a positive factor leads)
    c_dl, c_cost = cost_add(X[:3], Y[:3], 0, False, a_sz, c_sz)
    cond = (X[0] + Y[0], X[1] + Y[1], min(st, ax[2]), c_cost, c_dl)
    qint = (max(lo, ax[0]), max(hi, ax[1]), min(st, ax[2]))
    A, B, q, neg = ax, x, qint, ax[3] < 0
    if neg:  # (msb_mux of -a, -b under the mirrored qint, seen negated)
        A, B, q = (0.0 - A[1], 0.0 - A[0], A[2], -A[3]), (0.0 - B[1], 0.0 - B[0], B[2], -B[3]), (0.0 - qint[1], 0.0 - qint[0], qint[2])
    step = min(A[2], B[2])
    m_lo = max(floor(q[0] / step) * step, min(A[0], B[0]))
    m_hi = min(floor(q[1] / step) * step, max(A[1], B[1]))
    m_dl, m_cost = cost_add(A[:3], B[:3], 0, False, a_sz, c_sz)
    mux = (0.0 - m_hi, 0.0 - m_lo, step, m_cost / 2, m_dl) if neg else (m_lo, m_hi, step, m_cost / 2, m_dl)
    return _Mux((cond, mux, qint)), (*mux[:3], ax[3], False)


def chain_design(designs, activations, biases=None) -> RawPipeline:
    """A chain of solver designs with a relu or quantizer between consecutive layers, as ONE design: layer 0's stages, an
    activation stage, layer 1's stages, and so on.  ``price_pipelined`` prices and splits it as the reference's tracer
    pipelines the whole model: ``to_pipeline(comb_trace(inp, chain(inp)), c, retiming)``, where ``chain`` replays every
    layer with ``CombLogic.__call__`` and applies ``relu`` / ``quantize`` between them; its register stages can fall inside
    and across layers.

    ``designs``: solver results (``RawPipeline``, stage-dict lists or ``Pipeline`` containers), layer ``k``'s output count
    equal to layer ``k + 1``'s input count, all with the same ``adder_size`` / ``carry_size``.  ``activations[k]`` is the
    op between layer ``k`` and layer ``k + 1``: ``('relu', kif)`` for ``relu(i, f)`` or ``('quantize', kif)`` for
    ``quantize(k, i, f)``, with ``kif`` one ``(k, i, f)`` triple for every output or an ``[n_out_k, 3]`` int array (``k``
    is 0 for relu).  Rounding is TRN and overflow WRAP; an optional third and fourth element may name them, and any other
    mode is a ``ValueError``.

    ``('apply', fn, kif[, round_mode[, overflow_mode]])`` is what the tracer makes of ``x.apply(fn).quantize(k, i, f,
    overflow_mode, round_mode)``: per value a lookup table (opcode 8) of ``fn`` over the value's traced interval (in
    reversed order when the tracer's view of the value has a negative factor), each entry quantized to ``(k, i, f)``
    (``fixed_quantize``: TRN / RND, WRAP / SAT / SAT_SYM, which change only the table values).  ``fn`` maps a float64
    array to an array of the same shape.  Values with equal tables share one; a stage with lookups has
    ``lookup_tables`` (per table its int32 values and ``out_qint``, numbered by first use), and a lookup op's ``data`` is
    its table's index.  A lookup costs ``2**max(b_in - 5, 0) * ceil(b_out / 2)`` (times ``b_in / 5`` when ``b_in < 5``)
    and adds ``max(b_in - 6, 1)`` to its operand's latency.  A value whose table has one value becomes that constant:
    0 is a dead column, any other is refused.  ``activations[k]`` may be a non-empty list of activations, applied in
    order, e.g. ``[('quantize', (1, 2, 3)), ('apply', np.tanh, (1, 0, 6))]`` (a pre-quantizer keeps the table small); a
    one-element list is the activation itself.

    ``('leaky_relu', alpha)``, ``alpha`` a power of two in (0, 1), is what the tracer makes of ``np.maximum(x, alpha *
    x)``: per value a condition adder (opcode 1, ``x - alpha * x``) and an MSB mux (opcode 6) of ``alpha * x`` and ``x``
    on it, with the tracer's intervals, costs and latencies, or no op where the tracer returns ``x`` or the view ``alpha *
    x`` (``_leaky_op``).  A leaky ReLU ends its stage: the condition adders close it, and the next stage starts with the
    muxes (DESIGN.md, "Leaky ReLU in whole chains").

    An activation stage has one input op per value (opcode -1, the value's interval ``Pipeline.out_qint`` and latency), and
    one op per value the activation changes, with the fields the tracer records for it: opcode 2 (relu) or 3 (quantize)
    reading that input, data 0, the result's interval and the tracer's cost (``sum(kif) / 2`` for relu, 0 for quantize).
    Intervals are the ones the tracer's replay of the layers gives, which can be wider than the solver's.  Latencies are
    the value's as its layer's design records it (relu and quantize add none); a layer's design is solved as if its
    inputs arrived at 0, and ``price_pipelined`` re-traces every latency anyway.  A value the tracer passes through unchanged (``quantize`` to a
    wider format, ``relu`` of a non-negative value) gets no op: its output reads the input op.  A value that becomes the
    constant 0 (a dead column, or a format with no bits left) is a dead output column (``out_idx -1``).  A value that would
    become any other constant is refused with ``ValueError``.

    ``biases[k]`` (``None``, or one per layer: ``None`` or an ``[n_out_k]`` array) is added to layer ``k``'s outputs before
    activation ``k``, as ``x @ W_k + b_k`` adds it in a traced model (``FixedVariable._const_add``).  A non-zero bias gets
    the op the tracer records, in the activation stage between the input ops and the activation ops: opcode 4 reading the
    value's input op, ``data`` the bias in steps of the result, the interval ``(lo + b, hi + b)`` with step ``min(step,
    2**-_const_f(b))`` and the tracer's cost ``ceil(log2(|b / factor| + 2**-f)) + f`` (``f = _const_f(b / factor)``,
    ``factor`` the sign and scaling of the tracer's view of the value); the activation op of that value reads it.  A zero
    bias records nothing, so all-zero biases give the design without them.  The last layer's bias gets a trailing stage of
    its own, with no activation.  A bias is refused (``ValueError``) when it is not finite or not a multiple of 2**-32,
    when its op is not exact in the stage arrays (float32 intervals, ``|data| < 2**31``), when it makes a non-zero
    constant (a bias on a dead column or on a value the activation zeroed), and when the tracer would fold it into the
    bias of the layer before (a column that passes a biased value through unchanged: the folded op would read a node on
    the far side of the activation stage).  All checks run on the host, before any device call."""
    stages = [_design_stages(d) for d in designs]
    if not stages:
        raise ValueError('chain_design needs at least one design')
    acts = list(activations)
    if len(acts) != len(stages) - 1:
        raise ValueError(f'{len(stages)} designs need {len(stages) - 1} activations, got {len(acts)}')
    sizes = {(int(d[0]['adder_size']), int(d[0]['carry_size'])) for d in stages}
    if len(sizes) != 1:
        raise ValueError(f'the designs of a chain must share adder_size and carry_size, got {sorted(sizes)}')
    a_sz, c_sz = sizes.pop()
    for k in range(1, len(stages)):
        if stages[k - 1][-1]['shape'][1] != stages[k][0]['shape'][0]:
            raise ValueError(f"layer {k - 1} has {stages[k - 1][-1]['shape'][1]} outputs but layer {k} has {stages[k][0]['shape'][0]} inputs")
    n_outs = [int(st[-1]['shape'][1]) for st in stages]
    kinds = [_act_seq(k, act, n_outs[k]) for k, act in enumerate(acts)]
    bs = _biases_arg(biases, n_outs)
    vals = _input_intervals(stages[0])
    out = [dict(st) for st in stages[0]]
    for k in range(len(stages)):
        seq = kinds[k] if k < len(kinds) else []
        bias = None if bs is None else bs[k]
        if not seq and bias is None:
            break
        st, vals = _act_stage(stages[k], vals, k, seq, bias, a_sz, c_sz)
        out += st
        if k + 1 < len(stages):
            out += [dict(st) for st in stages[k + 1]]
    return RawPipeline.from_stages(out)


def _same_tables(a, b) -> bool:
    """Whether two stages' ``lookup_tables`` (or ``None``) hold the same tables in the same order."""
    a, b = a or [], b or []
    return len(a) == len(b) and all(np.array_equal(x['table'], y['table']) and tuple(x['out_qint']) == tuple(y['out_qint']) for x, y in zip(a, b))


def _act_stage(layer, vals, k, seq, bias, a_sz, c_sz):
    """(stages, values handed on) of the bias / activation stage after layer ``k`` (``layer``: its stages) of a chain
    design: one input op per value, then one constant addition per non-zero bias in value order, then for each
    activation of ``seq`` in order one op per value it changes, in value order, reading the value's latest op.  A
    lookup's ``data`` is its table's index in the stage's ``lookup_tables`` (tables numbered by first use, one per
    distinct content).  A leaky ReLU adds its condition adders (opcode 1, ``x - alpha * x``) in value order and ends the
    stage; the stage outputs every value (a ``_View`` at ``out_shift = log2(alpha)``), then for each mux ``alpha * x``
    (``out_shift = log2(alpha)``) and its condition, and the next stage starts with one input op per output and the muxes
    in value order (opcode 6 of ``alpha * x`` and ``x`` with shift 0 on the condition): a DAIS mux shifts only its second
    operand, so ``alpha * x`` has to reach it as a value of its own."""
    last = layer[-1]
    n = int(last['shape'][1])
    traced, biased, changed, nxt = _activated_intervals(layer, vals, k, seq, bias)
    idx = np.asarray(last['out_idxs'], np.int64)
    of = np.asarray(last['ops_f'], np.float64).reshape(-1, 5)
    ops_i, ops_f, out_idxs = [], [], np.arange(n, dtype=np.int64)
    for j in range(n):  # the input ops first, in value order: the traced interval and the solver's latency
        ops_i.append([j, -1, -1, 0])
        ops_f.append([*traced[j], float(of[idx[j], 3]) if idx[j] >= 0 else 0.0, 0.0])
    for j, c in enumerate(biased):  # constant additions: the bias in steps of the result, the tracer's cost
        if c is not None:
            out_idxs[j] = len(ops_i)
            ops_i.append([j, -1, 4, c[4]])
            ops_f.append([*c[:3], ops_f[j][3], c[3]])
    stages, tables, index = [], [], {}
    n_in = n

    def close(extra=(), shifts=None):
        st = dict(shape=(n_in, n + len(extra)), inp_shifts=np.zeros(n_in, np.int64), out_idxs=np.concatenate([out_idxs, np.asarray(extra, np.int64)]),
                  out_shifts=np.zeros(n + len(extra), np.int64) if shifts is None else np.asarray(shifts, np.int64), out_negs=np.zeros(n + len(extra), np.int64),
                  ops_i=np.asarray(ops_i, np.int64).reshape(-1, 4), ops_f=np.asarray(ops_f, np.float32).reshape(-1, 5), adder_size=a_sz, carry_size=c_sz)  # fmt: skip
        if tables:
            st['lookup_tables'] = list(tables)
        stages.append(st)

    for (kind, *rest), ops in zip(seq, changed):
        if kind == 'leaky_relu':
            muxes, conds = [j for j, a in enumerate(ops) if isinstance(a, _Mux)], {}
            for j in muxes:  # the condition adders: x - 2**log2(alpha) * x, the tracer's cost
                src = int(out_idxs[j])
                conds[j] = len(ops_i)
                ops_i.append([src, src, 1, int(np.log2(rest[0]))])
                ops_f.append([*ops[j].cond[:3], ops_f[src][3] + ops[j].cond[4], ops[j].cond[3]])
            sh = int(np.log2(rest[0]))
            extra = [v for j in muxes for v in (int(out_idxs[j]), conds[j])]
            shifts = [sh if isinstance(a, _View) else 0 for a in ops] + [v for _ in muxes for v in (sh, 0)]
            q_out = []  # (interval, latency) of every output of the closing stage, as the next stage's input ops record them
            for o, sft in zip(list(out_idxs) + extra, shifts):
                if o < 0:
                    q_out.append((0.0, 0.0, 1.0, 0.0))
                    continue
                lo, hi, st_ = (float(np.float32(x)) * 2.0**sft for x in ops_f[o][:3])
                q_out.append((lo, hi, st_, float(np.float32(ops_f[o][3]))))
            close(extra, shifts)
            n_in, tables, index = len(q_out), [], {}
            ops_i = [[j, -1, -1, 0] for j in range(n_in)]
            ops_f = [[*q[:3], q[3], 0.0] for q in q_out]
            out_idxs = np.arange(n, dtype=np.int64)
            for t, j in enumerate(muxes):  # the muxes: alpha * x (input n + 2t), x (input j), the condition (input n + 2t + 1)
                m = ops[j].mux
                out_idxs[j] = len(ops_i)
                ops_i.append([n + 2 * t, j, 6, n + 2 * t + 1])
                ops_f.append([*ops[j].qint, max(q_out[j][3], q_out[n + 2 * t + 1][3]) + m[4], m[3]])
            for j, a in enumerate(ops):
                if a is not None and not isinstance(a, (_Mux, _View)):  # (the constant 0)
                    out_idxs[j] = -1
                elif q_out[j][0] == q_out[j][1] == 0.0 and not isinstance(a, _Mux):
                    out_idxs[j] = -1
            continue
        for j, a in enumerate(ops):
            if a is None:
                continue
            if a[0] == a[1]:  # (the constant 0)
                out_idxs[j] = -1
                continue
            src = int(out_idxs[j])
            out_idxs[j] = len(ops_i)
            if kind == 'apply':
                sha, ints, out_q = a[5]
                if sha not in index:
                    index[sha] = len(tables)
                    tables.append(dict(table=ints, out_qint=out_q))
                ops_i.append([src, -1, 8, index[sha]])
                ops_f.append([*a[:3], a[4] + float(np.float32(ops_f[src][3])), a[3]])
            else:
                ops_i.append([src, -1, 2 if kind == 'relu' else 3, 0])
                ops_f.append([*a[:3], ops_f[src][3], a[3]])
    for j, v in enumerate(nxt):
        if v[0] == v[1] == 0.0:
            out_idxs[j] = -1
    close()
    return stages, nxt


PRICE_STATUS = ['ok', 'adder slower than the cutoff', 'not supported']  # PipelinePrice.status codes 0, 1, 2


class PipelinePrice:
    """What ``price_pipelined`` returns: arrays ``[n_designs, n_cutoffs]`` -- ``status`` (int32: 0 ok, 1 an adder is
    slower than the cutoff, the tracer's ``AssertionError``; 2 not supported, a constant intermediate value that
    ``emit`` refuses too; names in ``PRICE_STATUS``), ``stages`` (the number of register stages of the split),
    ``reg_bits`` (``Pipeline.reg_bits`` of the split), ``latency_max`` (the traced output latencies' maximum, float64)
    and ``cutoff`` (the cutoff retiming settled on, or the cutoff itself without retiming), ``cutoffs`` (the cutoffs
    asked for), and ``out_latency(d, j)``: design ``d``'s traced output latencies under cutoff ``j``.  A task that is not
    ok has ``stages`` and ``reg_bits`` -1 and NaN latencies.  ``profile``: the call's device time and launches (with
    ``keep_split``, also ``split_launches`` and ``split_bytes``, the bytes of op tables copied back).  ``split(d, j)``:
    design ``d``'s register stages under cutoff ``j`` when the call kept them."""

    def __init__(self, status, stages, reg_bits, latency_max, cutoff, cutoffs, out_lat, profile, splits=None):
        self.status, self.stages, self.reg_bits, self.latency_max, self.cutoff = status, stages, reg_bits, latency_max, cutoff
        self.cutoffs, self._out_lat, self.profile = cutoffs, out_lat, profile
        self._splits = splits  # None: not kept; else per design None (not priced) or per cutoff (status, tables)

    def split(self, d: int, j: int = 0) -> list[dict]:
        """The register stages of design ``d`` under cutoff ``j``: what the reference's ``to_pipeline(comb, c, retiming)``
        returns for the task -- without retiming the split of the trace under the design's input latencies; with it,
        ``retime_pipeline``'s (the first split when no bisection round succeeded, else the last successful round's, at
        cutoff ``self.cutoff[d, j]`` with every input at latency 0).  Stage dicts in the layout of ``RawPipeline.stages``
        (``ops_f`` float64), for ``emit.verilog_pipeline_logic_gen`` / ``types.pipeline_from_arrays``.  ``ValueError``
        when the splits were not kept, the task is not ok, or the reference's ``to_pipeline`` raises on it (a ``KeyError``:
        a stage would have no op or no output, as when every input arrives after the first stage)."""
        d, j = int(d), int(j)
        if self._splits is None or self._splits[d] is None:
            raise ValueError(f'the split of design {d} was not kept (price_pipelined(..., keep_split=True) keeps it)')
        if int(self.status[d, j]) != 0:
            raise ValueError(f'design {d} under cutoff {float(self.cutoffs[j])} is not ok ({PRICE_STATUS[int(self.status[d, j])]}): it has no split')
        code, tables = self._splits[d][j]
        if code == 2:
            raise ValueError(f"design {d} under cutoff {float(self.cutoffs[j])}: the reference's to_pipeline raises KeyError on this task "
                             '(a stage would have no op or no output, as when every input arrives after the first stage)')  # fmt: skip
        return _split_stages(*tables)

    def __len__(self):
        return len(self.status)

    @property
    def ok(self) -> np.ndarray:
        return self.status == 0

    def out_latency(self, d: int, j: int = 0) -> np.ndarray:
        """Traced latency of every output of design ``d`` under cutoff ``j`` (float64; 0.0 for a dead column)."""
        o = self._out_lat[int(d)]
        if o is None:
            raise ValueError(f'design {d} was not priced (its op tables were not kept)')
        return o[int(j)].copy()

    def _scatter(self, rows, n) -> 'PipelinePrice':
        """The same answers at rows ``rows`` of ``n`` (the others: not priced)."""
        m = len(self.cutoffs)

        def put(a, fill):
            out = np.full((n, m), fill, a.dtype)
            out[rows] = a
            return out

        out_lat = [None] * n
        splits = None if self._splits is None else [None] * n
        for k, r in enumerate(np.asarray(rows, np.int64).tolist()):
            out_lat[r] = self._out_lat[k]
            if splits is not None:
                splits[r] = self._splits[k]
        return PipelinePrice(put(self.status, -1), put(self.stages, -1), put(self.reg_bits, -1), put(self.latency_max, np.nan), put(self.cutoff, np.nan),
                             self.cutoffs, out_lat, self.profile, splits)  # fmt: skip


def _split_stages(meta, outs, shifts, negs, ops_i, ops_f, adder_size, carry_size, tables=None) -> list[dict]:
    """Stage dicts (fresh arrays) of one split from its concatenated tables.  ``tables``: the design's lookup tables
    (``_design_tables``), which the split's opcode 8 ops index; each stage then gets the ones it uses as its own
    ``lookup_tables``, in the order of their first use in the split (the order of the traced model's tables that
    ``remap_table_idxs`` of ``to_pipeline`` keeps), and its ops are renumbered to match."""
    from math import ceil

    stages, o, r = [], 0, 0
    first = {}  # design table -> first use in the split's op order, which is the order of the traced model's ops
    for d in ops_i[ops_i[:, 2] == 8, 3].tolist() if tables else ():
        first.setdefault(d, len(first))
    for n_in, n_out, n_ops in meta.tolist():
        st = dict(shape=(n_in, n_out), inp_shifts=np.zeros(n_in, np.int64), out_idxs=outs[o : o + n_out].copy(), out_shifts=shifts[o : o + n_out].copy(),
                  out_negs=negs[o : o + n_out].astype(bool), ops_i=ops_i[r : r + n_ops].copy(), ops_f=ops_f[r : r + n_ops].copy(), adder_size=adder_size,
                  carry_size=carry_size)  # fmt: skip
        lut = st['ops_i'][:, 2] == 8
        for q in np.flatnonzero(lut).tolist():  # a lookup's cost is a double (m * b_in / 5 for b_in < 5); the kernels hold a float
            m = ceil(sum(_kif_prop(*st['ops_f'][q, :3].tolist())) / 2)
            st['ops_f'][q, 4] = next((m * (b / 5) for b in range(1, 5) if np.float32(m * (b / 5)) == np.float32(st['ops_f'][q, 4])), st['ops_f'][q, 4])
        if tables and lut.any():
            used = sorted(set(st['ops_i'][lut, 3].tolist()), key=first.get)
            remap = {g: i for i, g in enumerate(used)}
            st['ops_i'][lut, 3] = [remap[g] for g in st['ops_i'][lut, 3].tolist()]
            st['lookup_tables'] = [dict(table=tables[g]['table'].copy(), out_qint=tuple(tables[g]['out_qint'])) for g in used]
        stages.append(st)
        o, r = o + n_out, r + n_ops
    return stages


def _design_tables(stages):
    """(tables, per-stage index maps) of a design: its distinct lookup tables over all stages, numbered by first use in
    op order, and for every stage the map from its own table indices to these."""
    tables, index, maps = [], {}, []
    for st in stages:
        own = st.get('lookup_tables') or []
        m = {}
        oi = np.asarray(st['ops_i'], np.int64).reshape(-1, 4)
        for d in oi[oi[:, 2] == 8, 3].tolist():
            if not 0 <= d < len(own):
                raise ValueError(f'an opcode 8 lookup reads table {d}, but its stage has {len(own)} lookup tables')
            if d not in m:
                t = own[d]
                key = (np.asarray(t['table'], np.int32).tobytes(), tuple(float(v) for v in t['out_qint']))
                if key not in index:
                    index[key] = len(tables)
                    tables.append(dict(table=np.asarray(t['table'], np.int32), out_qint=key[1]))
                m[d] = index[key]
        maps.append(m)
    return tables, maps


def _take_splits(designs, m, info, copy) -> list:
    """Per design, per cutoff (status, tables) of the splits a call kept; ``info(t, out[4])`` / ``copy(t, ...)`` read task
    ``t`` (``da4ml_split_info`` / ``da4ml_split_copy`` or the CPU harness's)."""
    q = np.zeros(4, np.int64)
    out = []
    for d, stages in enumerate(designs):
        row = []
        for j in range(m):
            info(d * m + j, q)
            code, n_st, n_rows, n_outs = (int(v) for v in q)
            if code != 0:
                row.append((code, None))
                continue
            meta = np.zeros((n_st, 3), np.int64)
            outs, shifts, negs = np.zeros(n_outs, np.int64), np.zeros(n_outs, np.int64), np.zeros(n_outs, np.int64)
            ops_i, ops_f = np.zeros((n_rows, 4), np.int64), np.zeros((n_rows, 5), np.float64)
            copy(d * m + j, meta, outs, shifts, negs, ops_i, ops_f)
            tables = _design_tables(stages)[0] if any('lookup_tables' in st for st in stages) else None
            row.append((0, (meta, outs, shifts, negs, ops_i, ops_f, int(stages[0]['adder_size']), int(stages[0]['carry_size']), tables)))
        out.append(row)
    return out


def _design_stages(design) -> list[dict]:
    from ..emit import _stages_of

    return _stages_of(design)


def _price_args(designs, latency_cutoff, latencies) -> dict:
    """The flat arrays of ``da4ml_pipeline_price`` for ``price_pipelined``'s arguments."""
    if hasattr(designs, 'stages') or hasattr(designs, 'solutions') or isinstance(designs, dict):
        designs = [designs]
    designs = [_design_stages(d) for d in designs]
    if not designs:
        raise ValueError('price_pipelined needs at least one design')
    cut = np.ascontiguousarray(np.atleast_1d(np.asarray(latency_cutoff, np.float64)).ravel())
    if cut.size == 0:
        raise ValueError('price_pipelined needs at least one latency cutoff')
    stages = [st for d in designs for st in d]
    if any('lookup_tables' in st or (np.asarray(st['ops_i']).reshape(-1, 4)[:, 2] == 8).any() for st in stages):
        stages = []  # (lookups read the design's tables, numbered over all its stages: _design_tables)
        for d in designs:
            for st, m in zip(d, _design_tables(d)[1]):
                if m:
                    st = dict(st, ops_i=np.asarray(st['ops_i'], np.int64).reshape(-1, 4).copy())
                    lut = st['ops_i'][:, 2] == 8
                    st['ops_i'][lut, 3] = [m[v] for v in st['ops_i'][lut, 3].tolist()]
                stages.append(st)
    meta = np.asarray([[st['shape'][0], st['shape'][1], len(st['ops_i']), st['carry_size'], st['adder_size']] for st in stages], np.int64).reshape(-1, 5)
    cat = lambda key, w: np.ascontiguousarray(np.concatenate([np.asarray(st[key], np.int64).reshape(-1, w) for st in stages]).ravel())  # noqa: E731
    ops_f = np.ascontiguousarray(np.concatenate([np.asarray(st['ops_f'], np.float32).reshape(-1, 5) for st in stages]).ravel())
    lat = None
    if latencies is not None:
        if len(latencies) != len(designs):
            raise ValueError(f'expected latencies for {len(designs)} designs, got {len(latencies)}')
        parts = []
        for d, l in zip(designs, latencies):
            n_in = d[0]['shape'][0]
            v = np.zeros(n_in) if l is None or len(l) == 0 else np.asarray(list(l), np.float64).ravel()
            if v.size != n_in:
                raise ValueError(f'expected {n_in} latencies, got {v.size}')
            parts.append(v)
        lat = np.ascontiguousarray(np.concatenate(parts) if parts else np.zeros(0))
    return dict(designs=designs, cutoffs=cut, latencies=lat, n_stages=np.asarray([len(d) for d in designs], np.int64), meta=np.ascontiguousarray(meta.ravel()),
                inp_shifts=cat('inp_shifts', 1), out_idxs=cat('out_idxs', 1), out_shifts=cat('out_shifts', 1), out_negs=cat('out_negs', 1), ops_i=cat('ops_i', 4),
                ops_f=ops_f)  # fmt: skip


def price_pipelined(designs, latency_cutoff, latencies=None, retiming: bool = True, keep_split: bool = False) -> PipelinePrice:
    """Price designs as they will be pipelined, on the GPU: for every design and every cutoff ``c`` what the reference gets
    by replaying the design through its tracer under ``HWConfig(adder_size, carry_size, c)`` with its inputs at
    ``latencies``, gathering it with ``comb_trace`` and splitting it with ``to_pipeline(comb, c, retiming)``.

    ``designs``: a sequence of ``RawPipeline``s, stage-dict lists or ``Pipeline`` containers (or one of them).
    ``latency_cutoff``: a positive number or a sequence of them.  ``latencies``: ``None`` (zeros) or, per design, ``None``
    or its input latencies.  With ``retiming`` the split is the one ``retime_pipeline`` keeps; its bisection re-traces
    with every input at latency 0, as the reference re-traces a split.  Traced latencies are those of the first trace
    (the given latencies and cutoff), as the next layer's tracer would see them.

    A task that is not ``ok`` (an adder slower than the cutoff, a constant intermediate value) does not raise: it is
    reported in ``status``, so one slow adder does not fail a sweep.  Argument errors raise ``ValueError`` before any
    device call.

    ``keep_split=True`` also builds every ok task's register stages on the GPU (two more launches, after pricing and the
    bisection) and keeps them: ``split(d, j)``.  A split is the reference's only where pricing is: the retimed split
    re-traces with every input at latency 0, which is the reference's re-trace when every input is in the first stage.
    The other arrays are the same with and without it."""
    pk = _price_args(designs, latency_cutoff, latencies)
    designs, cut, lat = pk['designs'], pk['cutoffs'], pk['latencies']
    n, m = len(designs), cut.size
    n_out = [d[-1]['shape'][1] for d in designs]
    st_ = np.zeros(n * m, np.int32)
    stg, rb = np.zeros(n * m, np.int64), np.zeros(n * m, np.int64)
    lm, co = np.zeros(n * m), np.zeros(n * m)
    ol = np.zeros(sum(n_out) * m)
    prof = np.zeros(4 if keep_split else 2)
    f64 = lambda a: a.ctypes.data_as(_f64p) if a is not None else None  # noqa: E731
    args = [n, *[_ip(pk[k]) for k in ('n_stages', 'meta', 'inp_shifts', 'out_idxs', 'out_shifts', 'out_negs', 'ops_i')], _fp(pk['ops_f']), f64(lat), f64(cut), m,
            int(bool(retiming)), st_.ctypes.data_as(_i32p), _ip(stg), _ip(rb), f64(lm), f64(co), f64(ol), f64(prof)]  # fmt: skip
    splits = None
    if keep_split:
        h = _vp()
        _check(_L.da4ml_pipeline_split(*args, C.byref(h)))
        try:
            f = lambda a: a.ctypes.data_as(_f64p if a.dtype == np.float64 else _i64p)  # noqa: E731
            splits = _take_splits(designs, m, lambda t, q: _check(_L.da4ml_split_info(h, t, _ip(q))), lambda t, *a: _check(_L.da4ml_split_copy(h, t, *map(f, a))))
        finally:
            _L.da4ml_split_free(h)
    else:
        _check(_L.da4ml_pipeline_price(*args))
    edges = np.concatenate([[0], np.cumsum(np.asarray(n_out, np.int64) * m)])
    out_lat = [ol[edges[d] : edges[d + 1]].reshape(m, n_out[d]) for d in range(n)]
    profile = dict(device_ms=float(prof[0]), launches=int(prof[1]))
    if keep_split:
        profile.update(split_launches=int(prof[2]), split_bytes=int(prof[3]))
    return PipelinePrice(st_.reshape(n, m), stg.reshape(n, m), rb.reshape(n, m), lm.reshape(n, m), co.reshape(n, m), cut, out_lat, profile, splits)


def csd_decompose(inp, center=True):
    """(csd int8[n_in,n_out,N], shift0 int8[n_in], shift1 int8[n_out])  (bindings.cc:63-103)."""
    k = _kernel_arg(inp)
    csd = np.zeros(k.size * 32, np.int8)
    s0 = np.zeros(k.shape[0], np.int8)
    s1 = np.zeros(k.shape[1], np.int8)
    nb = C.c_int64(0)
    _check(_L.da4ml_cmvm_csd_decompose(_fp(k), k.shape[0], k.shape[1], int(bool(center)), csd.ctypes.data_as(_i8p), s0.ctypes.data_as(_i8p), s1.ctypes.data_as(_i8p), C.byref(nb)))
    return csd[: k.size * nb.value].reshape(k.shape[0], k.shape[1], nb.value).copy(), s0, s1


def int_arr_to_csd(inp):
    """int32 ndarray -> int8[..., N] CSD digits (bindings.cc:43-61)."""
    if not isinstance(inp, np.ndarray) or inp.dtype != np.int32:
        raise TypeError('inp must be a numpy int32 ndarray')
    a = np.ascontiguousarray(inp)
    out = np.zeros(a.size * 32, np.int8)
    nb = C.c_int64(0)
    _check(_L.da4ml_cmvm_int_arr_to_csd(a.ctypes.data_as(_i32p), a.size, out.ctypes.data_as(_i8p), C.byref(nb)))
    return out[: a.size * nb.value].reshape(*a.shape, nb.value).copy()


def kernel_decompose(kernel, dc=-2):
    """W = m0 @ m1 graph decomposition (bindings.cc:232-234 -> mat_decompose.cc:62-137)."""
    k = _kernel_arg(kernel)
    m0 = np.zeros(k.shape, np.float32)
    m1 = np.zeros((k.shape[1], k.shape[1]), np.float32)
    _check(_L.da4ml_cmvm_kernel_decompose(_fp(k), k.shape[0], k.shape[1], int(dc), _fp(m0), _fp(m1)))
    return m0, m1


def dais_interp_run(bin_logic, data, n_threads: int = 1):
    """``da4ml._binary.dais_interp_run`` (reference _binary/__init__.py:8-16): run a DAIS program (int32 words of
    ``CombLogic.to_binary``) on a batch of inputs; float64 ``[n_samples, n_out]``.  Runs on the GPU (``n_threads`` is
    accepted for signature compatibility); programs are limited to what the CMVM path emits (opcodes -1/0/1)."""
    prog = np.ascontiguousarray(np.ravel(bin_logic), dtype=np.int32)
    x = np.ascontiguousarray(np.ravel(data), dtype=np.float64)
    if prog.size < 6 or prog[0] != 1 or min(prog[2:5]) < 0:  # let the library word the header error
        inp_size, out_size, n = 0, 0, 0
    else:
        inp_size, out_size = int(prog[2]), int(prog[3])
        assert inp_size == 0 or x.size % inp_size == 0, f'Input size {x.size} is not divisible by {inp_size}'
        n = x.size // inp_size if inp_size else 0
    out = np.zeros((n, out_size), np.float64)
    _check(_L.da4ml_dais_run(prog.ctypes.data_as(_i32p), prog.size, x.ctypes.data_as(C.POINTER(C.c_double)), n, out.ctypes.data_as(C.POINTER(C.c_double))))
    return out


def get_lsb_loc(x: float) -> int:
    return int(_L.da4ml_cmvm_get_lsb_loc(float(x)))


def iceil_log2(x: float) -> int:
    return int(_L.da4ml_cmvm_iceil_log2(float(x)))


def cost_add(q0, q1, shift: int, sub: bool, adder_size: int, carry_size: int):
    a = np.asarray(tuple(q0), np.float32)
    b = np.asarray(tuple(q1), np.float32)
    out = np.zeros(2, np.float32)
    _L.da4ml_cmvm_cost_add(_fp(a), _fp(b), int(shift), int(bool(sub)), int(adder_size), int(carry_size), _fp(out))
    return float(out[0]), float(out[1])


__all__ = [
    'solve', 'solve_batch', 'solve_raw', 'solve_batch_raw', 'solve_batch_device_raw', 'solve_single_raw', 'solve_sweep', 'solve_sweep_batch', 'SweepResult', 'sweep_front',
    'solve_best_of', 'solve_best_of_raw', 'tb_mask', 'price_pipelined', 'PipelinePrice', 'PRICE_STATUS',
    'network_front', 'NetworkFront', 'NetworkPoint', 'chain_front', 'ChainFront', 'csd_decompose', 'int_arr_to_csd',
    'kernel_decompose', 'get_lsb_loc', 'iceil_log2', 'cost_add', 'dais_interp_run', 'device_info', 'plan', 'set_stream', 'set_group_size', 'set_accounting',
]  # fmt: skip
