"""ctypes binding of libda4ml_b200_cmvm.so (C ABI: include/da4ml_b200_cmvm.h).

Mirror of the reference's ``da4ml._binary`` re-exports (``src/da4ml/_binary/__init__.py:4,19``;
nanobind module ``_binary/cmvm/bindings.cc:227-263``): ``solve, csd_decompose, int_arr_to_csd,
kernel_decompose, get_lsb_loc, iceil_log2, cost_add`` with the same signatures, defaults and exception
types.  Added on top: ``solve_batch`` (many independent problems in one launch) and ``solve_single``.

The shared library is the product's only compute path; importing this module without it raises.
"""

from __future__ import annotations

import copy
import ctypes as C
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
    'da4ml_pipeline_split', 'da4ml_split_info', 'da4ml_split_copy', 'da4ml_split_free',
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
                ms = np.zeros(63, np.int64)
                _check(_L.da4ml_pipeline_stage_milestones(handle, s, _ip(ms)))
                cd['milestones'] = {250 << k: [int(v) for v in ms[9 * k : 9 * k + 9]] for k in range(7) if ms[9 * k + 8] > 0}
                self.counters.append(cd)
            self.device_ms = float(_L.da4ml_pipeline_device_ms(handle))
            self.launches = int(_L.da4ml_pipeline_launches(handle))
            prof = (C.c_double * 8)()
            _L.da4ml_pipeline_profile(handle, prof)
            self.profile = dict(device_ms=prof[0], launches=int(prof[1]), solve_kernel_ms=prof[2], solve_kernel_launches=int(prof[3]), algo_bytes=prof[4], jobs_total=int(prof[5]), jobs_run=int(prof[6]))
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

    def to_pipeline(self, types_module=None):
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
                            jobs_total=int(prof[5]), jobs_run=int(prof[6]), candidates=n, candidates_solved=self.n_solved, candidates_kept=self.n_kept)

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

    Only host arrays are held (each point's designs are ``RawPipeline`` copies), so a front pickles as it is."""

    def __init__(self, cost, latency, choice, raws, calls, profile, latency_cutoff=0.0):
        super().__init__(cost, latency, choice)
        self._raws, self._calls, self.profile = raws, calls, profile
        self.latency_cutoff = float(latency_cutoff)
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

    def reference_calls(self, p: int) -> list[dict]:
        """Per layer, the keywords of the ``solve(kernels[k], **kw)`` call that returns layer ``k``'s design in point
        ``p``: the candidate's options, the layer's ``qintervals`` and its input ``latencies`` as Python floats (for
        ``k > 0``, the output latencies of the point's design of layer ``k - 1``).  A candidate of a seeded option set
        carries its ``seed``, as ``SweepResult.reference_call`` does."""
        return copy.deepcopy(self._calls[p])


def _chain_layer(points, state_of, sweeps, state_lats, traced=None):
    """Extend the points of the layers so far by the next layer and prune.  ``points`` is ``None`` at layer 0, else
    ``(cost, lat, choice, outs, raws, calls)``; ``state_of[p]`` is the index of point ``p``'s input-latency state in
    ``sweeps`` and ``state_lats`` (lists of Python floats); at layer 0 there is one state and ``state_of == [0]``.
    Parents are taken in order and each is extended by every ``front`` candidate of its state's sweep, in candidate
    order; cost is the float32 sum in layer order, latency the new design's ``latency_max``; then the ``sweep_front``
    rule.  ``outs[p]`` are the output latencies of point ``p``'s last design.  ``traced[s, i]`` (pipelined chains):
    ``(latency_max, output latencies)`` of front candidate ``i`` of state ``s`` as traced under the cutoff, which replace the
    solver's; a front candidate without an entry is dropped."""
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
    if points is not None:
        cost = points[0][par] + cost
    keep = sweep_front(cost, lat)
    par, sidx, cand, cost, lat = par[keep], sidx[keep], cand[keep], cost[keep], lat[keep]
    choice = cand[:, None] if points is None else np.concatenate([points[2][par], cand[:, None]], axis=1)
    designs = {}  # (state, candidate) -> (RawPipeline, solve() keywords, output latencies), shared by the points using it
    raws, calls, outs = [], [], []
    for p, s, i in zip(par.tolist(), sidx.tolist(), cand.tolist()):
        if (s, i) not in designs:
            r = sweeps[s].raw(i)
            designs[s, i] = (r, {**sweeps[s].reference_call(i), 'latencies': state_lats[s]}, _out_latencies(r) if traced is None else traced[s, i][1])
        r, call, o = designs[s, i]
        raws.append([r] if points is None else [*points[4][p], r])
        calls.append([call] if points is None else [*points[5][p], call])
        outs.append(o)
    return cost, lat, choice, outs, raws, calls


def chain_front(kernels, option_sets, qintervals=None, latencies=None, adder_size=-1, carry_size=-1, solver=None, latency_cutoff=0.0, pricer=None) -> ChainFront:
    """The cost / latency front of a chain of layers, each layer solved under the output latencies of the design chosen
    for the layer before it, as a traced model's matmuls are: every reported design is what
    ``solve(kernels[k], **front.reference_calls(p)[k])`` returns, and every reported cost and latency is the chain's own.

    ``kernels[k]`` is layer ``k``'s constant matrix (``kernels[k].shape[1] == kernels[k + 1].shape[0]``).
    ``option_sets`` and the cost model (``adder_size``, ``carry_size``) are those of ``solve_sweep`` and the same for
    every layer.  ``qintervals`` is ``None`` or one entry per layer: ``None`` (``solve``'s default) or that layer's input
    intervals, e.g. those of the quantizer in front of it; intervals are not carried over from a layer's outputs.
    ``latencies`` are layer 0's input latencies (default zeros).

    Search: layer 0 is swept once, and its ``front`` candidates are the first points.  At each later layer a point's
    input-latency state is the output latencies of its last design (``Pipeline.out_latencies``; 0.0 for a constant-zero
    output); points whose states are equal as float32 share one problem, and all the layer's states go into one
    ``solver`` call (``solve_sweep_batch``: one GPU pass per layer).  Each point is extended by every ``front`` candidate
    of its state's sweep; its cost is the float32 sum of the designs' costs in layer order, and its latency the new
    design's ``latency_max``, which already contains the upstream latency.  The points are pruned after each layer with
    the ``sweep_front`` rule, and the result is sorted by ascending latency.

    Latency model: with ``latency_cutoff = 0`` (the default) latency is the solver's op latency.  With ``latency_cutoff =
    c > 0`` it is the latency the tracer gives the design under ``HWConfig(adder_size, carry_size, c)``: after each
    layer's sweep every front candidate of every state is priced under that state's latencies (``price_pipelined``
    without retiming, one call per layer); a point's latency is the traced ``latency_max``, its next state the traced
    output latencies (what the traced model hands the next ``solve``), pruning uses (cost, traced latency), and a
    candidate whose status is not ok (an adder slower than ``c``) is dropped (``profile['layers'][k]['dropped']``).
    ``stages[p] = floor(latency / (c + 1e-9)) + 1`` is the clock count ``to_pipeline`` gives the chain when its network
    inputs arrive before ``c``; ``retime_pipeline`` never accepts a split with more stages, so retiming never adds a
    clock.  ``best_stages(n)`` is the cheapest point with at most ``n`` stages.  Register bits of a whole chain are not
    reported: the activation ops between layers have widths of their own, so they are not the sum of the layers'.
    Activations between layers add no latency, as ``relu`` and ``wrap`` in the tracer keep their input's latency.  The
    front is the front of the chains explored: the solver is not monotone in its input latencies, so pruning partial
    chains on (cost, latency) is a heuristic and a pruned chain could have led to a better design.  What is reported is
    exact.

    Limits: a layer's states all run in one call, and their op tables stay on the device until that call ends; if they do
    not fit (``DA4ML_E_CAPACITY``), or any set fails on any state, the call raises that layer's error prefixed with
    ``layer k: `` and returns nothing.  Branching networks are not covered.  ``solver(kernels, option_sets, **kw)`` stands
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
    qs = [None if qintervals is None else _prefixed(f'layer {k}', _qint_arg, qintervals[k], W.shape[0]) for k, W in enumerate(ks)]
    qs = [None if q is None else [tuple(map(float, r)) for r in q] for q in qs]
    l0 = _prefixed('layer 0', _lat_arg, latencies, ks[0].shape[0])
    c = float(latency_cutoff)
    if not (c >= 0 and np.isfinite(c)):
        raise ValueError(f'latency_cutoff must be a non-negative number, got {latency_cutoff!r}')
    dt = np.float64 if c > 0 else np.float32  # (traced latencies are the tracer's doubles)
    states = [np.zeros(ks[0].shape[0], dt) if l0 is None else l0.astype(dt)]
    solver = solve_sweep_batch if solver is None else solver
    pricer = price_pipelined if pricer is None else pricer
    prof = dict(launches=0, device_ms=0.0, jobs_run=0, jobs_total=0, layers=[])
    points, state_of = None, np.zeros(1, np.int64)
    for k, W in enumerate(ks):
        if k > 0:  # one state per distinct output-latency vector, in order of first use
            index = {}
            state_of = np.asarray([index.setdefault(np.asarray(o, dt).tobytes(), len(index)) for o in points[3]], np.int64)
            states = [np.frombuffer(b, dt) for b in index]
        n, lats = len(states), [[float(v) for v in s] for s in states]
        sweeps = _prefixed(f'layer {k}', solver, [W] * n, sets, qintervals=[qs[k]] * n, latencies=lats, adder_size=int(adder_size), carry_size=int(carry_size))
        traced, priced = None, {}
        if c > 0:  # every front candidate of every state, traced under its state's latencies: one pricing call
            keys = [(s, int(i)) for s, sw in enumerate(sweeps) for i in np.asarray(sw.front, np.int64).tolist()]
            pr = _prefixed(f'layer {k}', pricer, [sweeps[s].raw(i) for s, i in keys], c, latencies=[lats[s] for s, _ in keys], retiming=False)
            traced = {key: (float(pr.latency_max[j, 0]), np.asarray(pr.out_latency(j, 0), np.float64)) for j, key in enumerate(keys) if int(pr.status[j, 0]) == 0}
            priced = dict(dropped=len(keys) - len(traced), price_launches=int(pr.profile.get('launches', 0)), price_device_ms=float(pr.profile.get('device_ms', 0.0)))
        points = _chain_layer(points, state_of, sweeps, lats, traced)
        if len(points[0]) == 0:
            raise ValueError(f'layer {k}: every front candidate has an adder slower than the latency cutoff {c}')
        p0 = sweeps[0].profile  # (the whole call's)
        layer = dict(states=n, candidates=sum(len(sw.candidates['cost']) for sw in sweeps), points=len(points[0]),
                     **{key: p0[key] for key in ('launches', 'device_ms', 'jobs_run', 'jobs_total')}, **priced)
        prof['layers'].append(layer)
        for key in ('launches', 'device_ms', 'jobs_run', 'jobs_total'):
            prof[key] += layer[key]
        del sweeps  # (the designs are copied out: free the handles before the next layer's call)
    cost, lat, choice, _, raws, calls = points
    order = np.argsort(lat, kind='stable')
    return ChainFront(cost[order], lat[order], choice[order], [raws[p] for p in order], [calls[p] for p in order], prof, c)


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


def _split_stages(meta, outs, shifts, negs, ops_i, ops_f, adder_size, carry_size) -> list[dict]:
    """Stage dicts (fresh arrays) of one split from its concatenated tables."""
    stages, o, r = [], 0, 0
    for n_in, n_out, n_ops in meta.tolist():
        stages.append(dict(shape=(n_in, n_out), inp_shifts=np.zeros(n_in, np.int64), out_idxs=outs[o : o + n_out].copy(), out_shifts=shifts[o : o + n_out].copy(),
                           out_negs=negs[o : o + n_out].astype(bool), ops_i=ops_i[r : r + n_ops].copy(), ops_f=ops_f[r : r + n_ops].copy(), adder_size=adder_size,
                           carry_size=carry_size))  # fmt: skip
        o, r = o + n_out, r + n_ops
    return stages


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
            row.append((0, (meta, outs, shifts, negs, ops_i, ops_f, int(stages[0]['adder_size']), int(stages[0]['carry_size']))))
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
