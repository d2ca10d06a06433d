"""Result containers handed back by the CMVM solver.

Field-for-field mirrors of the reference's ``da4ml.types`` containers that the solver constructs
(reference: ``src/da4ml/types.py:21-64`` QInterval/Op, ``:176-215`` CombLogic, ``:584-619`` Pipeline;
built by ``_binary/cmvm/bindings.cc:106-151``).  Only what the CMVM path produces is implemented:
opcodes -1 (input copy), 0 (add) and 1 (subtract).  The rest of ``da4ml.types`` (symbolic replay,
relu/quantize/LUT opcodes, DAIS binary, code generators) belongs to components that are out of scope
for this path (SURVEY.md section 2 rows 12-18).

When the real ``da4ml`` package is importable, ``da4ml_b200.cmvm.solve(..., types_module=da4ml.types)``
builds the reference's own classes instead, see INTEGRATION.md.
"""

from __future__ import annotations

import gc
import json
from functools import reduce
from pathlib import Path
from typing import NamedTuple

import numpy as np


class QInterval(NamedTuple):
    """Quantized interval [min, max] with step (reference types.py:21-26)."""

    min: float
    max: float
    step: float


class Op(NamedTuple):
    """One buffer operation: ``buf[i] = buf[id0] +/- buf[id1] * 2**data`` (opcode 0/1) or an input
    copy (opcode -1) (reference types.py:37-64)."""

    id0: int
    id1: int
    opcode: int
    data: int
    qint: QInterval
    latency: float
    cost: float


def minimal_kif_array(q: np.ndarray) -> np.ndarray:
    """Vectorised ``minimal_kif`` (reference types.py:84-112, symmetric=False) for an ``[n, 3]`` array of
    (min, max, step): returns ``[n, 3]`` int32 (keep_negative, integers, fractional)."""
    q = np.asarray(q, dtype=np.float64).reshape(-1, 3)
    out = np.zeros((len(q), 3), dtype=np.int32)
    live = ~((q[:, 0] == 0) & (q[:, 1] == 0))
    if live.any():
        mn, mx, st = q[live, 0], q[live, 1], q[live, 2]
        frac = (-np.log2(st)).astype(np.int64)  # int() truncation; steps are powers of two
        int_min, int_max = np.round(mn / st), np.round(mx / st)
        bits = np.ceil(np.log2(np.maximum(np.abs(int_min), int_max + 1))).astype(np.int64)
        out[live, 0] = mn < 0
        out[live, 1] = bits - frac
        out[live, 2] = frac
    return out


class CombLogic(NamedTuple):
    """One adder graph (reference types.py:176-215)."""

    shape: tuple[int, int]
    inp_shifts: list[int]
    out_idxs: list[int]
    out_shifts: list[int]
    out_negs: list[bool]
    ops: list[Op]
    carry_size: int
    adder_size: int
    lookup_tables: tuple | None = None

    def __call__(self, inp, quantize=False, debug=False, dump=False):
        """Replay the graph on numeric input(s); ``inp`` is ``[n_in]`` or ``[batch, n_in]``
        (reference types.py:217-370, opcodes -1/0/1 only)."""
        if quantize:
            raise NotImplementedError('input quantization is outside the CMVM path')
        x = np.asarray(inp, dtype=np.float64)
        single = x.ndim == 1
        x = np.atleast_2d(x) * (2.0 ** np.asarray(self.inp_shifts, dtype=np.float64))
        buf = np.empty((len(self.ops), x.shape[0]), dtype=np.float64)
        for i, op in enumerate(self.ops):
            if op.opcode == -1:
                buf[i] = x[:, op.id0]
            elif op.opcode == 0:
                buf[i] = buf[op.id0] + buf[op.id1] * 2.0**op.data
            elif op.opcode == 1:
                buf[i] = buf[op.id0] - buf[op.id1] * 2.0**op.data
            else:
                raise ValueError(f'Unknown opcode {op.opcode} in {op}')
        if dump:
            return buf.T[0] if single else buf.T
        idx = np.asarray(self.out_idxs, dtype=np.int64)
        sf = 2.0 ** np.asarray(self.out_shifts, dtype=np.float64)
        sign = np.where(np.asarray(self.out_negs, dtype=bool), -1.0, 1.0)
        mask = (idx >= 0).astype(np.float64)
        out = buf[np.maximum(idx, 0)].T * sf * sign * mask
        return out[0] if single else out

    @property
    def kernel(self) -> np.ndarray:
        """The constant matrix this graph implements (reference types.py:372-378)."""
        return self(np.identity(self.shape[0])).astype(np.float32)

    @property
    def cost(self) -> float:
        return float(sum(op.cost for op in self.ops))

    @property
    def n_adders(self) -> int:
        return sum(1 for op in self.ops if op.opcode in (0, 1))

    @property
    def latency(self) -> tuple[float, float]:
        lat = [self.ops[i].latency for i in self.out_idxs]
        if not lat:
            return 0.0, 0.0
        return min(lat), max(lat)

    @property
    def out_latency(self) -> list[float]:
        return [self.ops[i].latency if i >= 0 else 0.0 for i in self.out_idxs]

    @property
    def out_qint(self) -> list[QInterval]:
        buf = []
        for i, idx in enumerate(self.out_idxs):
            _min, _max, _step = self.ops[idx].qint
            sf = 2.0 ** self.out_shifts[i]
            _min, _max, _step = _min * sf, _max * sf, _step * sf
            if self.out_negs[i]:
                _min, _max = -_max, -_min
            buf.append(QInterval(_min, _max, _step))
        return buf

    @property
    def inp_latency(self) -> list[float]:
        return [op.latency for op in self.ops if op.opcode == -1]

    @property
    def inp_qint(self) -> list[QInterval]:
        # reference types.py:428-435: one entry per input element, scattered by the input op's id0
        qints = [QInterval(0.0, 0.0, 1.0) for _ in range(self.shape[0])]
        for op in self.ops:
            if op.opcode == -1:
                qints[op.id0] = op.qint
        return qints

    def __repr__(self):
        n_in, n_out = self.shape
        lo, hi = self.latency
        return f'Solution([{n_in} -> {n_out}], cost={self.cost}, latency={lo}-{hi})'

    def to_binary(self, version: int = 0) -> np.ndarray:
        """DAIS program of this graph as int32 words (reference types.py:500-541, docs/dais.md): header
        ``[spec=1, version, n_in, n_out, n_ops, n_tables=0] + inp_shifts + out_idxs + out_shifts + out_negs`` followed
        by 8 words per op ``(opcode, id0, id1, data_lo, data_hi, keep_negative, integers, fractional)``.  Built
        straight from the flat op table, without a Python loop over ops."""
        n_in, n_out = self.shape
        n_ops = len(self.ops)
        header = np.concatenate([[1, version, n_in, n_out, n_ops, 0], self.inp_shifts, self.out_idxs, self.out_shifts, np.asarray(self.out_negs, dtype=np.int64)]).astype(np.int32)
        code = np.zeros((n_ops, 8), dtype=np.int32)
        if n_ops:
            oi = np.asarray([(op.opcode, op.id0, op.id1, op.data) for op in self.ops], dtype=np.int64)
            q = np.asarray([op.qint for op in self.ops], dtype=np.float64)
            code[:, 0:3] = oi[:, 0:3]
            code[:, 3:5] = oi[:, 3].astype(np.int64).view(np.int32).reshape(-1, 2)  # little-endian 64-bit data word
            code[:, 5:8] = minimal_kif_array(q)
        return np.concatenate([header, code.ravel()])

    def predict(self, data, n_threads: int = 0) -> np.ndarray:
        """Bit-exact replay of this graph on a batch of inputs with the DAIS fixed-point semantics
        (reference types.py:549-581, ``dais_interp_run``); here the interpreter runs on the GPU."""
        from ._binary import dais_interp_run  # noqa: PLC0415

        if isinstance(data, (list, tuple)):
            data = np.concatenate([np.asarray(a).reshape(np.asarray(a).shape[0], -1) for a in data], axis=-1)
        return dais_interp_run(self.to_binary(), data, n_threads)

    def save_binary(self, path: str | Path, version: int = 0):
        self.to_binary(version=version).tofile(path)

    # JSON layout = the NamedTuple as nested lists (reference types.py:442-477)
    def save(self, path: str | Path):
        with open(path, 'w') as f:
            json.dump(self, f, separators=(',', ':'))

    @classmethod
    def deserialize(cls, data: list):
        ops = [Op(*_op[:4], QInterval(*_op[4]), *_op[5:]) for _op in data[5]]
        return cls(tuple(data[0]), data[1], data[2], data[3], data[4], ops, data[6], data[7], None)

    @classmethod
    def load(cls, path: str | Path):
        with open(path) as f:
            return cls.deserialize(json.load(f))


class Pipeline(NamedTuple):
    """Cascade of adder graphs; the solver returns two stages (reference types.py:584-693)."""

    solutions: tuple[CombLogic, ...]

    def __call__(self, inp, quantize=False, debug=False):
        out = np.asarray(inp)
        for sol in self.solutions:
            out = sol(out, quantize=quantize, debug=debug)
        return out

    @property
    def kernel(self) -> np.ndarray:
        return reduce(lambda x, y: x @ y, [sol.kernel.astype(np.float64) for sol in self.solutions]).astype(np.float32)

    @property
    def cost(self) -> float:
        return sum(sol.cost for sol in self.solutions)

    @property
    def n_adders(self) -> int:
        return sum(sol.n_adders for sol in self.solutions)

    @property
    def latency(self):
        return self.solutions[-1].latency

    @property
    def inp_qint(self):
        return self.solutions[0].inp_qint

    @property
    def inp_latency(self):
        return self.solutions[0].inp_latency

    @property
    def out_qint(self):
        return self.solutions[-1].out_qint

    @property
    def out_latencies(self):
        return self.solutions[-1].out_latency

    @property
    def shape(self):
        return self.solutions[0].shape[0], self.solutions[-1].shape[1]

    @property
    def inp_shifts(self):
        return self.solutions[0].inp_shifts

    @property
    def out_shift(self):
        return self.solutions[-1].out_shifts

    @property
    def out_neg(self):
        return self.solutions[-1].out_negs

    def __repr__(self) -> str:
        n_ins = [sol.shape[0] for sol in self.solutions] + [self.shape[1]]
        lo, hi = self.latency
        return f'CascatedSolution([{" -> ".join(map(str, n_ins))}], cost={self.cost}, latency={lo}-{hi})'

    def save(self, path: str | Path):
        with open(path, 'w') as f:
            json.dump(self, f, separators=(',', ':'))

    @classmethod
    def deserialize(cls, data):
        return cls(solutions=tuple(CombLogic.deserialize(sol) for sol in data[0]))

    @classmethod
    def load(cls, path: str | Path):
        with open(path) as f:
            return cls.deserialize(json.load(f))


def stage_to_binary(st, version: int = 0) -> np.ndarray:
    """DAIS program (int32 words, reference types.py:500-541) of one stage given as flat arrays (the dict layout of
    ``pipeline_from_arrays``): the same words ``CombLogic.to_binary`` produces, without building any ``Op``."""
    n_in, n_out = (int(v) for v in st['shape'])
    oi = np.asarray(st['ops_i'], dtype=np.int64).reshape(-1, 4)
    of = np.asarray(st['ops_f'], dtype=np.float32).reshape(-1, 5)
    n_ops = oi.shape[0]
    tables = st.get('lookup_tables') or []
    header = np.concatenate([[1, version, n_in, n_out, n_ops, len(tables)], np.asarray(st['inp_shifts'], dtype=np.int64), np.asarray(st['out_idxs'], dtype=np.int64), np.asarray(st['out_shifts'], dtype=np.int64), (np.asarray(st['out_negs']) != 0).astype(np.int64)]).astype(np.int32)
    code = np.zeros((n_ops, 8), dtype=np.int32)
    if n_ops:
        code[:, 0] = oi[:, 2]
        code[:, 1:3] = oi[:, 0:2]
        code[:, 3:5] = np.ascontiguousarray(oi[:, 3]).view(np.int32).reshape(-1, 2)
        code[:, 5:8] = minimal_kif_array(of[:, 0:3].astype(np.float64))
        for r in np.flatnonzero(oi[:, 2] == 8).tolist():  # lookup: pad_left << 32 | table index (LookupTable._get_pads)
            lo, _, step = of[oi[r, 0], 0:3].astype(np.float64)
            k, i, _ = code[oi[r, 0], 5:8].tolist()
            pad = round((lo + 2.0**i) / step) if k else round(lo / step)
            code[r, 3:5] = np.asarray([(pad << 32) | int(oi[r, 3])], np.int64).view(np.int32)
    if not tables:
        return np.concatenate([header, code.ravel()])
    ints = [np.asarray(t['table'], np.int32) for t in tables]
    return np.concatenate([header, code.ravel(), np.asarray([len(t) for t in ints], np.int32), *ints]).astype(np.int32)


def stage_to_jsonable(st) -> list:
    """Nested-list form of one stage, equal to what ``json.dump(CombLogic)`` writes (reference types.py:442-477)."""
    oi = np.asarray(st['ops_i'], dtype=np.int64).reshape(-1, 4).tolist()
    of = np.asarray(st['ops_f'], dtype=np.float32).reshape(-1, 5).astype(np.float64).tolist()
    ops = [[a[0], a[1], a[2], a[3], [b[0], b[1], b[2]], b[3], b[4]] for a, b in zip(oi, of)]
    return [
        [int(st['shape'][0]), int(st['shape'][1])],
        [int(v) for v in st['inp_shifts']],
        [int(v) for v in st['out_idxs']],
        [int(v) for v in st['out_shifts']],
        [bool(v) for v in st['out_negs']],
        ops,
        int(st['carry_size']),
        int(st['adder_size']),
        None,  # lookup_tables: the solver emits adder graphs only
    ]


def stages_to_json(stages) -> str:
    """JSON text of a ``Pipeline`` (``Pipeline.save``) written from the flat per-stage arrays."""
    return json.dumps([[stage_to_jsonable(st) for st in stages]], separators=(',', ':'))


try:  # C-level builder of the op list (csrc_py/fastbuild.c, compiled by __graft_entry__.build()); plain Python otherwise
    from . import _fastbuild
except ImportError:  # pragma: no cover
    _fastbuild = None


def _build_ops(ops_i, ops_f, _Op, _Q) -> list:
    """``[n,4]`` int64 + ``[n,5]`` float32 op tables -> list of ``Op`` (host-side object construction only)."""
    oi = np.ascontiguousarray(np.asarray(ops_i, dtype=np.int64).reshape(-1, 4))
    of = np.ascontiguousarray(np.asarray(ops_f, dtype=np.float32).reshape(-1, 5))
    if _fastbuild is not None and isinstance(_Op, type) and isinstance(_Q, type) and issubclass(_Op, tuple) and issubclass(_Q, tuple):
        return _fastbuild.build_ops(oi, of, _Op, _Q)
    a, b = oi.tolist(), of.astype(np.float64).tolist()
    return [_Op(x[0], x[1], x[2], x[3], _Q(y[0], y[1], y[2]), y[3], y[4]) for x, y in zip(a, b)]


def pipeline_from_arrays(stages, types_module=None) -> Pipeline:
    """Build a Pipeline from flat per-stage arrays.

    ``stages``: iterable of dicts with keys shape, inp_shifts, out_idxs, out_shifts, out_negs,
    ops_i ([n,4] int64: id0,id1,opcode,data), ops_f ([n,5] float32: min,max,step,latency,cost),
    carry_size, adder_size.  Mirrors make_py_comblogic / make_py_pipeline (bindings.cc:106-151).
    """
    T = types_module
    _Q = T.QInterval if T else QInterval
    _Op = T.Op if T else Op
    _C = T.CombLogic if T else CombLogic
    _P = T.Pipeline if T else Pipeline
    sols = []
    # ~3 tuples per op and nothing among them can form a cycle: the generational collector would only re-scan the growing
    # list over and over (measured on the 65 k ops of a 256x256 solve: 150 ms with it, 30 ms without)
    gc_was_on = gc.isenabled()
    gc.disable()
    try:
        for st in stages:
            ops = _build_ops(st['ops_i'], st['ops_f'], _Op, _Q)
            sols.append(
                _C(
                    (int(st['shape'][0]), int(st['shape'][1])),
                    np.asarray(st['inp_shifts']).astype(np.int64).tolist(),
                    np.asarray(st['out_idxs']).astype(np.int64).tolist(),
                    np.asarray(st['out_shifts']).astype(np.int64).tolist(),
                    (np.asarray(st['out_negs']) != 0).tolist(),
                    ops,
                    int(st['carry_size']),
                    int(st['adder_size']),
                )
            )
    finally:
        if gc_was_on:
            gc.enable()
    return _P(tuple(sols))
