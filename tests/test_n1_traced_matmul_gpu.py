"""SURVEY 8f N1, CUDA side: the calling pattern of the reference's tracing front-end
(``da4ml.trace.FixedVariableArray.matmul``, trace/fixed_variable_array.py:361-373: a Python loop over the left-hand rows,
each calling ``cmvm()`` -> ``solve(W, qintervals=row intervals, latencies=row latencies, **solver_options)``) through
``SolveBatcher``: all rows in ONE batched GPU solve, identical rows solved once.  Every row's adder graph is compared with the
call-by-call CUDA result and with the CPU checker."""
import numpy as np
import pytest
from conftest import assert_stage_equal, int_matrix

import oracle
from da4ml_b200.batching import CmvmCall, SolveBatcher


def traced_rows(n_rows, n_in, seed):
    """Per-row input intervals / latencies as a traced (N, F) activation array would carry them."""
    rng = np.random.default_rng(seed)
    rows = []
    for r in range(n_rows):
        q = [(-float(2 ** rng.integers(1, 6)), float(2 ** rng.integers(1, 6)) - 1.0, 1.0) for _ in range(n_in)]
        lat = [float(v) for v in rng.integers(0, 3, n_in)]
        rows.append((q, lat))
    rows[2] = rows[0]  # two identical rows: solved once
    return rows


@pytest.mark.gpu
def test_rows_of_a_matmul_batched_equal_call_by_call_and_checker(cuda_binary):
    mod, _ = oracle.best()
    W = int_matrix(24, 18, 6, 77)
    rows = traced_rows(5, 24, 5)
    opts = dict(adder_size=-1, carry_size=-1, hard_dc=2)

    def matmul(solve):  # the calling pattern of FixedVariableArray.matmul: one solve per row, results used in order
        return [solve(W, qintervals=q, latencies=lat, **opts) for q, lat in rows]

    batcher = SolveBatcher()
    pipes = batcher.run(lambda: matmul(batcher.solve))
    assert len(batcher.calls) == 5 and len(pipes) == 5
    assert batcher.raw[0] is batcher.raw[2]  # identical calls share one solve
    seq = [cuda_binary.solve_raw(W, qintervals=q, latencies=lat, **opts) for q, lat in rows]
    for i, ((q, lat), raw, one) in enumerate(zip(rows, batcher.raw, seq, strict=True)):
        want = mod.solve(W, qintervals=q, latencies=lat, **opts)
        for s, (a, b, c) in enumerate(zip(raw.stages, want, one.stages, strict=True)):
            assert_stage_equal(a, b, f'row {i} stage {s} (batched vs checker) ')
            assert_stage_equal(c, b, f'row {i} stage {s} (call by call vs checker) ')
        assert np.array_equal(pipes[i].kernel, W)
    # a second pass that asks for something else is refused
    with pytest.raises(RuntimeError, match='different solve'):
        flip = {'n': 0}

        def odd():
            flip['n'] += 1
            return batcher.solve(W if flip['n'] == 1 else W * 2, **opts)

        batcher.run(odd)


@pytest.mark.gpu
def test_results_in_the_reference_result_types(cuda_binary):
    """``to_pipeline(types_module=...)`` with a stand-in for the reference's ``da4ml.types``: field-for-field the same
    containers, built by the caller's classes (bindings.cc:106-151 imports da4ml.types at call time)."""
    import types as pytypes
    from typing import NamedTuple

    class QInterval(NamedTuple):
        min: float
        max: float
        step: float

    class Op(NamedTuple):
        id0: int
        id1: int
        opcode: int
        data: int
        qint: QInterval
        latency: float
        cost: float

    class CombLogic(NamedTuple):
        shape: tuple
        inp_shifts: list
        out_idxs: list
        out_shifts: list
        out_negs: list
        ops: list
        carry_size: int
        adder_size: int

    class Pipeline(NamedTuple):
        solutions: tuple

    T = pytypes.SimpleNamespace(QInterval=QInterval, Op=Op, CombLogic=CombLogic, Pipeline=Pipeline)
    W = int_matrix(9, 7, 5, 3)
    raw = cuda_binary.solve_raw(W)
    theirs, ours = raw.to_pipeline(T), raw.to_pipeline()
    assert type(theirs) is Pipeline and type(theirs.solutions[0]) is CombLogic and type(theirs.solutions[0].ops[0]) is Op
    for a, b in zip(theirs.solutions, ours.solutions, strict=True):
        assert tuple(a) == tuple(b)[: len(tuple(a))]  # (this repository's mirror also carries the reference's trailing optional field)
