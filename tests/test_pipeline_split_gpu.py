"""Register stages of solver designs on the GPU: ``price_pipelined(..., keep_split=True).split(d, j)`` against the reference's
own splits (tests/golden/pipeline_split.json.gz), against ``emit``'s re-trace / split / retiming on live solves,
``SweepResult.pipelined(c, keep_split=True)`` and the Verilog the emitters make of a split."""
import numpy as np
import pytest

import da4ml_b200._binary as B
from da4ml_b200 import emit

from test_pipeline_price import _emit_split_numbers
from test_pipeline_price_gpu import _live_designs
from test_pipeline_split import check_splits_against_golden

pytestmark = pytest.mark.gpu

CUTS = [2.0, 3.0, 5.0, 8.0]


def test_split_equals_reference():
    check_splits_against_golden(lambda ds, cuts, lats, rt: B.price_pipelined(ds, cuts, lats, rt, keep_split=True))


def _assert_stages_equal(got, want, tag):
    assert len(got) == len(want), tag
    for a, b in zip(got, want):
        assert tuple(a['shape']) == tuple(b['shape']), tag
        for k in ('inp_shifts', 'out_idxs', 'out_shifts', 'out_negs', 'ops_i'):
            assert np.array_equal(np.asarray(a[k], np.int64), np.asarray(b[k], np.int64)), (tag, k)
        assert a['ops_f'].dtype == np.float64
        assert np.array_equal(a['ops_f'].view(np.uint64), np.asarray(b['ops_f'], np.float64).view(np.uint64)), tag  # (bit for bit)
        assert (a['adder_size'], a['carry_size']) == (b['adder_size'], b['carry_size']), tag


def _live():
    designs = []
    for W, kw in _live_designs():
        kw = {k: v for k, v in kw.items() if k in ('method0', 'method1', 'hard_dc', 'decompose_dc', 'qintervals', 'adder_size', 'carry_size')}
        designs.append([emit.as_stage(s) for s in B.solve_raw(W, **kw).stages])
    return designs


def test_split_equals_emit_on_live_solves():
    designs = _live()
    n_split = 0
    for rt in (False, True):
        pr = B.price_pipelined(designs, CUTS, retiming=rt, keep_split=True)
        plain = B.price_pipelined(designs, CUTS, retiming=rt)
        for key in ('status', 'stages', 'reg_bits'):
            assert np.array_equal(getattr(pr, key), getattr(plain, key)), key
        for key in ('latency_max', 'cutoff'):
            assert np.array_equal(getattr(pr, key), getattr(plain, key), equal_nan=True), key
        assert pr.profile['split_launches'] == 2 and pr.profile['launches'] == plain.profile['launches'] + 2
        for d, stages in enumerate(designs):
            for j, c in enumerate(CUTS):
                if int(pr.status[d, j]) != 0:
                    with pytest.raises(ValueError, match='is not ok'):
                        pr.split(d, j)
                    continue
                want = emit.to_pipeline(emit._retrace(stages, c, B.cost_add), c, retiming=rt)
                got = pr.split(d, j)
                _assert_stages_equal(got, want, (d, c, rt))
                assert _emit_split_numbers(got) == (int(pr.stages[d, j]), int(pr.reg_bits[d, j])), (d, c, rt)
                n_split += 1
    assert n_split > 30


def test_sweep_pipelined_split_equals_per_candidate():
    rng = np.random.default_rng(3)
    W = rng.integers(-32, 32, size=(24, 20)).astype(np.float32)
    sets = [dict(method0=m, hard_dc=h) for m in ('wmc', 'mc') for h in (-1, 1, 3)]
    lat = [float(v) for v in rng.choice([0.0, 1.0, 2.0], size=24)]
    sw = B.solve_sweep(W, sets, latencies=lat, adder_size=4, carry_size=2, keep_all=True)
    for rt in (False, True):
        pr = sw.pipelined([3.0, 6.0], retiming=rt, keep_split=True)
        for i in range(len(sw)):
            one = B.price_pipelined([sw.raw(i)], [3.0, 6.0], latencies=[lat], retiming=rt, keep_split=True)
            for j in range(2):
                if int(one.status[0, j]) != 0:
                    continue
                _assert_stages_equal(pr.split(i, j), one.split(0, j), (i, j, rt))


def test_split_through_verilog():
    W = np.random.default_rng(5).integers(-64, 64, size=(16, 12)).astype(np.float32)
    stages = [emit.as_stage(s) for s in B.solve_raw(W).stages]
    cuts = [2.0, 3.0, 5.0]
    pr = B.price_pipelined([stages], cuts, keep_split=True)
    j = next(j for j in range(len(cuts)) if pr.status[0, j] == 0 and pr.stages[0, j] > 1)
    want = emit.to_pipeline(emit._retrace(stages, cuts[j], B.cost_add), cuts[j], retiming=True)
    assert emit.verilog_pipeline_logic_gen(pr.split(0, j), 'dut', print_latency=True) == emit.verilog_pipeline_logic_gen(want, 'dut', print_latency=True)
