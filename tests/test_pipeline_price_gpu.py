"""Pipelined pricing on the GPU: ``price_pipelined`` against the reference tracer's answers (tests/golden/pipeline_price.json.gz),
against ``emit``'s re-trace / split / retiming on live solves, ``SweepResult.pipelined`` and ``chain_front(latency_cutoff=c)``."""
import numpy as np
import pytest

import da4ml_b200._binary as B
from da4ml_b200 import emit

from test_pipeline_price import _emit_split_numbers, check_against_golden

pytestmark = pytest.mark.gpu


def test_price_equals_reference_tracer():
    check_against_golden(lambda ds, cuts, lats, rt: B.price_pipelined(ds, cuts, lats, rt))


def _emit_answer(stages, c, retiming):
    try:
        comb = emit._retrace(stages, c, B.cost_add)
    except AssertionError:
        return 1, None
    except NotImplementedError:
        return 2, None
    o = [float(comb['ops_f'][i, 3]) if i >= 0 else 0.0 for i in comb['out_idxs']]
    return 0, (_emit_split_numbers(emit.to_pipeline(comb, c, retiming=retiming)), o)


def _live_designs():
    from conftest import golden_cases, load_golden

    ks = []
    for name in ['c1_8x8_int4_default', 'int_16x16_int8_default', 'int_32x32_int8_default', 'int_40x56_int6_mcdc_dc1', 'int_48x40_int8_harddc2_wmcpdc']:
        kw = dict(golden_cases()[name]['kwargs'])
        extra, _ = load_golden(name)
        ks.append((extra['kernel'].astype(np.float32), kw))
    rng = np.random.default_rng(17)
    for n, b in [(16, 6), (48, 8), (96, 6), (128, 8)]:
        ks.append((rng.integers(-(2 ** (b - 1)), 2 ** (b - 1), size=(n, n)).astype(np.float32), dict(adder_size=int(rng.integers(1, 8)), carry_size=int(rng.integers(1, 4)))))
    return ks


def test_price_equals_emit_on_live_solves():
    cuts = [2.0, 3.0, 5.0, 8.0]
    designs = []
    for W, kw in _live_designs():
        kw = {k: v for k, v in kw.items() if k in ('method0', 'method1', 'hard_dc', 'decompose_dc', 'qintervals', 'adder_size', 'carry_size')}
        designs.append([emit.as_stage(s) for s in B.solve_raw(W, **kw).stages])
    for rt in (False, True):
        pr = B.price_pipelined(designs, cuts, retiming=rt)
        assert pr.profile['launches'] >= 1
        for d, stages in enumerate(designs):
            for j, c in enumerate(cuts):
                st, ans = _emit_answer(stages, c, rt)
                assert int(pr.status[d, j]) == st, (d, c, rt)
                if st:
                    continue
                (n_st, bits), o = ans
                assert (int(pr.stages[d, j]), int(pr.reg_bits[d, j])) == (n_st, bits), (d, c, rt)
                assert list(pr.out_latency(d, j)) == o and float(pr.latency_max[d, j]) == max(o)


def test_sweep_pipelined_equals_per_candidate_pricing():
    rng = np.random.default_rng(3)
    W = rng.integers(-32, 32, size=(24, 20)).astype(np.float32)
    sets = [dict(method0=m, hard_dc=h) for m in ('wmc', 'mc') for h in (-1, 1, 3)]
    lat = [float(v) for v in rng.choice([0.0, 1.0, 2.0], size=24)]
    for keep_all in (False, True):
        sw = B.solve_sweep(W, sets, latencies=lat, adder_size=4, carry_size=2, keep_all=keep_all)
        pr = sw.pipelined([3.0, 6.0], retiming=False)
        assert pr.status.shape == (len(sw), 2)
        for i in range(len(sw)):
            if not sw.candidates['kept'][i]:
                assert (pr.status[i] == -1).all() and np.isnan(pr.latency_max[i]).all()
                continue
            one = B.price_pipelined([sw.raw(i)], [3.0, 6.0], latencies=[lat], retiming=False)
            for key in ('status', 'stages', 'reg_bits'):
                assert np.array_equal(getattr(pr, key)[i], getattr(one, key)[0]), key
            for key in ('cutoff', 'latency_max'):  # (NaN where a task is not ok)
                assert np.array_equal(getattr(pr, key)[i], getattr(one, key)[0], equal_nan=True), key
        if keep_all:
            assert (pr.status >= 0).all()


@pytest.mark.parametrize('c', [3.0, 5.0])
def test_chain_front_pipelined(c):
    rng = np.random.default_rng(11)
    kernels = [rng.integers(-32, 32, size=(12, 12)).astype(np.float32) for _ in range(3)]
    sets = [dict(method0='wmc'), dict(method0='wmc', hard_dc=2), dict(method0='mc', decompose_dc=1)]
    front = B.chain_front(kernels, sets, latencies=[0.0] * 12, latency_cutoff=c, adder_size=-1, carry_size=12)
    assert len(front) > 0 and len(front.profile['layers']) == 3
    assert np.array_equal(front.stages, np.floor(front.latency.astype(np.float64) / (c + 1e-9)).astype(np.int64) + 1)
    for n in sorted(set(front.stages.tolist())):
        assert front.best_stages(n).cost == float(front.cost[front.stages <= n].min())
    for p in range(len(front)):
        calls = front.reference_calls(p)
        lats = [0.0] * 12
        for k, call in enumerate(calls):
            assert call['latencies'] == lats
            raw = front.raw(p, k)
            ref = B.solve_raw(kernels[k], **call)
            for a, b in zip(raw.stages, ref.stages):
                assert np.array_equal(a['ops_i'], b['ops_i']) and np.array_equal(a['ops_f'], b['ops_f'])
            pr = B.price_pipelined([raw], c, latencies=[lats], retiming=False)
            assert int(pr.status[0, 0]) == 0
            lats = [float(v) for v in pr.out_latency(0, 0)]
        assert max(lats) == float(front.latency[p])
