"""Chains with leaky ReLU activations on the GPU: ``price_pipelined(keep_split=True)`` of a chain design with MSB muxes
against the SIMT run and the reference's splits (tests/golden/chain_leaky.json.gz), one call mixing leaky and plain
designs against separate calls, hand-made muxes on a condition of their own (opcodes 6 and -6), the split's DAIS
programs through ``DaisProgram`` against the traced model's outputs, and ``chain_front`` with the real sweeps and
pricing against the reference's traces."""
import numpy as np
import pytest

from da4ml_b200._binary import price_pipelined
from da4ml_b200.cmvm import chain_design
from da4ml_b200.dais import DaisProgram
from da4ml_b200.types import stage_to_binary

from simt import pipeline_split as SPLIT
from test_chain_bias import trace_designs
from test_chain_leaky import MODELS, acts_of, check_hand_muxes, golden, hand_design, model, stated_cost
from test_chain_lookup import emitted, tables_of
from test_pipeline_split import assert_split_equal

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('name', MODELS)
def test_gpu_split_equals_simt_and_golden(name):
    m = model(name)
    t = next(t for t in m['traces'] if t['choice'] == [0] * len(m['kernels']) and t['cutoff'] == 3.0)
    d = chain_design(trace_designs(m, t), acts_of(m), m['biases'])
    for retiming, rec in ((False, t['split']), (True, t['retimed'])):
        gpu = price_pipelined([d], 3.0, retiming=retiming, keep_split=True)
        sim = SPLIT.split([d], 3.0, retiming=retiming)
        assert int(gpu.reg_bits[0, 0]) == int(sim.reg_bits[0, 0]) == rec['reg_bits']
        assert_split_equal(gpu.split(0, 0), rec, (name, retiming))
        assert tables_of(gpu.split(0, 0)) == rec['tables']
        assert emitted(gpu.split(0, 0)) == (rec['text'], rec['mem'])
        if not retiming:
            np.testing.assert_array_equal(gpu.out_latency(0, 0), t['out_latency'])


def test_hand_muxes_split_equal_the_tracer():
    """MSB muxes on a condition of their own (opcodes 6 and -6) under late inputs: the GPU split is the reference's, and
    the traced output latencies are the tracer's."""
    assert check_hand_muxes(lambda d, c, lats, rt: price_pipelined([d], c, None if lats is None else [lats], retiming=rt, keep_split=True)) >= 16
    d = hand_design()
    for t in golden()['hand_muxes']['tasks']:
        pr = price_pipelined([d], t['cutoff'], None if t['latencies'] is None else [t['latencies']], retiming=False)
        np.testing.assert_array_equal(pr.out_latency(0, 0), t['out_latency'])


def test_mixed_call_equals_separate_calls():
    m = model('leaky_quantize_5x6x3')
    t = m['traces'][0]
    ds = trace_designs(m, t)
    leaky = chain_design(ds, acts_of(m))
    plain = chain_design(ds, [('quantize', (1, 6, 2))])
    both = price_pipelined([leaky, plain], [2.0, 5.0], keep_split=True)
    for i, d in enumerate((leaky, plain)):
        one = price_pipelined([d], [2.0, 5.0], keep_split=True)
        for key in ('status', 'stages', 'reg_bits', 'latency_max', 'cutoff'):
            np.testing.assert_array_equal(getattr(both, key)[i], getattr(one, key)[0])
        for j in range(2):
            a, b = both.split(i, j), one.split(0, j)
            assert all(np.array_equal(x['ops_i'], y['ops_i']) and np.array_equal(x['ops_f'], y['ops_f']) for x, y in zip(a, b))


@pytest.mark.parametrize('name', MODELS)
def test_dais_program_runs_the_traced_model(name):
    m = model(name)
    t = next(t for t in m['traces'] if t['choice'] == [0] * len(m['kernels']) and t['cutoff'] == 5.0)
    d = chain_design(trace_designs(m, t), acts_of(m), m['biases'])
    x = np.asarray(m['rows'], np.float64)
    for st in price_pipelined([d], 5.0, retiming=False, keep_split=True).split(0, 0):
        with DaisProgram(stage_to_binary(st)) as prog:
            x = np.asarray(prog(x), np.float64)
    np.testing.assert_array_equal(x, np.asarray(m['outputs'], np.float64))


@pytest.mark.parametrize('name', ['leaky_quantize_5x6x3', 'leaky_negated_3x4x2', 'bias_leaky_4x4x2', 'wide_leaky_4x3x2', 'leaky_noop_2x4x2', 'leaky_noop_relu_2x4x2'])
@pytest.mark.parametrize('c', [3.0, 5.0])
def test_front_equals_the_tracer(cuda_binary, name, c):
    """The real ``solve_sweep_batch`` and ``price_pipelined`` in ``chain_front``: every point is its choice's trace
    (designs, reference calls, cost, traced latency), and every design is what ``solve`` returns under its reference
    call."""
    import da4ml_b200._binary as B
    from golden.make_golden_chain_traced import digest

    g, m = golden(), model(name)
    kernels = [np.asarray(W, np.float32) for W in m['kernels']]
    cf = B.chain_front(kernels, g['sets'], qintervals=[[tuple(q) for q in m['qintervals']], None], latency_cutoff=c, activations=acts_of(m),
                       biases=m['biases'], adder_size=m['adder_size'], carry_size=m['carry_size'])  # fmt: skip
    traces = {(tuple(t['choice']), t['cutoff']): t for t in m['traces']}
    assert len(cf) > 0
    for p in range(len(cf)):
        calls = cf.reference_calls(p)
        t = traces[tuple(int(v) for v in cf.choice[p]), c]
        assert [call['latencies'] for call in calls] == [gc['latencies'] for gc in t['calls']], (name, c, p)
        assert [[list(q) for q in call['qintervals']] for call in calls] == [gc['qintervals'] for gc in t['calls']], (name, c, p)
        for k, (W, gc) in enumerate(zip(kernels, t['calls'])):
            assert digest(cf.raw(p, k).stages) == gc['digest'], (name, c, p, k)
            assert digest(B.solve_raw(W, **calls[k]).stages) == gc['digest'], (name, c, p, k)
        designs = [cf.raw(p, k).stages for k in range(len(kernels))]
        assert cf.cost[p].view(np.uint32) == stated_cost(cf.design(p), m, designs, [gc['cost'] for gc in t['calls']]).view(np.uint32), (name, c, p)
        assert float(cf.latency[p]) == max(t['out_latency']), (name, c, p)
