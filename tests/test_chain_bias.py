"""Chains with biases (``act(x @ W_k + b_k)``) without a GPU: ``chain_front(..., biases=)`` on the oracle-based sweep
stand-in and the pricing kernel under the SIMT shim, ``chain_design``'s constant additions, and the split kernels and
emitters under the SIMT shim, against the reference's own traces of whole models (tests/golden/chain_bias.json.gz);
the argument checks, the constant and folding refusals, and that zero biases change nothing."""
import gzip
import json
import pickle
from pathlib import Path

import numpy as np
import pytest

import da4ml_b200._binary as B
from da4ml_b200 import emit
from da4ml_b200.cmvm import chain_design, chain_front

from golden.make_golden_chain_pipeline import text_digests
from golden.make_golden_chain_traced import digest
from simt import pipeline_split as SPLIT
from test_chain_traced import OracleSolver, OracleSweep, oracle_stages, simt_pricer
from test_pipeline_split import assert_split_equal

GOLDEN = Path(__file__).resolve().parent / 'golden' / 'chain_bias.json.gz'


def bias_golden():
    return json.loads(gzip.decompress(GOLDEN.read_bytes()))


def model(name):
    g = bias_golden()
    return g, next(m for m in g['models'] if m['name'] == name)


def model_args(m):
    kernels = [np.asarray(W, np.float32) for W in m['kernels']]
    acts = [(kind, np.asarray(kif, np.int64)) for kind, kif in m['activations']]
    qs = [[tuple(q) for q in m['qintervals']]] + [None] * (len(kernels) - 1)
    return kernels, qs, acts, m['biases'], dict(adder_size=m['adder_size'], carry_size=m['carry_size'])


def trace_designs(m, t):
    """The designs of one golden trace, re-solved from its recorded calls."""
    kernels = [np.asarray(W, np.float32) for W in m['kernels']]
    designs = [oracle_stages(W, **gc['options'], qintervals=gc['qintervals'], latencies=gc['latencies']) for W, gc in zip(kernels, t['calls'])]
    assert [digest(d) for d in designs] == [gc['digest'] for gc in t['calls']]
    return designs


def stage_positions(m, designs):
    """Index of the bias / activation stage after each layer in the chain design (None: the layer has none)."""
    pos, out = 0, []
    for k, d in enumerate(designs):
        pos += len(d)
        if k < len(m['activations']) or m['biases'][k] is not None:
            out.append(pos)
            pos += 1
        else:
            out.append(None)
    return out


def stated_cost(d, m, designs, layer_costs):
    """The float32 sum in stage order of the chain design's cost column, each layer's cost taken as one value."""
    cost = np.float32(0.0)
    for k, (c, pos) in enumerate(zip(layer_costs, stage_positions(m, designs))):
        cost = np.float32(cost + np.float32(c))
        if pos is not None:
            for v in np.asarray(d.stages[pos]['ops_f'], np.float32)[:, 4]:
                cost = np.float32(cost + v)
    return cost


OK_MODELS = ['bias_relu_wrap_6x5x4x3', 'frac_dead_zero_bias_8x6x3']


@pytest.mark.parametrize('name', OK_MODELS)
@pytest.mark.parametrize('c', [3.0, 5.0])
def test_front_matches_the_tracer(name, c):
    g, m = model(name)
    kernels, qs, acts, biases, cm = model_args(m)
    cf = chain_front(kernels, g['sets'], qintervals=qs, latency_cutoff=c, activations=acts, biases=biases, solver=OracleSolver(), pricer=simt_pricer, **cm)
    traces = {(tuple(t['choice']), t['cutoff']): t for t in m['traces']}
    assert len(cf) >= 1
    for p in range(len(cf)):
        calls = cf.reference_calls(p)
        choice = tuple(next(s for s, o in enumerate(g['sets']) if all(call[key] == v for key, v in o.items())) for call in calls)
        t = traces[choice, c]
        for k, (call, gc) in enumerate(zip(calls, t['calls'])):
            assert np.array_equal(np.asarray(call['qintervals'], np.float32), np.asarray(gc['qintervals'], np.float32)), (name, choice, k)
            assert call['latencies'] == gc['latencies'], (name, choice, k)
            assert digest(cf.raw(p, k).stages) == gc['digest'], (name, choice, k)
        designs = [cf.raw(p, k).stages for k in range(len(kernels))]
        d = cf.design(p)
        assert cf.cost[p].view(np.uint32) == stated_cost(d, m, designs, [gc['cost'] for gc in t['calls']]).view(np.uint32), (name, choice)
        assert float(cf.latency[p]) == max(t['out_latency']), (name, choice)
    best = min(stated_cost(chain_design(ds, acts, biases), m, ds, [gc['cost'] for gc in t['calls']])
               for t in m['traces'] if t['cutoff'] == c for ds in [trace_designs(m, t)])  # fmt: skip
    assert float(cf.cost.min()) == float(best)
    assert all(layer['dropped_constant'] == 0 and layer['dropped_folded'] == 0 for layer in cf.profile['layers'])
    assert pickle.loads(pickle.dumps(cf)).biases[0].tolist() == cf.biases[0].tolist()


@pytest.mark.parametrize('name', OK_MODELS)
def test_chain_design_bias_ops_match_the_tracer(name):
    _, m = model(name)
    _, _, acts, biases, _ = model_args(m)
    n = 0
    for t in m['traces']:
        designs = trace_designs(m, t)
        d = chain_design(designs, acts, biases)
        for k, pos in enumerate(stage_positions(m, designs)):
            recs = t['bias_ops'][k]
            if pos is None or recs is None:
                continue
            st = d.stages[pos]
            for j, rec in enumerate(recs):
                reads = st['ops_i'][:, 0] == j
                ops = np.flatnonzero(reads & (st['ops_i'][:, 2] == 4))
                if rec is None:
                    assert ops.size == 0, (name, k, j)
                    continue
                opcode, data, q, cost = rec
                (o,) = ops
                assert st['ops_i'][o].tolist() == [j, -1, opcode, data], (name, k, j)
                assert st['ops_f'][o].tolist() == np.asarray([*q, st['ops_f'][j, 3], cost], np.float32).tolist(), (name, k, j)
                later = st['ops_i'][o + 1 :]
                assert (later[:, 0] != j).all() or (later[:, 2] != 4).all()
                n += 1
    assert n > 20


def _check_splits(name, threads=64):
    _, m = model(name)
    _, _, acts, biases, _ = model_args(m)
    n = 0
    for t in m['traces']:
        d = chain_design(trace_designs(m, t), acts, biases)
        for rt, key in ((False, 'split'), (True, 'retimed')):
            pr = SPLIT.split([d], [t['cutoff']], None, rt, threads=threads)
            tag = (name, t['choice'], t['cutoff'], rt)
            assert int(pr.status[0, 0]) == 0, tag
            if pr._out_lat[0] is not None:
                assert pr.out_latency(0, 0).tolist() == t['out_latency'], tag
            r = t[key]
            assert (int(pr.stages[0, 0]), int(pr.reg_bits[0, 0])) == (r['stages'], r['reg_bits']), tag
            if rt:
                assert float(pr.cutoff[0, 0]) == r['cutoff'], tag
            sp = pr.split(0, 0)
            assert_split_equal(sp, r, tag)
            if r['text'] is not None:
                got = text_digests(emit.verilog_pipeline_logic_gen(sp, 'chain', print_latency=True), emit.vhdl_pipeline_logic_gen(sp, 'chain'),
                                   [emit.hls_logic_and_bridge_gen(s, f'chain{k}', 'vitis', print_latency=True) for k, s in enumerate(sp)])  # fmt: skip
                assert got == r['text'], tag
            n += 1
    return n


@pytest.mark.parametrize('name', OK_MODELS)
def test_simulated_split_and_text_equal_reference(name):
    assert _check_splits(name) >= 16


def test_golden_covers_the_cases():
    g = bias_golden()
    recs = [r for m in g['models'] for t in m['traces'] for ops in t.get('bias_ops') or [] for r in ops or []]
    data = [r for r in recs if isinstance(r, list) and r[0] == 4]
    assert any(r[1] > 0 for r in data) and any(r[1] < 0 for r in data) and None in recs
    assert any(r[2][2] < 1.0 for r in data)  # a fractional bias step
    assert any(isinstance(r, list) and r[0] == 'const' for r in recs) and 'folded' in recs
    opc = {o[2] for m in g['models'] for t in m['traces'] if t.get('split') and 'full' in t['split'] for st in t['split']['full'] for o in st['ops_i']}
    assert {4, 2, 3} <= opc


def test_constant_and_folded_biases_are_refused():
    g, m = model('dead_nonzero_bias_5x4x3')
    kernels, qs, acts, biases, cm = model_args(m)
    t = m['traces'][0]
    with pytest.raises(ValueError, match='constant'):
        chain_design(trace_designs(m, t), acts, biases)
    solver = OracleSolver()
    with pytest.raises(ValueError, match='non-zero constant'):
        chain_front(kernels, g['sets'], qintervals=qs, activations=acts, biases=biases, solver=solver, **cm)
    assert len(solver.calls) == 1  # (refused in layer 0's replay: the constant is the layer's own)
    g, m = model('folded_bias_4x4x3')
    kernels, qs, acts, biases, cm = model_args(m)
    for t in m['traces']:
        with pytest.raises(ValueError, match='folds'):
            chain_design(trace_designs(m, t), acts, biases)
    with pytest.raises(ValueError, match='folds'):
        chain_front(kernels, g['sets'], qintervals=qs, activations=acts, biases=biases, solver=OracleSolver(), **cm)
    # without the folding column's bias the same model is covered
    ok = [biases[0], [0.0, 0.0, -0.25]]
    cf = chain_front(kernels, g['sets'], qintervals=qs, activations=acts, biases=ok, solver=OracleSolver(), **cm)
    assert len(cf) >= 1 and all(layer['dropped_folded'] == 0 for layer in cf.profile['layers'])


def test_argument_errors_come_before_any_solve():
    g, m = model('bias_relu_wrap_6x5x4x3')
    kernels, qs, acts, biases, cm = model_args(m)
    cases = [([None, None], 'need 3 biases'), ([[1.0] * 4, None, None], r'shape \(5,\)'), ([[np.nan] * 5, None, None], 'finite'),
             ([[2.0**-40] * 5, None, None], r'2\*\*-32'), ([['x'] * 5, None, None], 'bias 0')]  # fmt: skip
    for bad, msg in cases:
        solver = OracleSolver()
        with pytest.raises(ValueError, match=msg):
            chain_front(kernels, g['sets'], qintervals=qs, activations=acts, biases=bad, solver=solver, **cm)
        assert solver.calls == []
    with pytest.raises(ValueError, match='need activations'):
        chain_front(kernels, g['sets'], qintervals=qs, biases=biases, solver=OracleSolver(), **cm)
    t = m['traces'][0]
    designs = trace_designs(m, t)
    for bad, msg in cases:
        with pytest.raises(ValueError, match=msg):
            chain_design(designs, acts, bad)
    with pytest.raises(ValueError, match='not exact'):  # (lo + b needs more bits than float32 has)
        chain_design(designs, acts, [[2.0**-30] * 5, None, None])


def test_zero_biases_change_nothing():
    g, m = model('bias_relu_wrap_6x5x4x3')
    kernels, qs, acts, _, cm = model_args(m)
    fronts = [chain_front(kernels, g['sets'], qintervals=qs, latency_cutoff=3.0, activations=acts, solver=OracleSolver(), pricer=simt_pricer, **cm, **kw)
              for kw in ({}, dict(biases=None), dict(biases=[None, np.zeros(4), [0.0] * 3]))]  # fmt: skip
    a = fronts[0]
    for b in fronts[1:]:
        assert a.cost.tobytes() == b.cost.tobytes() and a.latency.tobytes() == b.latency.tobytes() and np.array_equal(a.choice, b.choice)
        assert b.biases is None and 'biases' not in b.__dict__
        for p in range(len(a)):
            assert a.reference_calls(p) == b.reference_calls(p)
            assert all(np.array_equal(x['ops_f'], y['ops_f']) and np.array_equal(x['ops_i'], y['ops_i']) for x, y in zip(a.design(p).stages, b.design(p).stages))
    t = m['traces'][0]
    designs = trace_designs(m, t)
    x, y = chain_design(designs, acts), chain_design(designs, acts, [np.zeros(5), None, np.zeros(3)])
    assert len(x.stages) == len(y.stages) and all(np.array_equal(s['ops_f'], r['ops_f']) for s, r in zip(x.stages, y.stages))


def test_design_refuses_other_biases():
    g, m = model('bias_relu_wrap_6x5x4x3')
    kernels, qs, acts, biases, cm = model_args(m)
    cf = chain_front(kernels, g['sets'], qintervals=qs, activations=acts, biases=biases, solver=OracleSolver(), **cm)
    assert cf.design(0, biases=biases).stages[-1]['ops_i'].tolist() == cf.design(0).stages[-1]['ops_i'].tolist()
    with pytest.raises(ValueError, match='differ'):
        cf.design(0, biases=[None, None, [1.0, 1.0, 1.0]])


def test_retrace_refuses_constant_additions():
    _, m = model('bias_relu_wrap_6x5x4x3')
    _, _, acts, biases, _ = model_args(m)
    d = chain_design(trace_designs(m, m['traces'][0]), acts, biases)
    with pytest.raises(ValueError, match='opcode 4'):
        emit.retime_pipeline(d.stages)


def test_pricing_checks_constant_additions_on_the_host():
    _, m = model('bias_relu_wrap_6x5x4x3')
    _, _, acts, biases, _ = model_args(m)
    d = chain_design(trace_designs(m, m['traces'][0]), acts, biases)
    stages = [dict(st) for st in d.stages]
    k = next(i for i, st in enumerate(stages) if (st['ops_i'][:, 2] == 4).any())
    st = stages[k] = dict(stages[k], ops_i=stages[k]['ops_i'].copy())
    r = int(np.flatnonzero(st['ops_i'][:, 2] == 4)[0])
    st['ops_i'][r, 3] = 0  # (the tracer records no constant addition of 0)
    with pytest.raises(ValueError, match='opcode 4'):
        SPLIT.split([stages], 2.0)


class MixedSolver(OracleSolver):
    """``OracleSolver`` whose sweep of layer ``k`` also holds the designs of ``alt[k]`` (a second kernel of the same
    shape), and keeps every candidate on its front: a stand-in whose candidates differ in which bias pairs are dropped."""

    def __init__(self, alt):
        super().__init__()
        self.alt, self.sweeps = alt, []

    def __call__(self, kernels, option_sets, qintervals=None, latencies=None, adder_size=-1, carry_size=-1):
        k = len(self.calls)
        sweeps = super().__call__(kernels, option_sets, qintervals, latencies, adder_size, carry_size)
        if self.alt.get(k) is not None:
            for sw, q, l in zip(sweeps, qintervals, latencies):
                other = OracleSweep(self.alt[k], option_sets, q, l, adder_size, carry_size)
                sw._designs += other._designs
                sw._sets = sw._sets + other._sets
                sw.candidates = {key: np.concatenate([sw.candidates[key], other.candidates[key]]) for key in sw.candidates}
        for sw in sweeps:
            sw.front = np.arange(len(sw._designs), dtype=np.int64)
        self.sweeps.append(sweeps)
        return sweeps


@pytest.mark.parametrize('case', ['constant', 'folded', 'inexact'])
def test_drop_counters_count_the_dropped_pairs(case):
    """A layer whose candidates come from two kernels, one of which makes the dropped case: exactly that kernel's
    candidates are dropped and counted, and the front is made of the other's."""
    g = bias_golden()
    sets = g['sets']
    if case == 'constant':  # the golden kernel's dead column 1 gets a non-zero bias; the other kernel's column is not dead
        _, m = model('dead_nonzero_bias_5x4x3')
        kernels, qs, acts, biases, cm = model_args(m)
        alt = kernels[0].copy()
        alt[0, 1] = 3.0
        layer, alt_map = 0, {0: alt}
    elif case == 'folded':  # layer 1's column 0 passes its biased input 0 through; the other kernel's column does not
        _, m = model('folded_bias_4x4x3')
        kernels, qs, acts, biases, cm = model_args(m)
        sets = sets[:1]
        alt = kernels[1].copy()
        alt[1, 0] = 1.0
        layer, alt_map = 1, {1: alt}
    else:  # a bias of 2**-20 on a value of [-8, 7] is exact in float32, on the golden kernel's wide sum it is not
        _, m = model('bias_relu_wrap_6x5x4x3')
        kernels, qs, acts, _, cm = model_args(m)
        biases = [[2.0**-20, 0.0, 0.0, 0.0, 0.0], None, None]
        alt = kernels[0].copy()
        alt[:, 0] = 0.0
        alt[0, 0] = 1.0
        layer, alt_map = 0, {0: alt}
    solver = MixedSolver(alt_map)
    cf = chain_front(kernels, sets, qintervals=qs, activations=acts, biases=biases, solver=solver, **cm)
    counts = {key: [layer_[f'dropped_{key}'] for layer_ in cf.profile['layers']] for key in ('constant', 'folded', 'inexact')}
    n_states = cf.profile['layers'][layer]['states']
    assert counts[case][layer] == len(sets) * n_states, counts  # (one replay group per state here)
    assert sum(sum(v) for v in counts.values()) == counts[case][layer], counts
    if case == 'inexact':
        with pytest.raises(ValueError, match='not exact'):
            chain_design([oracle_stages(kernels[0], **sets[0], qintervals=qs[0])], [], [biases[0]])


def test_traced_split_computes_the_traced_model():
    """The SIMT split of the chain design of option set 0 at cutoff 5, each stage run by the reference's DAIS
    interpreter on the golden's input rows, gives the traced model's outputs exactly."""
    from oracle import dais_ref

    if not dais_ref.available():
        pytest.skip("the reference's DAIS interpreter is not built")
    for name in OK_MODELS:
        _, m = model(name)
        _, _, acts, biases, _ = model_args(m)
        t = next(t for t in m['traces'] if t['choice'] == [0] * len(m['kernels']) and t['cutoff'] == 5.0)
        d = chain_design(trace_designs(m, t), acts, biases)
        for rt in (False, True):
            x = np.asarray(m['rows'], np.float64)
            for st in SPLIT.split([d], [5.0], None, rt, threads=64).split(0, 0):
                x = dais_ref.run(np.asarray(B.RawPipeline.from_stages([st]).to_binary()[0]), x)
            assert x.tolist() == m['outputs'], (name, rt)
