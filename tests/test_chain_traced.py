"""chain_front with activations (each layer solved under the intervals its relu / quantizer hands it) without a GPU: the
search on an oracle-based sweep stand-in and the pricing kernel under the SIMT shim, against the reference's own traces
of whole models (tests/golden/chain_traced.json.gz); the argument checks; a relu that saturates every value against the
intervals given by hand; and one problem per distinct state."""
import gzip
import json
import pickle
from pathlib import Path

import numpy as np
import pytest

import da4ml_b200._binary as B

from golden.make_golden_chain_traced import digest, seq_cost
from simt import pipeline_price as SIM

GOLDEN = Path(__file__).resolve().parent / 'golden' / 'chain_traced.json.gz'


def traced_golden():
    return json.loads(gzip.decompress(GOLDEN.read_bytes()))


def model_args(m):
    """(kernels, qintervals, activations, adder_size / carry_size keywords) of a golden model."""
    kernels = [np.asarray(W, np.float32) for W in m['kernels']]
    acts = [(kind, np.asarray(kif, np.int64)) for kind, kif in m['activations']]
    return kernels, [[tuple(q) for q in m['qintervals']]] + [None] * (len(kernels) - 1), acts, dict(adder_size=m['adder_size'], carry_size=m['carry_size'])


def oracle_stages(W, **call):
    """The oracle's ``solve`` as stage dicts that carry their shape and cost model."""
    from oracle import oracle_solve

    kw = {k: v for k, v in call.items() if k != 'seed'}
    stages, _ = oracle_solve(np.asarray(W, np.float32), **kw)
    return [dict(st, shape=(len(st['inp_shifts']), len(st['out_idxs'])), adder_size=kw.get('adder_size', -1), carry_size=kw.get('carry_size', -1)) for st in stages]


class OracleSweep:
    """``solve_sweep``'s result as chain_front reads it, one oracle solve per option set (sets with
    ``search_all_decompose_dc=False``: one candidate each)."""

    def __init__(self, W, sets, q, l, adder_size, carry_size):
        self._call = dict(qintervals=None if q is None else [tuple(float(v) for v in np.asarray(r, np.float32)) for r in q],
                          latencies=None if l is None else [float(v) for v in np.asarray(l, np.float32)], adder_size=adder_size, carry_size=carry_size)  # fmt: skip
        self._sets = [{**B.SWEEP_SET_DEFAULTS, **s} for s in sets]
        self._designs = [oracle_stages(W, **self.reference_call(i)) for i in range(len(sets))]
        cost = [seq_cost(d) for d in self._designs]
        lat = [float(max(np.asarray(d[-1]['ops_f'], np.float32)[j, 3] for j in d[-1]['out_idxs'].tolist())) for d in self._designs]
        self.candidates = dict(cost=np.asarray(cost, np.float32), latency_max=np.asarray(lat, np.float32))
        self.front = B.sweep_front(self.candidates['cost'], self.candidates['latency_max'])
        self.profile = dict(launches=1, device_ms=0.0, jobs_run=len(sets), jobs_total=len(sets))

    def raw(self, i):
        return B.RawPipeline.from_stages([dict(st) for st in self._designs[int(i)]])

    def reference_call(self, i):
        s = self._sets[int(i)]
        assert not s['search_all_decompose_dc']
        return dict(method0=s['method0'], method1=s['method1'], hard_dc=int(s['hard_dc']), decompose_dc=int(s['decompose_dc']), search_all_decompose_dc=False, **self._call)


class OracleSolver:
    """``solve_sweep_batch``'s signature on the oracle; records every call."""

    def __init__(self):
        self.calls = []

    def __call__(self, kernels, option_sets, qintervals=None, latencies=None, adder_size=-1, carry_size=-1):
        self.calls.append(dict(n=len(kernels), qintervals=qintervals, latencies=latencies))
        return [OracleSweep(W, option_sets, q, l, adder_size, carry_size) for W, q, l in zip(kernels, qintervals, latencies)]


def simt_pricer(designs, latency_cutoff, latencies=None, retiming=True):
    """``price_pipelined`` on the pricing kernel under the SIMT shim."""
    r = SIM.price(designs, latency_cutoff, latencies, retiming, threads=64)
    cuts = np.atleast_1d(np.asarray(latency_cutoff, np.float64))
    return B.PipelinePrice(r['status'], r['stages'], r['reg_bits'], r['latency_max'], r['cutoff'], cuts, r['out_latency'], dict(device_ms=0.0, launches=r['launches']))


def stated_cost(cf, p, layer_costs):
    """The float32 sum, in stage order, of the cost column of point ``p``'s chain design: each layer's design cost (here
    ``layer_costs[k]``), then the cost of each op of the activation stage after it."""
    d = cf.design(p)
    n_stages = [len(cf.raw(p, k).stages) for k in range(len(layer_costs))]
    cost, pos = np.float32(0.0), 0
    for k, c in enumerate(layer_costs):
        cost = np.float32(cost + np.float32(c))
        pos += n_stages[k]
        if k < len(layer_costs) - 1:
            for v in np.asarray(d.stages[pos]['ops_f'], np.float32)[:, 4]:
                cost = np.float32(cost + v)
            pos += 1
    return cost


def check_front_against_golden(cf, m, sets, c, solve_stages):
    """Every point of ``cf`` (a front of golden model ``m`` at cutoff ``c``) against the tracer's traces of the same tuple
    of option sets: its reference calls, its designs, its cost (the stated sum) and its latency; and the golden's
    cheapest chain is on the front.  ``solve_stages(W, **call)`` solves one recorded call."""
    traces = {(tuple(t['choice']), t['cutoff']): t for t in m['traces']}
    kernels, _, acts, _ = model_args(m)
    assert len(cf) >= 1
    for p in range(len(cf)):
        calls = cf.reference_calls(p)
        choice = tuple(next(s for s, o in enumerate(sets) if all(call[key] == v for key, v in o.items())) for call in calls)
        t = traces[choice, c]
        assert not t['raised'], (m['name'], choice, c)
        costs = []
        for k, (call, gc) in enumerate(zip(calls, t['calls'])):
            tag = (m['name'], choice, c, k)
            assert all(call[key] == v for key, v in gc['options'].items()), tag
            assert all(type(v) is float for q in call['qintervals'] for v in q) and all(type(v) is float for v in call['latencies']), tag
            assert np.array_equal(np.asarray(call['qintervals'], np.float32), np.asarray(gc['qintervals'], np.float32)), tag
            assert call['latencies'] == gc['latencies'], tag
            assert digest(cf.raw(p, k).stages) == gc['digest'], tag
            costs.append(gc['cost'])
        assert cf.cost[p].view(np.uint32) == stated_cost(cf, p, costs).view(np.uint32), (m['name'], choice, c)
        assert float(cf.latency[p]) == max(t['out_latency']), (m['name'], choice, c)
    # the cheapest chain of every tuple the tracer could trace survives the pruning
    best = None
    for t in m['traces']:
        if t['cutoff'] != c or t['raised']:
            continue
        designs = [solve_stages(W, **gc['options'], qintervals=gc['qintervals'], latencies=gc['latencies']) for W, gc in zip(kernels, t['calls'])]
        assert [digest(d) for d in designs] == [gc['digest'] for gc in t['calls']]
        d = B.chain_design(designs, acts)
        cost, pos = np.float32(0.0), 0
        for k, gc in enumerate(t['calls']):
            cost = np.float32(cost + np.float32(gc['cost']))
            pos += len(designs[k])
            if k < len(acts):
                for v in np.asarray(d.stages[pos]['ops_f'], np.float32)[:, 4]:
                    cost = np.float32(cost + v)
                pos += 1
        best = cost if best is None else min(best, cost)
    assert float(cf.cost.min()) == float(best), (m['name'], c)


@pytest.mark.parametrize('c', [3.0, 5.0])
def test_front_matches_the_tracer(c):
    g = traced_golden()
    for m in g['models']:
        kernels, qs, acts, cost_model = model_args(m)
        cf = B.chain_front(kernels, g['sets'], qintervals=qs, latency_cutoff=c, activations=acts, solver=OracleSolver(), pricer=simt_pricer, **cost_model)
        check_front_against_golden(cf, m, g['sets'], c, oracle_stages)
        assert all(layer['replay_ms'] >= 0.0 and layer['dropped_constant'] == 0 for layer in cf.profile['layers'])


def test_golden_covers_the_cases():
    g = traced_golden()
    zero = (0.0, 0.0, 2.0**32)
    qs = [[tuple(q) for q in call['qintervals']] for m in g['models'] for t in m['traces'] for call in t['calls'][1:]]
    assert any(zero in q for q in qs)  # a value with no bits left, handed on as the tracer's constant 0
    per_model = [{json.dumps(t['calls'][1]['qintervals']) for t in m['traces']} for m in g['models']]
    assert len(per_model[0]) == 1 and len(per_model[1]) > 1  # design-independent and design-dependent intervals
    assert any(len({json.dumps(t['calls'][2]['qintervals']) for t in m['traces']}) > 1 for m in g['models'] if len(m['kernels']) > 2)
    assert any(kind == 'quantize' and min(r[1] for r in kif) < 5 for m in g['models'] for kind, kif in m['activations'])


def test_cutoff_zero_agrees_with_itself():
    """At latency_cutoff 0 (the solver's latencies): every reference call's intervals are the host replay of the chosen
    designs through the activations, its latencies the designs' output latencies, and every design what the call solves."""
    g = traced_golden()
    for m in g['models']:
        kernels, qs, acts, cost_model = model_args(m)
        cf = B.chain_front(kernels, g['sets'], qintervals=qs, activations=acts, solver=OracleSolver(), **cost_model)
        for p in range(len(cf)):
            calls, d = cf.reference_calls(p), cf.design(p)
            pos = 0
            for k, W in enumerate(kernels):
                raw = cf.raw(p, k)
                assert digest(raw.stages) == digest(oracle_stages(W, **calls[k])), (m['name'], p, k)
                pos += len(raw.stages)
                if k == len(acts):
                    break
                act = d.stages[pos]
                pos += 1
                idx = np.asarray(act['out_idxs'], np.int64)
                want_q = [(0.0, 0.0, 2.0**32) if i < 0 else tuple(np.asarray(act['ops_f'], np.float32)[i, :3].tolist()) for i in idx.tolist()]
                want_l = [0.0 if i < 0 else float(np.asarray(act['ops_f'], np.float32)[i, 3]) for i in idx.tolist()]
                assert [tuple(q) for q in calls[k + 1]['qintervals']] == want_q, (m['name'], p, k)
                assert calls[k + 1]['latencies'] == want_l, (m['name'], p, k)


def test_argument_errors_come_before_any_solve():
    g = traced_golden()
    kernels, qs, acts, _ = model_args(g['models'][0])

    def no_solver(*a, **k):
        pytest.fail('the solver was called')

    with pytest.raises(ValueError, match='^3 layers need 2 activations, got 1$'):
        B.chain_front(kernels, g['sets'], activations=acts[:1], solver=no_solver)
    with pytest.raises(ValueError, match="^activation 1: 'tanh' is not"):
        B.chain_front(kernels, g['sets'], activations=[acts[0], ('tanh', (0, 4, 0))], solver=no_solver)
    with pytest.raises(ValueError, match=r'^activation 0: kif must be one \(k, i, f\) triple or \[8, 3\]'):
        B.chain_front(kernels, g['sets'], activations=[('relu', np.zeros((6, 3), np.int64)), acts[1]], solver=no_solver)
    with pytest.raises(ValueError, match='^activation 1: rounding mode'):
        B.chain_front(kernels, g['sets'], activations=[acts[0], ('quantize', (1, 4, 0), 'RND')], solver=no_solver)
    with pytest.raises(ValueError, match='^layer 2: with activations'):
        B.chain_front(kernels, g['sets'], qintervals=[qs[0], None, [(-1.0, 1.0, 1.0)] * 6], activations=acts, solver=no_solver)


def test_without_activations_nothing_changes():
    g = traced_golden()
    kernels, qs, acts, cost_model = model_args(g['models'][1])
    a = B.chain_front(kernels, g['sets'], qintervals=qs, latency_cutoff=3.0, solver=OracleSolver(), pricer=simt_pricer, **cost_model)
    b = B.chain_front(kernels, g['sets'], qintervals=qs, latency_cutoff=3.0, solver=OracleSolver(), pricer=simt_pricer, activations=None, **cost_model)
    assert pickle.dumps(a) == pickle.dumps(b)
    assert b.activations is None and 'activations' not in vars(b)
    assert all('replay_ms' not in layer and 'dropped_constant' not in layer for layer in b.profile['layers'])
    with pytest.raises(TypeError, match='without activations'):
        b.design(0)
    assert len(b.design(0, acts).stages) == len(a.design(0, acts).stages)


def test_design_uses_the_fronts_activations():
    g = traced_golden()
    kernels, qs, acts, cost_model = model_args(g['models'][1])
    cf = B.chain_front(kernels, g['sets'], qintervals=qs, activations=acts, solver=OracleSolver(), **cost_model)
    back = pickle.loads(pickle.dumps(cf))
    for p in range(len(cf)):
        d = cf.design(p)
        same = cf.design(p, [(kind, kif.tolist(), 'TRN', 'WRAP') for kind, kif in acts])
        assert digest(d.stages) == digest(same.stages) == digest(back.design(p).stages)
    with pytest.raises(ValueError, match='differ from the ones the front was searched with'):
        cf.design(0, [acts[0], ('quantize', (1, 5, 0))])
    with pytest.raises(ValueError, match='differ from the ones the front was searched with'):
        cf.design(0, acts[:1])


def test_saturating_relu_is_the_intervals_given_by_hand():
    """A relu that saturates every value hands every design's next layer the same intervals: the front equals the old
    search given those intervals by hand, with costs that differ exactly by the relu ops' cost."""
    g = traced_golden()
    m = g['models'][0]
    kernels, qs, acts, cost_model = model_args(m)
    kernels, qs, acts = kernels[:2], qs[:2], acts[:1]
    for c in (0.0, 3.0):
        a = B.chain_front(kernels, g['sets'], qintervals=qs, latency_cutoff=c, activations=acts, solver=OracleSolver(), pricer=simt_pricer, **cost_model)
        given = {json.dumps(a.reference_calls(p)[1]['qintervals']) for p in range(len(a))}
        assert len(given) == 1  # (every design's activated intervals are the same list)
        q1 = json.loads(given.pop())
        b = B.chain_front(kernels, g['sets'], qintervals=[qs[0], q1], latency_cutoff=c, solver=OracleSolver(), pricer=simt_pricer, **cost_model)
        assert np.array_equal(a.choice, b.choice) and np.array_equal(a.latency, b.latency)
        assert [a.reference_calls(p) for p in range(len(a))] == [b.reference_calls(p) for p in range(len(b))]
        for p in range(len(a)):
            act = a.design(p).stages[len(a.raw(p, 0).stages)]
            relu = float(np.asarray(act['ops_f'], np.float64)[:, 4].sum())
            assert relu > 0 and float(a.cost[p]) == float(b.cost[p]) + relu, (c, p)


def test_equal_states_share_one_problem():
    g = traced_golden()
    for m in g['models']:
        kernels, qs, acts, cost_model = model_args(m)
        solver = OracleSolver()
        cf = B.chain_front(kernels, g['sets'], qintervals=qs, latency_cutoff=5.0, activations=acts, solver=solver, pricer=simt_pricer, **cost_model)
        assert [call['n'] for call in solver.calls] == [layer['states'] for layer in cf.profile['layers']]
        for k, call in enumerate(solver.calls):
            states = [(np.asarray(q, np.float32).tobytes(), np.asarray(l, np.float32).tobytes()) for q, l in zip(call['qintervals'], call['latencies'])]
            assert len(set(states)) == len(states), (m['name'], k)  # one problem per distinct state
            for p in range(len(cf)):
                rc = cf.reference_calls(p)[k]
                assert (np.asarray(rc['qintervals'], np.float32).tobytes(), np.asarray(rc['latencies'], np.float32).tobytes()) in states
    # the saturating relu: the intervals of every point are equal, so layer 1 has one state per latency vector
    m = g['models'][0]
    kernels, qs, acts, cost_model = model_args(m)
    solver = OracleSolver()
    B.chain_front(kernels, g['sets'], qintervals=qs, activations=acts, solver=solver, **cost_model)
    assert len({json.dumps(q) for q in solver.calls[1]['qintervals']}) == 1
