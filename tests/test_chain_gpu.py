"""chain_front on the GPU: every design of every front point against the reference's solve under the propagated input
latencies, a one-layer chain against solve_sweep, batched against per-state sweeps, and the dense stand-in.  -m gpu."""
import pickle

import numpy as np
import pytest
from conftest import int_matrix
from test_sweep_batch_gpu import dense_stack, hetero
from test_sweep_gpu import digest, seq_cost

import oracle

pytestmark = pytest.mark.gpu

SETS = [dict(method0=m, hard_dc=h) for m in ('wmc', 'mc-dc', 'wmc-dc') for h in (-1, 0, 2) if (m, h) != ('wmc-dc', -1)]


def chain3():
    """12x16, 16x10, 10x6 int6 with their own input intervals, and non-zero latencies at the chain's inputs."""
    rng = np.random.default_rng(77)
    Ws = [int_matrix(12, 16, 6, 71), int_matrix(16, 10, 6, 72), int_matrix(10, 6, 6, 73)]
    qs = [hetero(rng, W.shape[0])[0] for W in Ws]
    return Ws, qs, [float(v) for v in rng.integers(1, 4, 12)]


def test_every_design_is_the_reference_solve(cuda_binary):
    B = cuda_binary
    mod, _ = oracle.best()
    Ws, qs, l0 = chain3()
    cf = B.chain_front(Ws, SETS, qintervals=qs, latencies=l0)
    assert len(cf) >= 2 and max(layer['states'] for layer in cf.profile['layers']) > 1
    assert np.all(np.diff(cf.latency) > 0) and np.all(np.diff(cf.cost) < 0)
    for p in range(len(cf)):
        calls, pipes = cf.reference_calls(p), cf.pipelines(p)
        cost = None
        for k, W in enumerate(Ws):
            tag = f'point {p} layer {k} {calls[k]}'
            assert calls[k]['qintervals'] == [tuple(map(float, v)) for v in qs[k]], tag
            assert calls[k]['latencies'] == (l0 if k == 0 else [float(v) for v in pipes[k - 1].out_latencies]), tag
            assert all(type(v) is float for v in calls[k]['latencies'])
            st = cf.raw(p, k).stages
            assert digest(st) == digest(mod.solve(W, **calls[k])), tag
            assert digest(st) == digest(B.solve_raw(W, **calls[k]).stages), tag
            assert np.array_equal(cf.raw(p, k).kernel, W), tag
            c = seq_cost(st)
            cost = c if cost is None else np.float32(cost + c)
        assert cost.view(np.uint32) == cf.cost[p].view(np.uint32)
        assert cf.latency[p] == max(pipes[-1].out_latencies)


def test_one_layer_chain_is_the_sweeps_front(cuda_binary):
    B = cuda_binary
    Ws, qs, l0 = chain3()
    cf = B.chain_front(Ws[:1], SETS, qintervals=qs[:1], latencies=l0, adder_size=2, carry_size=3)
    sw = B.solve_sweep(Ws[0], SETS, qintervals=qs[0], latencies=l0, adder_size=2, carry_size=3)
    front = sw.front[np.argsort(sw.candidates['latency_max'][sw.front], kind='stable')]
    assert cf.choice[:, 0].tolist() == front.tolist()
    assert np.array_equal(cf.cost, sw.candidates['cost'][front]) and np.array_equal(cf.latency, sw.candidates['latency_max'][front])
    for p, i in enumerate(front):
        assert digest(cf.raw(p, 0).stages) == digest(sw.raw(i).stages)
        assert cf.reference_calls(p) == [sw.reference_call(i)]
    assert cf.profile['layers'][0]['candidates'] == len(sw) and cf.profile['launches'] == sw.profile['launches']


def test_batching_the_states_is_result_neutral(cuda_binary):
    B = cuda_binary
    Ws, qs, l0 = chain3()
    cost_model = dict(adder_size=4, carry_size=2)

    def per_state(kernels, option_sets, qintervals, latencies, **kw):
        return [B.solve_sweep(W, option_sets, qintervals=q, latencies=l, **kw) for W, q, l in zip(kernels, qintervals, latencies)]

    a = B.chain_front(Ws, SETS, qintervals=qs, latencies=l0, **cost_model)
    b = B.chain_front(Ws, SETS, qintervals=qs, latencies=l0, solver=per_state, **cost_model)
    assert np.array_equal(a.cost.view(np.uint32), b.cost.view(np.uint32)) and np.array_equal(a.latency, b.latency)
    assert np.array_equal(a.choice, b.choice)
    assert [x['states'] for x in a.profile['layers']] == [x['states'] for x in b.profile['layers']]
    assert [x['candidates'] for x in a.profile['layers']] == [x['candidates'] for x in b.profile['layers']]
    assert max(x['states'] for x in a.profile['layers']) > 1
    for p in range(len(a)):
        assert a.reference_calls(p) == b.reference_calls(p)
        for k in range(len(Ws)):
            assert digest(a.raw(p, k).stages) == digest(b.raw(p, k).stages)


def test_dense_stack_chain(cuda_binary):
    B = cuda_binary
    layers = dense_stack()
    sets = [dict(), dict(method0='mc', hard_dc=0), dict(method0='wmc-dc', hard_dc=2), dict(method0='mc', hard_dc=4)]
    cf = B.chain_front(layers, sets)
    assert len(cf) >= 1 and len(cf.profile['layers']) == len(layers)
    for p in range(len(cf)):
        for k, W in enumerate(layers):
            assert np.array_equal(cf.raw(p, k).kernel, W), (p, k)
    back = pickle.loads(pickle.dumps(cf))
    assert np.array_equal(back.cost, cf.cost) and np.array_equal(back.latency, cf.latency) and np.array_equal(back.choice, cf.choice)
    assert back.profile == cf.profile
    for b in sorted({*cf.latency.tolist(), float(cf.latency[-1]) + 1.0}):
        assert back.best(b) == cf.best(b)
    with pytest.raises(ValueError, match='latency budget'):
        back.best(float(cf.latency[0]) - 1.0)
    for p in range(len(cf)):
        assert back.reference_calls(p) == cf.reference_calls(p)
        assert back.reference_calls(p)[0]['latencies'] == [0.0] * layers[0].shape[0]
        for k in range(len(layers)):
            assert digest(back.raw(p, k).stages) == digest(cf.raw(p, k).stages)
