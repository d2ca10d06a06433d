"""chain_front without a device: argument checks, the no-CPU-fallback error, and the chain search on stand-in sweeps
against brute force over every chain of front candidates."""
import pickle
import zlib

import numpy as np
import pytest

W0 = np.arange(12, dtype=np.float32).reshape(3, 4)
W1 = np.arange(8, dtype=np.float32).reshape(4, 2)


def test_argument_checks():
    from da4ml_b200.cmvm import chain_front

    with pytest.raises(ValueError, match='^layer 0 has 4 outputs but layer 1 has 2 inputs$'):
        chain_front([W0, W1.T], [dict()])
    with pytest.raises(ValueError, match='^chain_front needs at least one layer$'):
        chain_front([], [dict()])
    with pytest.raises(ValueError, match='^expected qintervals for 2 layers, got 1$'):
        chain_front([W0, W1], [dict()], qintervals=[None])
    with pytest.raises(ValueError, match='^layer 1: expected 4 qintervals, got 3$'):
        chain_front([W0, W1], [dict()], qintervals=[None, [(-1.0, 1.0, 1.0)] * 3])
    with pytest.raises(ValueError, match='^layer 0: expected 3 latencies, got 4$'):
        chain_front([W0, W1], [dict()], latencies=[0.0] * 4)
    with pytest.raises(TypeError, match='^layer 1: kernel must be a numpy float32 ndarray$'):
        chain_front([W0, W1.astype(np.float64)], [dict()])
    for bad in (dict(adder_size=1), dict(offload_fn=None), dict(latencies=[0.0] * 3)):
        with pytest.raises(TypeError, match='unsupported keys'):
            chain_front([W0, W1], [dict(), bad])


def test_no_cpu_fallback():
    import da4ml_b200._binary as B
    from da4ml_b200.cmvm import chain_front

    if B.device_info()['cuda_devices'] > 0:
        pytest.skip('a GPU is present')
    with pytest.raises(RuntimeError, match='^layer 0: .*no CUDA device'):
        chain_front([W0, W1], [dict(), dict(hard_dc=2, method0='mc')])


# ---- the search on stand-in sweeps ----------------------------------------------------------------------------------------
class FakeSweep:
    """A sweep as chain_front reads it.  ``outs[i]`` are candidate i's output latencies; NaN marks a constant-zero column
    (``out_idx == -1``).  The unreferenced last op has latency 99, so reading it in place of 0.0 shows."""

    def __init__(self, cost, lat, outs, call):
        import da4ml_b200._binary as B

        self.candidates = dict(cost=np.asarray(cost, np.float32), latency_max=np.asarray(lat, np.float32))
        self.front = B.sweep_front(self.candidates['cost'], self.candidates['latency_max'])
        self._outs, self._call = np.asarray(outs, np.float32), call
        self.profile = dict(launches=3, device_ms=0.25, jobs_run=2, jobs_total=5)

    def raw(self, i):
        import da4ml_b200._binary as B

        o = self._outs[i]
        zero = np.isnan(o)
        ops_f = np.zeros((o.size + 1, 5), np.float32)
        ops_f[:-1, 3] = np.where(zero, 99.0, o)
        ops_f[-1, 3] = 99.0
        return B.RawPipeline.from_stages([dict(out_idxs=np.where(zero, -1, np.arange(o.size)), ops_f=ops_f)])

    def reference_call(self, i):
        return dict(candidate=int(i), **self._call)


class FakeSolver:
    """``solve_sweep_batch``'s signature; ``model(layer, n_out, input_latencies) -> (cost, latency_max, outs)``."""

    def __init__(self, model):
        self.model, self.calls = model, []

    def __call__(self, kernels, option_sets, qintervals=None, latencies=None, adder_size=-1, carry_size=-1):
        k = len(self.calls)
        self.calls.append(dict(n=len(kernels), sets=option_sets, qintervals=qintervals, latencies=latencies, adder_size=adder_size, carry_size=carry_size))
        assert all(W is kernels[0] for W in kernels) and len(qintervals) == len(latencies) == len(kernels)
        call = dict(qintervals=qintervals[0], adder_size=adder_size, carry_size=carry_size)
        return [FakeSweep(*self.model(k, W.shape[1], np.asarray(l, np.float32)), call=dict(call, latencies=l)) for W, l in zip(kernels, latencies)]


def max_plus_model(seed, widths):
    """Layer k has a menu of candidates with integer costs and per-output latency offsets.  Under input latencies v a
    candidate's outputs are max(v) + its offsets, permuted by a hash of v (so states depend on the whole vector), with a
    constant-zero column in some candidates; its latency_max is max(v) + its largest offset.  Cost and latency_max depend
    on max(v) only, so pruning after each layer loses nothing and the front equals brute force over every chain."""
    rng = np.random.default_rng(seed)
    menus = []
    for n_out in widths:
        n = int(rng.integers(1, 10))
        cost = rng.integers(0, 8, n).astype(np.float32) * np.float32(rng.choice([1, 3, 1000]))
        off = rng.integers(0, 4, (n, n_out)).astype(np.float32)
        for i in range(n):
            if n_out > 1 and rng.integers(0, 2):
                j = int(np.argmin(off[i]))  # (never the column of the largest offset)
                if off[i, j] < off[i].max():
                    off[i, j] = np.nan
        menus.append((cost, off))

    def model(k, n_out, v):
        cost, off = menus[k]
        assert off.shape[1] == n_out
        m = np.float32(v.max()) if v.size else np.float32(0)
        perm = np.random.default_rng(zlib.crc32(v.tobytes())).permutation(n_out)
        return cost, m + np.nanmax(off, axis=1), m + off[:, perm]

    return model


def brute_force(model, widths, l0):
    """Every chain of front candidates, parents in order and candidates in order, then the sweep_front rule."""
    import da4ml_b200._binary as B

    chains = [((), np.float32(0), np.float32(0), np.asarray(l0, np.float32), [])]
    for k, n_out in enumerate(widths):
        grown = []
        for choice, c, _, v, lats in chains:
            cost, lat, outs = model(k, n_out, v)
            for i in B.sweep_front(cost, lat):
                o = np.where(np.isnan(outs[i]), np.float32(0), outs[i]).astype(np.float32)
                grown.append((choice + (int(i),), cost[i] if k == 0 else np.float32(c + cost[i]), lat[i], o, lats + [[float(x) for x in v]]))
        chains = grown
    cost = np.asarray([c[1] for c in chains], np.float32)
    lat = np.asarray([c[2] for c in chains], np.float32)
    keep = B.sweep_front(cost, lat)
    keep = keep[np.argsort(lat[keep], kind='stable')]
    return cost[keep], lat[keep], np.asarray([chains[p][0] for p in keep], np.int64), [chains[p][4] for p in keep]


def chain_of(widths, n_in=3):
    dims = [n_in, *widths]
    return [np.ones((dims[k], dims[k + 1]), np.float32) for k in range(len(widths))]


@pytest.mark.parametrize('seed', range(16))
def test_search_matches_brute_force(seed):
    from da4ml_b200.cmvm import chain_front

    rng = np.random.default_rng(40 + seed)
    widths = [int(v) for v in rng.integers(1, 5, 1 + seed % 5)]
    model = max_plus_model(seed, widths)
    l0 = [float(v) for v in rng.integers(0, 3, 3)]
    sets = [dict(), dict(hard_dc=2)]
    solver = FakeSolver(model)
    cf = chain_front(chain_of(widths), sets, latencies=l0, adder_size=2, carry_size=3, solver=solver)
    cost, lat, choice, lats = brute_force(model, widths, l0)
    assert cf.cost.dtype == cf.latency.dtype == np.float32 and cf.choice.dtype == np.int64
    assert cf.choice.shape == (len(cf), len(widths))
    assert np.array_equal(cf.cost.view(np.uint32), cost.view(np.uint32))
    assert np.array_equal(cf.latency.view(np.uint32), lat.view(np.uint32))
    assert np.array_equal(cf.choice, choice)
    for p in range(len(cf)):
        calls = cf.reference_calls(p)
        assert [c['latencies'] for c in calls] == lats[p]
        assert [c['candidate'] for c in calls] == cf.choice[p].tolist()
        assert all(c['adder_size'] == 2 and c['carry_size'] == 3 and c['qintervals'] is None for c in calls)
    # one problem per distinct state, in order of first use; every call under the same sets and cost model
    assert [c['n'] for c in solver.calls] == [layer['states'] for layer in cf.profile['layers']]
    assert solver.calls[0]['latencies'] == [l0]
    for c in solver.calls:
        assert c['sets'] == sets and (c['adder_size'], c['carry_size']) == (2, 3)
        assert len({tuple(l) for l in c['latencies']}) == c['n']
    assert cf.profile['launches'] == 3 * len(widths) and cf.profile['jobs_total'] == 5 * len(widths)
    assert len(cf) == cf.profile['layers'][-1]['points']


def test_one_layer_chain_is_the_sweeps_front():
    from da4ml_b200.cmvm import chain_front, network_front

    model = max_plus_model(7, [4])
    solver = FakeSolver(model)
    cf = chain_front(chain_of([4]), [dict()], latencies=[1.0, 0.0, 2.0], solver=solver)
    (sw,) = FakeSolver(model)(chain_of([4]), [dict()], qintervals=[None], latencies=[[1.0, 0.0, 2.0]])
    nf = network_front([sw])
    assert np.array_equal(cf.cost, nf.cost) and np.array_equal(cf.latency, nf.latency) and np.array_equal(cf.choice, nf.choice)
    order = np.argsort(sw.candidates['latency_max'][sw.front], kind='stable')
    assert cf.choice[:, 0].tolist() == sw.front[order].tolist()


def table_model(tables):
    """``tables[k][input latencies as a tuple] = (cost, latency_max, outs)``: hand-built sweeps."""
    return lambda k, n_out, v: tables[k][tuple(float(x) for x in v)]


def test_points_with_equal_output_latencies_share_one_problem():
    from da4ml_b200.cmvm import chain_front

    # layer 0: two front points whose designs have the same output latencies (one's latency_max counts an unused op)
    t0 = {(0.0, 0.0): ([5.0, 3.0], [2.0, 4.0], [[2.0, 2.0], [2.0, 2.0]])}
    t1 = {(2.0, 2.0): ([1.0, 0.5], [3.0, 5.0], [[3.0], [5.0]])}
    solver = FakeSolver(table_model([t0, t1]))
    cf = chain_front(chain_of([2, 1], n_in=2), [dict()], solver=solver)
    assert [c['n'] for c in solver.calls] == [1, 1] and solver.calls[1]['latencies'] == [[2.0, 2.0]]
    assert cf.profile['layers'][1]['states'] == 1
    # both parents are extended from that one sweep: (6, 3), (5.5, 5) from the first, (4, 3), (3.5, 5) from the second
    assert cf.cost.tolist() == [4.0, 3.5] and cf.latency.tolist() == [3.0, 5.0]
    assert cf.choice.tolist() == [[1, 0], [1, 1]]
    assert [c['latencies'] for c in cf.reference_calls(0)] == [[0.0, 0.0], [2.0, 2.0]]


def test_ties_keep_the_first_parent():
    from da4ml_b200.cmvm import chain_front

    t0 = {(1.0,): ([5.0, 3.0, 9.0], [2.0, 4.0, 1.0], [[2.0, np.nan], [4.0, 4.0], [1.0, 1.0]])}
    t1 = {(2.0, 0.0): ([4.0, 1.0], [6.0, 9.0], [[6.0], [9.0]]),  # (a zero column feeds 0.0 on)
          (4.0, 4.0): ([6.0, 0.0], [6.0, 10.0], [[6.0], [10.0]]),
          (1.0, 1.0): ([0.0], [6.0], [[6.0]])}
    solver = FakeSolver(table_model([t0, t1]))
    cf = chain_front(chain_of([2, 1], n_in=1), [dict()], latencies=[1.0], solver=solver)
    assert solver.calls[1]['latencies'] == [[2.0, 0.0], [4.0, 4.0], [1.0, 1.0]]
    # (9, 6) comes from each of the three parents: the first parent's is kept
    assert cf.latency.tolist() == [6.0, 9.0, 10.0] and cf.cost.tolist() == [9.0, 6.0, 3.0]
    assert cf.choice.tolist() == [[0, 0], [0, 1], [1, 1]]
    assert cf.reference_calls(0)[1]['latencies'] == [2.0, 0.0]
    assert cf.best(8) == (9.0, 6.0, (0, 0)) and cf.best(10) == (3.0, 10.0, (1, 1))


def test_layer_errors_are_named():
    from da4ml_b200.cmvm import chain_front

    model = max_plus_model(3, [2, 2])

    def failing(kernels, option_sets, **kw):
        if failing.n == 1:
            raise RuntimeError('sweep failed')
        failing.n += 1
        return FakeSolver(model)(kernels, option_sets, **kw)

    failing.n = 0
    with pytest.raises(RuntimeError, match='^layer 1: sweep failed$'):
        chain_front(chain_of([2, 2]), [dict()], solver=failing)


def test_pickled_front_answers_as_the_original():
    from da4ml_b200.cmvm import chain_front

    widths = [3, 2, 4]
    cf = chain_front(chain_of(widths), [dict()], qintervals=[[(-1.0, 1.0, 1.0)] * 3, None, [(0.0, 3.0, 0.5)] * 2], solver=FakeSolver(max_plus_model(11, widths)))
    back = pickle.loads(pickle.dumps(cf))
    assert np.array_equal(back.cost, cf.cost) and np.array_equal(back.latency, cf.latency) and np.array_equal(back.choice, cf.choice)
    assert back.profile == cf.profile
    for b in (float(cf.latency[0]), float(cf.latency[-1]) + 1):
        assert back.best(b) == cf.best(b)
    for p in range(len(cf)):
        calls = back.reference_calls(p)
        assert calls == cf.reference_calls(p)
        assert calls[0]['qintervals'] == [(-1.0, 1.0, 1.0)] * 3 and calls[1]['qintervals'] is None and calls[2]['qintervals'] == [(0.0, 3.0, 0.5)] * 2
        for k in range(len(widths)):
            assert np.array_equal(back.raw(p, k).stages[0]['ops_f'], cf.raw(p, k).stages[0]['ops_f'])
    with pytest.raises(ValueError, match='latency budget of -1'):
        back.best(-1)
