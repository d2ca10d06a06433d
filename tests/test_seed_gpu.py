"""Seeded tie-breaks on the GPU: seeded solve_single / solve against the seeded oracle op for op (with step traces), seed 0
through the new entries against the existing ones, the 64 x 64 row of the measurements, seeded sweeps, batches and chains
against their seeded solve calls, job sharing, and solve_best_of.  -m gpu."""
import numpy as np
import pytest
from conftest import assert_stage_equal, int_matrix
from test_chain_gpu import chain3
from test_sweep_batch_gpu import hetero
from test_sweep_gpu import digest, seq_cost

import seeded

pytestmark = pytest.mark.gpu

METHODS = ['mc', 'mc-dc', 'mc-pdc', 'wmc', 'wmc-dc', 'wmc-pdc']
SHAPES = [(8, 8), (12, 10), (16, 16), (20, 24), (24, 20), (32, 32), (40, 24), (48, 48)]


def check_trace(raw, trace, stage, tag):
    """Trace row t is greedy step t: the pair of op n_in + t, and |F| summed over the steps is the oracle's sum_F."""
    n_in = stage['shape'][0]
    T = stage['counters']['T']
    assert trace.shape[0] == T, tag
    ops = np.asarray(raw.stages[0]['ops_i'])[n_in : n_in + T]
    assert np.array_equal(trace[:, 0], ops[:, 0]) and np.array_equal(trace[:, 1], ops[:, 1]), tag
    assert np.array_equal(trace[:, 2], ops[:, 3]) and np.array_equal(trace[:, 3], ops[:, 2]), tag
    assert int(trace[:, 4].astype(np.int64).sum()) == stage['counters']['sum_F'], tag


@pytest.mark.parametrize('case', range(len(SHAPES)))
def test_seeded_solve_single_is_the_seeded_oracle(cuda_binary, case):
    B = cuda_binary
    n_in, n_out = SHAPES[case]
    rng = np.random.default_rng(900 + case)
    W = int_matrix(n_in, n_out, int(rng.integers(4, 9)), 910 + case)
    q, lat = hetero(rng, n_in) if case % 2 else (None, None)
    for method in METHODS:
        for adder_size in (-1, 3):
            seed = int(rng.integers(1, 2**63))
            kw = dict(qintervals=q, latencies=lat, adder_size=adder_size, carry_size=2 if adder_size > 0 else -1)
            want = seeded.solve_single(W, method, seed=seed, **kw)
            raw, trace = B.solve_single_raw(W, method, trace_cap=4 * W.size * 8, seed=seed, **kw)
            tag = f'{n_in}x{n_out} {method} adder {adder_size} seed {seed} '
            assert_stage_equal(raw.stages[0], want, tag)
            check_trace(raw, trace, want, tag)


@pytest.mark.parametrize('case', range(4))
def test_seeded_solve_is_the_seeded_oracle(cuda_binary, case):
    B = cuda_binary
    n_in, n_out = [(8, 8), (16, 12), (24, 24), (32, 20)][case]
    rng = np.random.default_rng(950 + case)
    W = int_matrix(n_in, n_out, 6, 960 + case)
    q, lat = hetero(rng, n_in) if case % 2 else (None, None)
    for kw in (dict(), dict(method0='mc', hard_dc=2), dict(method0='wmc-dc', hard_dc=1, adder_size=2, carry_size=3)):
        for seed in (1, 3, 2**64 - 1):
            raw = B.solve_raw(W, qintervals=q, latencies=lat, seed=seed, **kw)
            want = seeded.solve(W, qintervals=q, latencies=lat, seed=seed, **kw)
            for a, b in zip(raw.stages, want, strict=True):
                assert_stage_equal(a, b, f'{n_in}x{n_out} {kw} seed {seed} ')
            assert np.array_equal(raw.kernel, W)


def test_seed0_through_the_new_entries_is_the_existing_entries(cuda_binary):
    import ctypes as C

    B = cuda_binary
    W = np.ascontiguousarray(int_matrix(20, 16, 7, 5))
    fp = W.ctypes.data_as(C.POINTER(C.c_float))
    h0, h1 = C.c_void_p(), C.c_void_p()
    B._check(B._L.da4ml_cmvm_solve(fp, 20, 16, b'wmc', b'auto', -1, -2, None, None, -1, -1, 1, C.byref(h0)))
    B._check(B._L.da4ml_cmvm_solve_seeded(fp, 20, 16, b'wmc', b'auto', -1, -2, None, None, -1, -1, 1, 0, C.byref(h1)))
    assert digest(B.RawPipeline(h0).stages) == digest(B.RawPipeline(h1).stages)
    tr0, tr1 = np.zeros((4000, 5), np.int32), np.zeros((4000, 5), np.int32)
    ip = lambda a: a.ctypes.data_as(C.POINTER(C.c_int32))  # noqa: E731
    B._check(B._L.da4ml_cmvm_solve_single(fp, 20, 16, b'mc', None, None, -1, -1, ip(tr0), 4000, C.byref(h0)))
    B._check(B._L.da4ml_cmvm_solve_single_seeded(fp, 20, 16, b'mc', None, None, -1, -1, ip(tr1), 4000, 0, C.byref(h1)))
    assert digest(B.RawPipeline(h0).stages) == digest(B.RawPipeline(h1).stages) and np.array_equal(tr0, tr1)
    sets = [dict(method0='wmc', hard_dc=1), dict(method0='mc-dc')]
    a, b = B.solve_sweep(W, sets), B.solve_sweep(W, [{**s, 'seed': 0} for s in sets])
    assert all(np.array_equal(a.candidates[k], b.candidates[k]) for k in a.candidates)
    assert [a.reference_call(i) for i in range(len(a))] == [b.reference_call(i) for i in range(len(b))]


def test_the_64x64_row(cuda_binary):
    """64 x 64 int8, rng 1, default solve: 4866 adders at seed 0, 4831 at seed 3, op for op the seeded oracle."""
    B = cuda_binary
    W = np.random.default_rng(1).integers(-128, 128, (64, 64)).astype(np.float32)
    assert B.solve_raw(W).n_adders == 4866
    raw = B.solve_raw(W, seed=3)
    assert raw.n_adders == 4831
    for a, b in zip(raw.stages, seeded.solve(W, seed=3), strict=True):
        assert_stage_equal(a, b, 'seed 3 ')
    assert np.array_equal(raw.kernel, W)


SETS = [dict(), dict(seed=1), dict(seed=2), dict(method0='mc', hard_dc=2, seed=5), dict(method0='mc', hard_dc=2), dict(seed=1)]


def test_seeded_sweep_is_its_solve_calls(cuda_binary):
    B = cuda_binary
    W = int_matrix(24, 20, 7, 33)
    sw = B.solve_sweep(W, SETS, keep_all=True)
    plain = B.solve_sweep(W, [s for s in SETS if not s.get('seed')], keep_all=True)
    assert sw.n_solved < len(sw)  # the repeated (seed 1) set is solved once
    for i in range(len(sw)):
        call = sw.reference_call(i)
        assert ('seed' in call) == bool(SETS[int(sw.candidates['set'][i])].get('seed')), call
        st = sw.raw(i).stages
        assert digest(st) == digest(B.solve_raw(W, **call).stages), call
        assert digest(st) == digest(seeded.solve(W, **call)), call
        assert seq_cost(st).view(np.uint32) == sw.candidates['cost'][i].view(np.uint32)
    for s, w in enumerate(sw.winners):
        assert digest(sw.raw(w).stages) == digest(B.solve_raw(W, **SETS[s]).stages), SETS[s]
    # the unseeded sets give what the sweep without seeds gives
    j = 0
    for s, opts in enumerate(SETS):
        if opts.get('seed'):
            continue
        a, b = np.flatnonzero(sw.candidates['set'] == s), np.flatnonzero(plain.candidates['set'] == j)
        assert [digest(sw.raw(i).stages) for i in a] == [digest(plain.raw(i).stages) for i in b]
        j += 1


def test_seeded_sweep_batch_is_each_matrix_sweep(cuda_binary):
    B = cuda_binary
    rng = np.random.default_rng(71)
    Ws = [int_matrix(16, 12, 6, 72), int_matrix(12, 20, 7, 73), int_matrix(16, 12, 6, 72)]
    ql = [hetero(rng, W.shape[0]) for W in Ws]
    qs, ls = [q for q, _ in ql], [l for _, l in ql]
    batch = B.solve_sweep_batch(Ws, SETS, qintervals=qs, latencies=ls, adder_size=2, carry_size=3, keep_all=True)
    for p, W in enumerate(Ws):
        one = B.solve_sweep(W, SETS, qintervals=qs[p], latencies=ls[p], adder_size=2, carry_size=3, keep_all=True)
        for k in ('set', 'hard_dc', 'decompose_dc_start', 'decompose_dc', 'n_adders', 'cost', 'latency_max', 'winner', 'front'):
            assert np.array_equal(batch[p].candidates[k], one.candidates[k]), (p, k)
        for i in range(len(one)):
            d = digest(batch[p].raw(i).stages)
            assert d == digest(one.raw(i).stages), (p, i)
            assert d == digest(B.solve_raw(W, **batch[p].reference_call(i)).stages), (p, i)


def test_job_sharing_does_not_change_seeded_results(cuda_binary):
    B = cuda_binary
    W = int_matrix(20, 20, 6, 81)
    on = B.solve_sweep(W, SETS, keep_all=True)
    try:
        B.set_job_sharing(False)
        off = B.solve_sweep(W, SETS, keep_all=True)
    finally:
        B.set_job_sharing(True)
    assert on.profile['jobs_run'] < off.profile['jobs_run']
    assert [digest(on.raw(i).stages) for i in range(len(on))] == [digest(off.raw(i).stages) for i in range(len(off))]


def test_solve_best_of(cuda_binary):
    B = cuda_binary
    from da4ml_b200.cmvm import solve_best_of

    W = np.random.default_rng(2).integers(-128, 128, (16, 16)).astype(np.float32)
    raw, s = B.solve_best_of_raw(W, n_seeds=6)
    costs = [seq_cost(B.solve_raw(W, seed=k).stages) for k in range(6)]
    assert s == int(np.argmin(costs)) and seq_cost(raw.stages) == min(costs) <= costs[0]
    assert digest(raw.stages) == digest(B.solve_raw(W, seed=s).stages)
    pipe, s1 = solve_best_of(W, n_seeds=6)
    assert s1 == s and np.array_equal(pipe.kernel, W)
    # one seed is seed 0 itself; equal costs go to the lowest seed
    raw1, s1 = B.solve_best_of_raw(W, n_seeds=1, method0='mc')
    assert s1 == 0 and digest(raw1.stages) == digest(B.solve_raw(W, method0='mc').stages)
    Z = np.diag(np.arange(1, 9, dtype=np.float32))  # no pair repeats: every seed gives the same graph
    raw2, s2 = B.solve_best_of_raw(Z, n_seeds=4)
    assert s2 == 0


def test_chain_front_with_seeds(cuda_binary):
    """The invariants of test_chain_gpu under seeded option sets: every design is its reference_calls solve."""
    B = cuda_binary
    Ws, qs, l0 = chain3()
    sets = [dict(method0='wmc', hard_dc=h, seed=s) for h in (-1, 2) for s in (0, 1, 4)] + [dict(method0='mc-dc', hard_dc=0, seed=2)]
    cf = B.chain_front(Ws, sets, qintervals=qs, latencies=l0)
    assert len(cf) >= 1
    for p in range(len(cf)):
        calls, pipes = cf.reference_calls(p), cf.pipelines(p)
        cost = None
        for k, W in enumerate(Ws):
            tag = f'point {p} layer {k} {calls[k]}'
            assert calls[k]['latencies'] == (l0 if k == 0 else [float(v) for v in pipes[k - 1].out_latencies]), tag
            st = cf.raw(p, k).stages
            assert digest(st) == digest(B.solve_raw(W, **calls[k]).stages), tag
            assert digest(st) == digest(seeded.solve(W, **calls[k])), tag
            assert np.array_equal(cf.raw(p, k).kernel, W), tag
            c = seq_cost(st)
            cost = c if cost is None else np.float32(cost + c)
        assert cost.view(np.uint32) == cf.cost[p].view(np.uint32)
        assert cf.latency[p] == max(pipes[-1].out_latencies)
