"""solve_sweep_batch, network_front, pickled results and sweep_sharded on the GPU: every matrix of a batch against the
reference's stored and live answers and against its own solve_sweep.  -m gpu."""
import pickle
import socket
import subprocess
import sys
from pathlib import Path

import numpy as np
import pytest
from conftest import assert_stage_equal, golden_cases, int_matrix
from test_sweep_gpu import SWEEPS, check_consistent, digest, latency, random_sets, seq_cost, summaries

import oracle

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]
CALL_PROFILE = ['device_ms', 'launches', 'solve_kernel_ms', 'solve_kernel_launches', 'jobs_total', 'jobs_run']


def hetero(rng, n_in):
    q = [(-float(2 ** rng.integers(0, 7)), float(2 ** rng.integers(0, 7)) - 0.5, 0.5) for _ in range(n_in)]
    return q, [float(v) for v in rng.integers(0, 3, n_in)]


def assert_same_sweep(a, b, tag=''):
    """Field for field, op tables by digest."""
    assert summaries(a) == summaries(b), tag
    assert np.array_equal(a.candidates['kept'], b.candidates['kept']), tag
    assert a.front.tolist() == b.front.tolist() and a.winners.tolist() == b.winners.tolist(), tag
    assert (a.n_sets, a.n_solved, a.n_kept) == (b.n_sets, b.n_solved, b.n_kept), tag
    for i in np.flatnonzero(a.candidates['kept']):
        assert digest(a.raw(i).stages) == digest(b.raw(i).stages), f'{tag} candidate {i}'
        assert a.reference_call(i) == b.reference_call(i), f'{tag} candidate {i}'


def golden_sets(B, W, m, kw):
    """The stored option sets, without the known dummy-dc failure of this library's solve (see test_golden_sweep)."""
    sets = []
    for s in m['sets']:
        o = s['options']
        if o['method0'] == 'dummy' and o['method1'] == 'auto' and 0 < o['hard_dc'] < 6:
            try:
                B.solve_raw(W, **o, **kw)
            except RuntimeError as e:
                assert str(e) == 'Unknown method: dummy-dc'
                continue
        sets.append(s)
    return sets


@pytest.mark.parametrize('name', [m['name'] for m in SWEEPS])
def test_golden_sweep_in_a_batch(cuda_binary, name):
    B = cuda_binary
    m = next(m for m in SWEEPS if m['name'] == name)
    W = np.asarray(m['kernel'], np.float32).reshape(m['shape'])
    cost_model = dict(adder_size=m['adder_size'], carry_size=m['carry_size'])
    kw = dict(qintervals=m['qintervals'], latencies=m['latencies'], **cost_model)
    sets = golden_sets(B, W, m, kw)
    rng = np.random.default_rng(len(name))
    comp = [int_matrix(12, 20, 6, 61), int_matrix(24, 9, 8, 62)]  # companions of other shapes, with their own intervals
    (q0, l0), (q2, l2) = hetero(rng, 12), hetero(rng, 24)
    opts = [s['options'] for s in sets]
    res = B.solve_sweep_batch([comp[0], W, comp[1]], opts, qintervals=[q0, m['qintervals'], q2], latencies=[l0, m['latencies'], None], keep_all=True, **cost_model)
    assert len(res) == 3
    r = res[1]
    c = r.candidates
    assert len(r) == sum(len(s['candidates']) for s in sets)
    i = 0
    for si, s in enumerate(sets):
        assert r.winners[si] == i + s['winner'], (si, s['options'])
        for g in s['candidates']:
            tag = f'set {si} {s["options"]} H={g["hard_dc"]} d={g["decompose_dc"]}'
            assert (c['set'][i], c['hard_dc'][i], c['decompose_dc_start'][i]) == (si, g['hard_dc'], g['decompose_dc']), tag
            assert digest(r.raw(i).stages) == g['sha256'], tag
            assert c['cost'][i] == np.float32(g['cost']), tag
            assert [c['latency_min'][i], c['latency_max'][i]] == g['latency'], tag
            assert c['n_adders'][i] == g['n_adders'], tag
            i += 1
    assert r.reference_call(0)['qintervals'] == (None if not m['qintervals'] else [tuple(map(float, v)) for v in m['qintervals']])
    for p, (K, q, l) in ((0, (comp[0], q0, l0)), (2, (comp[1], q2, None))):
        alone = B.solve_sweep(K, opts, qintervals=q, latencies=l, keep_all=True, **cost_model)
        assert_same_sweep(res[p], alone, f'companion {p}')
        assert res[p].reference_call(0)['latencies'] == (l if l is None else [float(v) for v in l])
    for x in res:
        check_consistent(x)
        assert {k: x.profile[k] for k in CALL_PROFILE} == {k: res[0].profile[k] for k in CALL_PROFILE}  # the whole call's


@pytest.mark.parametrize('seed', range(4))
def test_random_batches_vs_reference(cuda_binary, seed):
    B = cuda_binary
    mod, _ = oracle.best()
    rng = np.random.default_rng(1500 + seed)
    n = 2 + seed
    shapes = [(int(rng.integers(8, 33)), int(rng.integers(8, 33))) for _ in range(n)]
    Ws = [int_matrix(a, b, int(rng.integers(4, 9)), 1700 + 10 * seed + i) for i, (a, b) in enumerate(shapes)]
    cost_model = dict(adder_size=int(rng.choice([-1, 1, 4])), carry_size=int(rng.choice([-1, 2, 8])))
    qs, ls = [], []
    for i, (a, _) in enumerate(shapes):  # mixed: defaults, intervals only, intervals and latencies
        q, l = hetero(rng, a)
        qs.append(q if i % 3 else None)
        ls.append(l if i % 3 == 2 else None)
    sets = random_sets(rng, 4)
    sets.append(dict(sets[0]))
    res = B.solve_sweep_batch(Ws, sets, qintervals=qs, latencies=ls, keep_all=True, **cost_model)
    assert len(res) == n
    for p, (W, r) in enumerate(zip(Ws, res)):
        assert r.n_solved < len(r)
        for i in range(len(r)):
            call = r.reference_call(i)
            assert call['qintervals'] == (None if qs[p] is None else [tuple(map(float, v)) for v in qs[p]]) and call['latencies'] == ls[p]
            want = mod.solve(W, **call)
            for a, b in zip(r.raw(i).stages, want, strict=True):
                assert_stage_equal(a, b, f'matrix {p} candidate {i} {call} ')
        for s, w in enumerate(r.winners):
            for a, b in zip(r.raw(w).stages, mod.solve(W, **sets[s], qintervals=qs[p], latencies=ls[p], **cost_model), strict=True):
                assert_stage_equal(a, b, f'matrix {p} winner of {sets[s]} ')
        check_consistent(r)


def test_job_sharing_and_keep_all_are_result_neutral(cuda_binary):
    B = cuda_binary
    Ws = [int_matrix(24, 20, 8, 11), int_matrix(16, 16, 6, 12), int_matrix(24, 20, 8, 11)]  # (the same matrix twice: nothing is shared across matrices)
    sets = [dict(), dict(hard_dc=2), dict(method0='mc', hard_dc=0), dict(decompose_dc=-1, search_all_decompose_dc=False)]
    base = B.solve_sweep_batch(Ws, sets)
    every = B.solve_sweep_batch(Ws, sets, keep_all=True)
    B.set_job_sharing(False)
    try:
        alone = B.solve_sweep_batch(Ws, sets, keep_all=True)
    finally:
        B.set_job_sharing(True)
    assert base[0].profile['jobs_run'] <= alone[0].profile['jobs_run'] == alone[0].profile['jobs_total']
    for p in range(len(Ws)):
        assert summaries(base[p]) == summaries(every[p]) == summaries(alone[p])
        assert every[p].candidates['kept'].all()
        for i in range(len(every[p])):
            assert digest(every[p].raw(i).stages) == digest(alone[p].raw(i).stages)
            if base[p].candidates['kept'][i]:
                assert digest(base[p].raw(i).stages) == digest(every[p].raw(i).stages)
    assert_same_sweep(base[0], base[2])
    assert base[0].n_solved == B.solve_sweep(Ws[0], sets).n_solved  # (candidates are deduplicated within a matrix only)


def test_batch_of_one_equals_solve_sweep(cuda_binary):
    B = cuda_binary
    W = int_matrix(20, 12, 7, 21)
    rng = np.random.default_rng(21)
    q, l = hetero(rng, 20)
    sets = [dict(), dict(hard_dc=1), dict(method0='wmc-pdc', hard_dc=3)]
    (one,) = B.solve_sweep_batch([W], sets, qintervals=[q], latencies=[l], adder_size=2, carry_size=3)
    ref = B.solve_sweep(W, sets, qintervals=q, latencies=l, adder_size=2, carry_size=3)
    assert_same_sweep(one, ref)
    assert one.profile['launches'] == ref.profile['launches'] and one.profile['jobs_run'] == ref.profile['jobs_run']


def test_failing_set_fails_the_whole_batch(cuda_binary):
    B = cuda_binary
    W, V = int_matrix(16, 16, 8, 4), int_matrix(12, 8, 6, 5)
    bad = dict(method0='dummy', method1='mc', hard_dc=0)  # (see test_failing_set_fails_the_whole_sweep)
    with pytest.raises(RuntimeError, match='Unknown method: dummy-dc') as want:
        B.solve_raw(W, **bad)
    with pytest.raises(RuntimeError) as got:
        B.solve_sweep_batch([V, W], [dict(), bad, dict(hard_dc=1)])
    assert str(got.value) == str(want.value)
    with pytest.raises(RuntimeError, match='Unknown method: nope'):
        B.solve_sweep_batch([V, W], [dict(), dict(method1='nope')])
    res = B.solve_sweep_batch([V, W], [dict(hard_dc=1)])
    assert [len(r) for r in res] == [len(B.solve_sweep(V, [dict(hard_dc=1)])), len(B.solve_sweep(W, [dict(hard_dc=1)]))]


def test_bench_matrix_with_a_small_one(cuda_binary):
    """The 256x256 int8 benchmark matrix next to a 64x64 one in one pass, under the sets of test_bench_matrix_sweep."""
    B = cuda_binary
    large = golden_cases(full_only=False)
    W, V = int_matrix(256, 256, 8, 0), int_matrix(64, 64, 8, 1)
    sets = [dict(), dict(decompose_dc=-1, search_all_decompose_dc=False), dict(hard_dc=2, search_all_decompose_dc=False), dict(method0='mc', hard_dc=4)]
    big, small = B.solve_sweep_batch([W, V], sets)
    for s, name in ((0, 'c3_256x256_int8_default'), (1, 'c3_256x256_int8_dc-1')):
        meta = large[name]
        raw = big.raw(big.winners[s])
        assert raw.n_adders == meta['n_adders'] == big.candidates['n_adders'][big.winners[s]]
        assert digest(raw.stages) == meta['sha256'], name
    assert_same_sweep(small, B.solve_sweep(V, sets))
    check_consistent(big)
    check_consistent(small)


DENSE_SHAPES = [(16, 64), (64, 64), (64, 32), (32, 32), (32, 5)]  # the config-5 stand-in of test_dense_stack_batch_vs_checker


def dense_stack():
    return [int_matrix(a, b, 6, 40 + i) for i, (a, b) in enumerate(DENSE_SHAPES)]


def test_network_front_of_the_dense_stack(cuda_binary):
    B = cuda_binary
    from da4ml_b200.cmvm import network_front

    layers = dense_stack()
    sets = [dict(method0=m, hard_dc=h) for m in ('wmc', 'mc', 'wmc-dc') for h in (-1, 0, 1, 2, 4)]
    sweeps = B.solve_sweep_batch(layers, sets)
    nf = network_front(sweeps)
    assert len(nf) >= 1
    for p in range(len(nf)):
        cost, lat = None, None
        for sw, i in zip(sweeps, nf.choice[p]):
            st = sw.raw(i).stages  # (on its layer's front, so kept)
            c, lm = seq_cost(st), np.float32(latency(st)[1])
            cost, lat = (c, lm) if cost is None else (np.float32(cost + c), np.float32(lat + lm))
        assert cost.view(np.uint32) == nf.cost[p].view(np.uint32) and lat == nf.latency[p]
    # best(b) against brute force over every candidate's (cost, latency_max), float32 sums in layer order
    pts = [np.unique(np.stack([sw.candidates['cost'], sw.candidates['latency_max']], 1), axis=0) for sw in sweeps]
    tot_c, tot_l = pts[0][:, 0], pts[0][:, 1]
    for p in pts[1:]:
        tot_c = (tot_c[:, None] + p[None, :, 0]).ravel()
        tot_l = (tot_l[:, None] + p[None, :, 1]).ravel()
    for b in sorted({*nf.latency.tolist(), float(nf.latency[0]) + 0.5, float(nf.latency[-1]) + 3.0}):
        ok = tot_l <= b
        pt = nf.best(b)
        assert pt.cost == tot_c[ok].min() and pt.latency <= b
        assert pt.choice == tuple(nf.choice[list(nf.latency).index(pt.latency)])
    with pytest.raises(ValueError):
        nf.best(float(tot_l.min()) - 1.0)


def test_pickled_results_match(cuda_binary):
    B = cuda_binary
    Ws = [int_matrix(20, 16, 8, 31), int_matrix(12, 24, 6, 32)]
    sets = [dict(), dict(hard_dc=1), dict(method0='mc', hard_dc=2)]
    rng = np.random.default_rng(31)
    q, l = hetero(rng, 20)
    res = B.solve_sweep_batch(Ws, sets, qintervals=[q, None], latencies=[l, None])
    for r in res:
        back = pickle.loads(pickle.dumps(r))
        again = pickle.loads(pickle.dumps(back))  # (a detached copy pickles too)
        for x in (back, again):
            assert x._h is None
            assert_same_sweep(x, r)
            assert {k: x.candidates[k].tolist() for k in x.candidates} == {k: r.candidates[k].tolist() for k in r.candidates}
            assert x.profile == r.profile and x.option_sets == r.option_sets and np.array_equal(x.kernel, r.kernel)
            for i in range(len(r)):
                assert x.reference_call(i) == r.reference_call(i)
            for i in np.flatnonzero(r.candidates['kept']):
                for a, b in zip(x.raw(i).stages, r.raw(i).stages, strict=True):
                    assert_stage_equal(a, b)
                assert x.raw(i).counters == r.raw(i).counters
                assert x.pipeline(i).latency == r.pipeline(i).latency
            missing = int(np.flatnonzero(~r.candidates['kept'])[0])
            for j in (missing, len(r), -1):
                with pytest.raises(ValueError) as want:
                    r.raw(j)
                with pytest.raises(ValueError) as got:
                    x.raw(j)
                assert str(got.value) == str(want.value)


def test_sweep_sharded_two_ranks_nccl(cuda_binary):
    n_dev = cuda_binary.device_info()['cuda_devices']
    if n_dev < 2:
        pytest.skip('needs two GPUs')
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    out = subprocess.run([sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node=2', '--master-addr', '127.0.0.1', '--master-port', str(port),
                          str(ROOT / 'tests' / 'dist_sweep_gpu_worker.py')], capture_output=True, text=True, timeout=900, cwd=ROOT)
    assert out.returncode == 0, (out.stdout + out.stderr)[-3000:]
    assert 'SWEEP_DIST_OK world=2' in out.stdout, (out.stdout + out.stderr)[-3000:]

