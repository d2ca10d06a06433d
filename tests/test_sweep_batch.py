"""solve_sweep_batch, network_front and sweep_sharded without a device: argument checks on the host, the no-CPU-fallback
error, the network front against brute force, and the sharding of sweeps over two gloo ranks."""
import ctypes as C
import itertools
import os
import socket
from types import SimpleNamespace

import numpy as np
import pytest
import torch.distributed as dist
import torch.multiprocessing as mp
from conftest import int_matrix

W = np.arange(16, dtype=np.float32).reshape(4, 4)
W2 = np.arange(15, dtype=np.float32).reshape(5, 3)


def test_argument_checks_name_the_matrix():
    import da4ml_b200._binary as B

    with pytest.raises(ValueError, match='^matrix 1: expected 5 qintervals, got 3$'):
        B.solve_sweep_batch([W, W2], [dict()], qintervals=[None, [(-1.0, 1.0, 1.0)] * 3])
    with pytest.raises(ValueError, match='^matrix 0: expected 4 latencies, got 5$'):
        B.solve_sweep_batch([W, W2], [dict()], latencies=[[0.0] * 5, [0.0] * 5])
    with pytest.raises(ValueError, match='^expected qintervals for 2 matrices, got 1$'):
        B.solve_sweep_batch([W, W2], [dict()], qintervals=[None])
    with pytest.raises(ValueError, match='^expected latencies for 2 matrices, got 3$'):
        B.solve_sweep_batch([W, W2], [dict()], latencies=[None] * 3)
    with pytest.raises(TypeError, match='^matrix 1: kernel must be a numpy float32 ndarray$'):
        B.solve_sweep_batch([W, W2.astype(np.float64)], [dict()])
    with pytest.raises(RuntimeError, match='^matrix 0: csd_decompose only supports 2D arrays.$'):
        B.solve_sweep_batch([W[0], W2], [dict()])
    for bad in (dict(adder_size=1), dict(offload_fn=None), dict(hard_dc=1, search_all=True)):
        with pytest.raises(TypeError, match='unsupported keys'):
            B.solve_sweep_batch([W, W2], [dict(), bad])
    with pytest.raises(ValueError, match='n_sets must be positive'):
        B.solve_sweep_batch([W, W2], [])
    with pytest.raises(RuntimeError, match='Unknown method: nope'):
        B.solve_sweep_batch([W, W2], [dict(), dict(method0='nope')])
    # a lone matrix keeps solve_sweep's messages
    with pytest.raises(ValueError, match='^expected 4 qintervals, got 3$'):
        B.solve_sweep_batch([W], [dict()], qintervals=[[(-1.0, 1.0, 1.0)] * 3])


def test_empty_batch_needs_no_device():
    import da4ml_b200._binary as B

    assert B.solve_sweep_batch([], [dict(), dict(hard_dc=2)]) == []
    assert B.solve_sweep_batch([], [dict()], qintervals=[], latencies=[]) == []


def _c_batch(n_problems, kernels, n_in, n_out):
    import da4ml_b200._binary as B

    m = (C.c_char_p * 1)(b'wmc')
    m1 = (C.c_char_p * 1)(b'auto')
    z = np.zeros(1, np.int32)
    i32 = z.ctypes.data_as(C.POINTER(C.c_int32))
    out = (C.c_void_p * 2)()
    rc = B._L.da4ml_cmvm_solve_sweep_batch(n_problems, kernels, n_in, n_out, None, None, -1, -1, 1, m, m1, i32, i32, i32, 0, out)
    return rc, B._L.da4ml_cmvm_last_error().decode(), list(out)


def test_c_entry_checks():
    import da4ml_b200._binary as B

    for n in (0, -1):
        rc, msg, out = _c_batch(n, None, None, None)
        assert rc == 1 and msg == f'solve_sweep: n_problems must be positive (got {n})' and out == [None, None]  # DA4ML_E_INVALID
    ks = (B._f32p * 2)(B._fp(W), B._fp(W2))
    n_in, n_out = np.asarray([4, 0], np.int64), np.asarray([4, 3], np.int64)
    rc, msg, out = _c_batch(2, ks, B._ip(n_in), B._ip(n_out))
    assert rc == 1 and msg == 'solve_sweep: kernel 1 must be a non-empty 2D array' and out == [None, None]


def test_no_cpu_fallback():
    import da4ml_b200._binary as B
    from da4ml_b200.cmvm import solve_sweep_batch

    if B.device_info()['cuda_devices'] > 0:
        pytest.skip('a GPU is present')
    with pytest.raises(RuntimeError, match='no CUDA device'):
        solve_sweep_batch([W, W2], [dict(), dict(hard_dc=2, method0='mc')])


# ---- network_front --------------------------------------------------------------------------------------------------
def layer(rng, n, hi):
    """A stand-in sweep of n candidates with small integer costs and latencies (many exact ties)."""
    import da4ml_b200._binary as B

    c = rng.integers(0, hi, n).astype(np.float32) * np.float32(rng.choice([1, 3, 1000]))
    l = rng.integers(0, hi, n).astype(np.float32)
    return SimpleNamespace(candidates=dict(cost=c, latency_max=l), front=B.sweep_front(c, l))


def brute_force(sweeps, fronts_only=True):
    """Every combination of candidates in lexicographic order, float32 sums in layer order, the sweep_front rule."""
    import da4ml_b200._binary as B

    pools = [sw.front if fronts_only else np.arange(len(sw.candidates['cost'])) for sw in sweeps]
    combos = np.asarray(list(itertools.product(*pools)), np.int64).reshape(-1, len(sweeps))
    cost = sweeps[0].candidates['cost'][combos[:, 0]]
    lat = sweeps[0].candidates['latency_max'][combos[:, 0]]
    for k in range(1, len(sweeps)):
        cost = cost + sweeps[k].candidates['cost'][combos[:, k]]
        lat = lat + sweeps[k].candidates['latency_max'][combos[:, k]]
    keep = B.sweep_front(cost, lat)
    order = np.argsort(lat[keep], kind='stable')
    return cost[keep][order], lat[keep][order], combos[keep][order]


@pytest.mark.parametrize('seed', range(12))
def test_network_front_matches_brute_force_over_fronts(seed):
    from da4ml_b200.cmvm import network_front

    rng = np.random.default_rng(900 + seed)
    sweeps = [layer(rng, int(rng.integers(1, 12)), int(rng.integers(2, 7))) for _ in range(1 + seed % 5)]
    nf = network_front(sweeps)
    cost, lat, choice = brute_force(sweeps)
    assert nf.cost.dtype == nf.latency.dtype == np.float32 and nf.choice.dtype == np.int64
    assert nf.choice.shape == (len(nf), len(sweeps))
    assert np.array_equal(nf.cost.view(np.uint32), cost.view(np.uint32))
    assert np.array_equal(nf.latency.view(np.uint32), lat.view(np.uint32))
    assert np.array_equal(nf.choice, choice)
    assert np.all(np.diff(nf.latency) > 0) and np.all(np.diff(nf.cost) < 0)  # a front: faster is dearer
    for k, sw in enumerate(sweeps):
        assert np.isin(nf.choice[:, k], sw.front).all()


@pytest.mark.parametrize('seed', range(6))
def test_network_front_points_match_brute_force_over_all_candidates(seed):
    from da4ml_b200.cmvm import network_front

    rng = np.random.default_rng(300 + seed)
    sweeps = [layer(rng, int(rng.integers(1, 6)), int(rng.integers(2, 8))) for _ in range(1 + seed % 5)]
    nf = network_front(sweeps)
    cost, lat, _ = brute_force(sweeps, fronts_only=False)
    assert np.array_equal(nf.cost, cost) and np.array_equal(nf.latency, lat)


def test_network_front_sums_float32_in_layer_order():
    from da4ml_b200.cmvm import network_front

    big, tiny = np.float32(2**24), np.float32(1.0)  # (2^24 + 1) + 1 rounds to 2^24 twice in float32
    sw = [SimpleNamespace(candidates=dict(cost=np.asarray([v], np.float32), latency_max=np.asarray([1.0], np.float32)), front=np.asarray([0])) for v in (big, tiny, tiny)]
    nf = network_front(sw)
    assert nf.cost[0] == big and nf.latency[0] == 3.0
    assert network_front(sw[::-1]).cost[0] == big + 2


def test_best():
    from da4ml_b200._binary import NetworkFront

    nf = NetworkFront(np.asarray([9.0, 5.0, 4.0], np.float32), np.asarray([2.0, 4.0, 7.5], np.float32), np.asarray([[0, 1], [2, 3], [4, 5]], np.int64))
    assert nf.best(2.0) == (9.0, 2.0, (0, 1))  # at a point's latency
    assert nf.best(3.9) == (9.0, 2.0, (0, 1))  # between points
    assert nf.best(4) == (5.0, 4.0, (2, 3))
    assert nf.best(7.5) == nf.best(100.0) == (4.0, 7.5, (4, 5))
    assert nf.best(7.49999) == (5.0, 4.0, (2, 3))
    p = nf.best(5)
    assert (p.cost, p.latency, p.choice) == (5.0, 4.0, (2, 3))
    with pytest.raises(ValueError, match='latency budget of 1.5'):
        nf.best(1.5)


def test_network_front_needs_a_layer():
    from da4ml_b200.cmvm import network_front

    with pytest.raises(ValueError, match='at least one layer'):
        network_front([])


# ---- sweep_sharded over two gloo ranks, a CPU stand-in for the GPU sweep ---------------------------------------------------
SETS = [dict(), dict(hard_dc=2, method0='mc')]


def _cpu_sweeper(kernels, option_sets, qintervals=None, latencies=None, **kw):
    n = len(kernels)
    return [dict(kernel=k, sets=option_sets, qintervals=q, latencies=l, kw=kw) for k, q, l in zip(kernels, qintervals or [None] * n, latencies or [None] * n)]


def _problems():
    kernels = [int_matrix(6 + i % 3, 5 + i % 4, 4, i) for i in range(7)]
    rng = np.random.default_rng(5)
    qs = [[(-1.0, float(rng.integers(1, 9)), 1.0)] * k.shape[0] for k in kernels]
    ls = [[float(v) for v in rng.integers(0, 3, k.shape[0])] for k in kernels]
    return kernels, qs, ls


def _worker(rank, world, port_no, q):
    from da4ml_b200.distributed import sweep_sharded

    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port_no)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        kernels, qs, ls = _problems()
        got = sweep_sharded(kernels, SETS, solver=_cpu_sweeper, qintervals=qs, latencies=ls, keep_all=True)
        local = sweep_sharded(kernels, SETS, solver=_cpu_sweeper, gather=False, adder_size=1)
        q.put((rank, got, local))
    finally:
        dist.destroy_process_group()


def test_sweep_sharded_world2_gloo():
    from da4ml_b200.distributed import problem_weight, shard_assignment

    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port_no = s.getsockname()[1]
    s.close()
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port_no, q)) for r in range(2)]
    for p in procs:
        p.start()
    got_all = {r: (g, loc) for r, g, loc in [q.get(timeout=120) for _ in procs]}
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    kernels, qs, ls = _problems()
    want = _cpu_sweeper(kernels, SETS, qintervals=qs, latencies=ls, keep_all=True)
    for rank in (0, 1):
        got, local = got_all[rank]
        assert len(got) == len(want)
        for a, b in zip(got, want, strict=True):
            assert np.array_equal(a['kernel'], b['kernel']) and a['qintervals'] == b['qintervals'] and a['latencies'] == b['latencies']
            assert a['sets'] == SETS and a['kw'] == dict(keep_all=True)
    shards = shard_assignment([problem_weight(k) for k in kernels], 2)
    for rank in (0, 1):
        _, local = got_all[rank]
        assert sorted(local) == shards[rank]  # (gather=False: this rank's share only)
        for i, r in local.items():
            assert np.array_equal(r['kernel'], kernels[i]) and r['kw'] == dict(adder_size=1) and r['qintervals'] is None
    assert sorted(list(got_all[0][1]) + list(got_all[1][1])) == list(range(len(kernels)))
