"""Seeded tie-breaks of the greedy pair selection, without a GPU: the rule, the seeded oracle against the unseeded oracle
and the issue's measured rows, the simulated kernels against the seeded oracle op for op, and the host-side argument
handling of the seeded entry points."""
import numpy as np
import pytest
from conftest import assert_stage_equal, golden_cases, int_matrix, load_golden

import seeded
from oracle import port, ref

METHODS = ['mc', 'mc-dc', 'mc-pdc', 'wmc', 'wmc-dc', 'wmc-pdc']


def splitmix_mask(s):
    """The rule restated: tb_mask(0) = 0, else splitmix64(s) & (2^36 - 1)."""
    if s == 0:
        return 0
    M = 2**64 - 1
    x = (s + 0x9E3779B97F4A7C15) & M
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & M
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & M
    return (x ^ (x >> 31)) & (2**36 - 1)


def test_tb_mask_values():
    import da4ml_b200._binary as B

    assert B.tb_mask(0) == seeded.tb_mask(0) == 0
    for s in (1, 2, 3, 7, 12, 2**32 + 5, 2**63, 2**64 - 1):
        want = splitmix_mask(s)
        assert B.tb_mask(s) == seeded.tb_mask(s) == want, s
        assert want < 2**36  # id1 (bits 36 and up) is never masked
    assert splitmix_mask(1) == 0x910A2DEC89025CC1 & (2**36 - 1)  # splitmix64(1) of the published generator


@pytest.mark.parametrize('name', sorted(golden_cases()))
def test_seed0_is_the_oracle(name):
    """Seed 0 of the seeded oracle is the oracle (and the reference, where it is built) on every stored golden case."""
    extra, stages = load_golden(name)
    meta = golden_cases()[name]
    kw = dict(meta['kwargs'])
    if name.startswith('single_'):
        kw = {k: v for k, v in kw.items() if k in ('method', 'adder_size', 'carry_size')}
        got = [seeded.solve_single(extra['kernel'], qintervals=extra.get('qint'), latencies=extra.get('lat'), seed=0, **kw)]
        want = [port.solve_single(extra['kernel'], qintervals=extra.get('qint'), latencies=extra.get('lat'), **kw)]
    else:
        kw.update(qintervals=extra.get('qint'), latencies=extra.get('lat'))
        got = seeded.solve(extra['kernel'], seed=0, **kw)
        want = port.solve(extra['kernel'], **kw)
        if ref.available():
            for a, b in zip(got, ref.solve(extra['kernel'], **kw), strict=True):
                assert_stage_equal(a, b, f'{name} ref ')
    for a, b in zip(got, want, strict=True):
        assert_stage_equal(a, b, f'{name} ')
    for a, b in zip(got, stages, strict=True):
        assert_stage_equal(a, b, f'{name} golden ')


# the issue's bold entries at 32 x 32 and below: (n, bits, rng, method0, seed, adders at seed 0, adders at the seed)
TABLE = [(16, 8, 2, 'wmc', 2, 356, 350), (32, 8, 0, 'wmc', 12, 1318, 1310), (16, 6, 2, 'mc', 3, 274, 267), (24, 6, 3, 'wmc-dc', 11, 642, 636),
         (24, 6, 4, 'wmc-dc', 1, 652, 642)]  # fmt: skip


@pytest.mark.parametrize('n,bits,r,method0,seed,a0,a_s', TABLE)
def test_oracle_reproduces_the_measured_rows(n, bits, r, method0, seed, a0, a_s):
    W = np.random.default_rng(r).integers(-(2 ** (bits - 1)), 2 ** (bits - 1), (n, n)).astype(np.float32)
    assert seeded.n_adders(seeded.solve(W, method0=method0, seed=0)) == a0
    assert seeded.n_adders(seeded.solve(W, method0=method0, seed=seed)) == a_s


def test_a_seed_changes_the_graph():
    W = int_matrix(16, 16, 8, 2)
    a, b = seeded.solve(W, seed=0), seeded.solve(W, seed=2)
    assert not all(np.array_equal(x['ops_i'], y['ops_i']) for x, y in zip(a, b))


# ---- the simulated kernels against the seeded oracle -------------------------------------------------------------------
@pytest.mark.parametrize('method', METHODS)
@pytest.mark.parametrize('seed', [1, 2, 12])
def test_sim_every_selector(method, seed):
    W = int_matrix(10, 9, 5, 40 + seed)
    got, meta = seeded.sim_solve_single(W, method, seed, ctas=2, cta_threads=64)
    assert_stage_equal(got, seeded.solve_single(W, method, seed=seed), f'{method} seed {seed} ')
    assert meta[0] == 0


@pytest.mark.parametrize('ctas,threads', [(1, 32), (2, 64), (3, 64), (4, 32), (5, 32)])
def test_sim_group_sizes(ctas, threads):
    W = int_matrix(14, 11, 6, 3)
    for seed in (0, 5):
        got, _ = seeded.sim_solve_single(W, 'wmc', seed, ctas=ctas, cta_threads=threads)
        assert_stage_equal(got, seeded.solve_single(W, 'wmc', seed=seed), f'{ctas}x{threads} seed {seed} ')


def test_sim_heterogeneous_intervals_and_latencies():
    rng = np.random.default_rng(5)
    W = int_matrix(16, 12, 7, 9) * np.float32(0.25)
    q = np.stack([-(2.0 ** rng.integers(0, 8, 16)), 2.0 ** rng.integers(0, 8, 16) - 0.5, np.full(16, 0.5)], axis=1).astype(np.float32)
    q[3] = (0.0, 0.0, 1.0)
    lat = rng.integers(0, 3, 16).astype(np.float32)
    for method in ('wmc-dc', 'mc-pdc', 'wmc'):
        for seed in (3, 9):
            kw = dict(qintervals=[tuple(map(float, r)) for r in q], latencies=[float(v) for v in lat], adder_size=2, carry_size=4)
            got, _ = seeded.sim_solve_single(W, method, seed, ctas=3, cta_threads=64, **kw)
            assert_stage_equal(got, seeded.solve_single(W, method, seed=seed, **kw), f'{method} seed {seed} ')


def test_sim_split_counter_passes():
    """A pair-counter table small enough to force several counting passes per recount."""
    W = int_matrix(16, 16, 8, 21)
    try:
        seeded.sim_lib().sim_set_own_caps(8, -1)  # 256 slots, 160 usable per pass: the owned rows' counters do not fit in one
        for seed in (0, 4):
            got, _ = seeded.sim_solve_single(W, 'wmc', seed, ctas=2, cta_threads=64)
            assert_stage_equal(got, seeded.solve_single(W, 'wmc', seed=seed), f'seed {seed} ')
    finally:
        seeded.sim_lib().sim_set_own_caps(0, -1)


def test_sim_compaction_and_capacity_status():
    """A histogram segment small enough to force compactions gives the seeded graph; one too small for the problem
    reports the capacity status, and the retry with room gives the same graph."""
    W = int_matrix(16, 16, 8, 7)
    want = seeded.solve_single(W, 'wmc', seed=6)
    L = seeded.sim_lib()
    try:
        L.sim_set_segment_cap(4096)
        got, meta = seeded.sim_solve_single(W, 'wmc', 6, ctas=2, cta_threads=64)
        assert_stage_equal(got, want, 'compacting ')
        assert meta[9] > 0, 'no compaction happened'
        L.sim_set_segment_cap(64)
        with pytest.raises(RuntimeError, match='capacity status'):
            seeded.sim_solve_single(W, 'wmc', 6, ctas=2, cta_threads=64)
    finally:
        L.sim_set_segment_cap(0)
    got, _ = seeded.sim_solve_single(W, 'wmc', 6, ctas=2, cta_threads=64)
    assert_stage_equal(got, want, 'retry ')


def test_sim_one_launch_mixes_seeds():
    """Jobs of one launch under different seeds (0 included, one matrix twice) each give their own seeded graph."""
    ks = [int_matrix(12, 10, 6, 1), int_matrix(9, 14, 7, 2), int_matrix(12, 10, 6, 1), int_matrix(8, 8, 4, 3)]
    seeds = [0, 3, 11, 2**64 - 1]
    got = seeded.sim_solve_many(ks, seeds, 'wmc', ctas=2, groups=2, cta_threads=64)
    for i, (W, s) in enumerate(zip(ks, seeds)):
        assert_stage_equal(got[i], seeded.solve_single(W, 'wmc', seed=s), f'job {i} ')


# ---- host-side arguments ----------------------------------------------------------------------------------------------
def test_seed_arguments_are_checked_before_any_device_call():
    import da4ml_b200._binary as B

    W = int_matrix(4, 4, 4, 0)
    for bad in (-1, 2**64):
        with pytest.raises(ValueError, match='seed must be in'):
            B.solve_raw(W, seed=bad)
        with pytest.raises(ValueError, match='seed must be in'):
            B.solve_single_raw(W, seed=bad)
        with pytest.raises(ValueError, match='seed must be in'):
            B.solve_sweep(W, [dict(), dict(seed=bad)])
        with pytest.raises(ValueError, match='seed must be in'):
            B.solve_sweep_batch([W, W], [dict(seed=bad)])
    for bad in (1.5, '3', True, None):
        with pytest.raises(TypeError, match='seed must be an integer'):
            B.solve_raw(W, seed=bad)
    with pytest.raises(TypeError, match='unsupported keys'):
        B.solve_sweep(W, [dict(seeds=1)])
    with pytest.raises(ValueError, match='n_seeds must be a positive integer'):
        B.solve_best_of(W, n_seeds=0)
    with pytest.raises(TypeError, match='no seed keyword'):
        B.solve_best_of(W, seed=3)


def test_seed_is_a_solver_option():
    from da4ml_b200.cmvm import solve_best_of, solver_options_t

    assert 'seed' in solver_options_t.__annotations__
    assert callable(solve_best_of)


def test_new_entries_without_a_device():
    """Each seeded entry fails cleanly, with the library's message, when there is no device."""
    import ctypes as C

    import da4ml_b200._binary as B

    if B.device_info()['cuda_devices'] > 0:
        pytest.skip('a device is present')
    W = np.ascontiguousarray(int_matrix(4, 4, 4, 0))
    h = C.c_void_p()
    fp = W.ctypes.data_as(C.POINTER(C.c_float))
    rc = B._L.da4ml_cmvm_solve_seeded(fp, 4, 4, b'wmc', b'auto', -1, -2, None, None, -1, -1, 1, 5, C.byref(h))
    assert rc != 0 and B._L.da4ml_cmvm_last_error()
    rc = B._L.da4ml_cmvm_solve_single_seeded(fp, 4, 4, b'wmc', None, None, -1, -1, None, 0, 5, C.byref(h))
    assert rc != 0 and B._L.da4ml_cmvm_last_error()
    with pytest.raises(RuntimeError):
        B.solve_sweep(W, [dict(seed=1), dict(seed=2)])
    for f in (lambda: B.solve_raw(W, seed=1), lambda: B.solve_single_raw(W, seed=1)):
        with pytest.raises(RuntimeError):
            f()


# ---- reference_call and solve_best_of with stand-ins -------------------------------------------------------------------
class FakeSweep:
    """A hand-built SweepResult: one candidate per set, the given costs; raw(i) returns a marker."""

    def __init__(self, costs, sets):
        self.candidates = dict(cost=np.asarray(costs, np.float32), set=np.arange(len(costs)))
        self.winners = np.arange(len(costs))
        self.option_sets = sets

    def raw(self, i):
        import da4ml_b200._binary as B

        r = B.RawPipeline.from_stages([])
        r.marker = int(i)
        return r


def test_solve_best_of_picks_the_cheapest_and_ties_go_to_the_lowest_seed():
    import da4ml_b200._binary as B

    seen = {}

    def solver(kernel, sets, **kw):
        seen.update(sets=sets, kw=kw)
        return FakeSweep(costs, sets)

    W = int_matrix(4, 4, 4, 0)
    costs = [10.0, 9.0, 7.0, 8.0, 7.0]
    raw, s = B.solve_best_of_raw(W, n_seeds=5, solver=solver, method0='mc', hard_dc=2, adder_size=3, latencies=[0.0] * 4)
    assert s == 2 and raw.marker == 2
    assert seen['sets'] == [dict(method0='mc', hard_dc=2, seed=k) for k in range(5)]
    assert seen['kw'] == dict(latencies=[0.0] * 4, adder_size=3)
    costs = [5.0, 5.0, 6.0]
    raw, s = B.solve_best_of_raw(W, n_seeds=3, solver=solver)
    assert s == 0 and raw.marker == 0  # never costlier than seed 0, and seed 0 itself on a tie


def test_reference_call_adds_seed_only_when_non_zero():
    import da4ml_b200._binary as B

    class Handleless(B.SweepResult):
        def __init__(self, sets):
            self.option_sets = sets
            self._call = dict(qintervals=None, latencies=None, adder_size=-1, carry_size=-1)
            self.candidates = dict(set=np.array([0, 1, 2]), hard_dc=np.array([10**9] * 3), decompose_dc_start=np.array([-1, 0, 1]))

        def __del__(self):
            pass

    sw = Handleless([dict(), dict(seed=0), dict(seed=7, method0='mc')])
    base = dict(method0='wmc', method1='auto', hard_dc=10**9, search_all_decompose_dc=False, qintervals=None, latencies=None, adder_size=-1, carry_size=-1)
    assert sw.reference_call(0) == {**base, 'decompose_dc': -1}
    assert list(sw.reference_call(0)) == ['method0', 'method1', 'hard_dc', 'decompose_dc', 'search_all_decompose_dc', 'qintervals', 'latencies', 'adder_size', 'carry_size']
    assert sw.reference_call(1) == {**base, 'decompose_dc': 0}
    assert sw.reference_call(2) == {**base, 'method0': 'mc', 'decompose_dc': 1, 'seed': 7}
