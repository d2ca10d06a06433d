"""Parity of the CUDA path (through the C ABI) with the CPU checkers and the golden vectors.  -m gpu."""
import hashlib
import os

import numpy as np
import pytest
from conftest import STAGE_KEYS, assert_stage_equal, golden_cases, int_matrix, load_golden

import oracle
from oracle import port

pytestmark = pytest.mark.gpu

FULL = golden_cases()
ALL = golden_cases(full_only=False)
SOLVE_CASES = sorted(k for k, v in FULL.items() if not v.get('single'))
SINGLE_CASES = sorted(k for k, v in FULL.items() if v.get('single'))
LARGE_CASES = sorted(k for k, v in ALL.items() if not v['full'])


def digest(stages):
    h = hashlib.sha256()
    for st in stages:
        for k in STAGE_KEYS:
            a = np.ascontiguousarray(st[k])
            h.update(k.encode())
            h.update(str(a.shape).encode())
            h.update(a.tobytes())
    return h.hexdigest()


@pytest.mark.parametrize('name', SOLVE_CASES)
def test_golden_solve(cuda_binary, name):
    extra, stages = load_golden(name)
    raw = cuda_binary.solve_raw(extra['kernel'], **FULL[name]['kwargs'])
    assert len(raw.stages) == 2
    for i, (a, b) in enumerate(zip(raw.stages, stages)):
        assert_stage_equal(a, b, f'{name} stage{i} ')
    assert raw.n_adders == FULL[name]['n_adders']


@pytest.mark.parametrize('name', SINGLE_CASES)
def test_golden_single_stage_with_trace(cuda_binary, name):
    extra, stages = load_golden(name)
    kw = FULL[name]['kwargs']
    raw, tr = cuda_binary.solve_single_raw(extra['kernel'], kw['method'], extra['qint'], extra['lat'], kw['adder_size'], kw['carry_size'], trace_cap=4096)
    assert_stage_equal(raw.stages[0], stages[0], name + ' ')
    # per-iteration chosen pair and live histogram size (cmvm_core.cc:36-70)
    assert np.array_equal(tr[:, :4], extra['pairs'])
    assert np.array_equal(tr[:, 4], extra['f_sizes'])


@pytest.mark.parametrize('name', LARGE_CASES)
def test_golden_large_digest(cuda_binary, name):
    meta = ALL[name]
    W = int_matrix(*meta['spec'][1:])
    raw = cuda_binary.solve_raw(W, **meta['kwargs'])
    assert raw.n_adders == meta['n_adders']
    assert [len(st['ops_i']) for st in raw.stages] == meta['stage_ops']
    assert digest(raw.stages) == meta['sha256']
    assert np.array_equal(raw.to_pipeline().kernel, W)


@pytest.mark.parametrize('seed', range(10))
def test_random_options_vs_checker(cuda_binary, seed):
    mod, _ = oracle.best()
    rng = np.random.default_rng(1000 + seed)
    n_in, n_out, bits = int(rng.integers(1, 24)), int(rng.integers(1, 24)), int(rng.integers(1, 9))
    W = int_matrix(n_in, n_out, bits, 50 + seed)
    if seed % 3 == 0:
        W[:, int(rng.integers(0, n_out))] = 0  # all-zero column -> out_idx -1
        W[int(rng.integers(0, n_in))] *= 4  # row with a power-of-two factor
    if seed % 4 == 1:
        W = W * 0.25  # fractional weights
    kw = dict(
        method0=str(rng.choice(['mc', 'wmc', 'mc-dc', 'wmc-dc', 'mc-pdc', 'wmc-pdc'])),
        method1=str(rng.choice(['auto', 'mc', 'wmc'])),
        hard_dc=int(rng.choice([-1, 0, 1, 2, 7])),
        decompose_dc=int(rng.choice([-2, -1, 0, 1])),
        adder_size=int(rng.choice([-1, 1, 4])),
        carry_size=int(rng.choice([-1, 2, 8])),
        search_all_decompose_dc=bool(rng.integers(0, 2)),
    )
    if seed % 2:
        q = np.stack([-(2.0 ** rng.integers(0, 8, n_in)), 2.0 ** rng.integers(0, 8, n_in) - 0.5, np.full(n_in, 0.5)], axis=1).astype(np.float32)
        q[int(rng.integers(0, n_in))] = (0.0, 0.0, 1.0)
        kw['qintervals'] = [tuple(map(float, r)) for r in q]
        kw['latencies'] = [float(v) for v in rng.integers(0, 3, n_in)]
    raw = cuda_binary.solve_raw(np.ascontiguousarray(W, dtype=np.float32), **kw)
    want = mod.solve(W, **kw)
    for i, (a, b) in enumerate(zip(raw.stages, want, strict=True)):
        assert_stage_equal(a, b, f'{kw} stage{i} ')


@pytest.mark.parametrize('method', ['mc', 'mc-dc', 'mc-pdc', 'wmc', 'wmc-dc', 'wmc-pdc', 'dummy'])
def test_every_selector_single_stage(cuda_binary, method):
    mod, _ = oracle.best()
    W = int_matrix(24, 20, 7, 77)
    rng = np.random.default_rng(7)
    lat = rng.integers(0, 5, 24).astype(np.float32)
    q = np.stack([-(2.0 ** rng.integers(2, 9, 24)), 2.0 ** rng.integers(2, 9, 24) - 1, np.ones(24)], axis=1).astype(np.float32)
    raw, _ = cuda_binary.solve_single_raw(W, method, q, lat, 2, 4)
    assert_stage_equal(raw.stages[0], mod.solve_single(W, method, q, lat, 2, 4), method + ' ')


def test_helpers_match_checker(cuda_binary):
    B = cuda_binary
    for n_in, n_out, bits, seed in [(8, 8, 4, 0), (16, 12, 8, 1), (5, 33, 6, 2), (40, 40, 8, 3)]:
        W = int_matrix(n_in, n_out, bits, seed)
        W[:, 0] *= 2
        for center in (True, False):
            for a, b in zip(B.csd_decompose(W, center), port.csd_decompose(W, center), strict=True):
                assert np.array_equal(a, b)
        for dc in (-2, -1, 0, 1, 2, 5):
            for a, b in zip(B.kernel_decompose(W, dc), port.kernel_decompose(W, dc), strict=True):
                assert np.array_equal(a, b), (n_in, n_out, dc)
    x = np.random.default_rng(0).integers(-(2**20), 2**20, size=(7, 9)).astype(np.int32)
    assert np.array_equal(B.int_arr_to_csd(x), port.int_arr_to_csd(x))


def test_batch_equals_individual_and_group_size_invariance(cuda_binary):
    B = cuda_binary
    kernels = [int_matrix(10 + 3 * i, 8 + 2 * i, 4 + i % 4, i) for i in range(9)]
    batch = B.solve_batch_raw(kernels)
    for k, r in zip(kernels, batch):
        single = B.solve_raw(k)
        for a, b in zip(r.stages, single.stages, strict=True):
            assert_stage_equal(a, b)
    # the partition of columns and histogram segments over CTAs must not change the result
    W = int_matrix(48, 40, 8, 5)
    base = None
    try:
        for g in (1, 2, 7, 32, 132):
            B.set_group_size(g)
            raw, tr = B.solve_single_raw(W, 'wmc', trace_cap=1 << 14)
            cur = (digest(raw.stages), tr.tobytes())
            base = base or cur
            assert cur == base, f'group size {g} changed the adder graph'
    finally:
        B.set_group_size(0)


def test_error_behaviour(cuda_binary):
    with pytest.raises(RuntimeError, match='Unknown method'):  # cmvm_core.cc:63
        cuda_binary.solve(int_matrix(4, 4, 4, 0), method0='nope')


def test_full_size_reconstruction_properties(cuda_binary):
    """BASELINE configs 3-4 sizes: no CPU answer in reasonable time, so size-independent properties:
    the graph reproduces W exactly, op ids are topologically ordered, outputs are consistent."""
    for n, bits, kw in [(256, 8, dict(search_all_decompose_dc=False, decompose_dc=-1)), (128, 6, {})]:
        W = int_matrix(n, n, bits, 0)
        raw = cuda_binary.solve_raw(W, **kw)
        assert np.array_equal(raw.to_pipeline().kernel, W)
        for st, c in zip(raw.stages, raw.counters):
            oi = st['ops_i']
            n_in = st['shape'][0]
            idx = np.arange(len(oi))
            assert np.all(oi[n_in:, 0] < idx[n_in:]) and np.all(oi[n_in:, 1] < idx[n_in:])
            assert c['status'] == 0 and c['n_ops'] == len(oi)
            # every op after the inputs is an adder: T CSE ops + one per remaining digit pair
            assert np.all(oi[:n_in, 2] == -1) and np.all((oi[n_in:, 2] == 0) | (oi[n_in:, 2] == 1))
            assert c['T'] + (c['D_final'] - np.count_nonzero(st['out_idxs'] >= 0)) == len(oi) - n_in


def test_accounting_mode_is_result_neutral(cuda_binary):
    """Exact work accounting re-reads the whole histogram every step; the adder graph must not change, and the
    exact counters must agree with the CPU checker's."""
    B = cuda_binary
    W = int_matrix(40, 36, 8, 9)
    fast = B.solve_raw(W)
    try:
        B.set_accounting(True)
        exact = B.solve_raw(W)
        single, _ = B.solve_single_raw(W, 'wmc')
    finally:
        B.set_accounting(False)
    for a, b in zip(fast.stages, exact.stages, strict=True):
        assert_stage_equal(a, b)
    ref_single = port.solve_single(W, 'wmc')
    c, r = single.counters[0], ref_single['counters']
    for k in ('T', 'sum_F', 'sum_R', 'F0', 'R0', 'D0', 'D_final'):
        assert c[k] == r[k], k


def test_device_resident_inputs(cuda_binary):
    torch = pytest.importorskip('torch')
    B = cuda_binary
    mats = [int_matrix(20, 16, 6, 3), int_matrix(12, 30, 8, 4)]
    dev = [torch.from_numpy(m).cuda() for m in mats]
    torch.cuda.synchronize()
    got = B.solve_batch_device_raw([t.data_ptr() for t in dev], [m.shape for m in mats])
    for m, r in zip(mats, got):
        want = B.solve_raw(m)
        for a, b in zip(r.stages, want.stages, strict=True):
            assert_stage_equal(a, b)


EDGE_CASES = {
    'one_by_one': lambda: np.array([[5.0]], np.float32),
    'single_input': lambda: int_matrix(1, 9, 8, 1),
    'single_output': lambda: int_matrix(9, 1, 8, 2),
    'all_zero': lambda: np.zeros((6, 7), np.float32),
    'zero_rows_and_cols': lambda: np.pad(int_matrix(5, 4, 6, 3), ((1, 2), (2, 1))),
    'identity_times_pow2': lambda: (np.eye(12, dtype=np.float32) * 2.0 ** np.arange(12)).astype(np.float32),
    'wide_csd_20bit': lambda: int_matrix(6, 5, 20, 4),
    'fractional_2^-7': lambda: int_matrix(10, 10, 8, 5) * np.float32(2.0**-7),
    'tall_200x3': lambda: int_matrix(200, 3, 8, 6),
    'flat_3x200': lambda: int_matrix(3, 200, 8, 7),
    'repeated_columns': lambda: np.tile(int_matrix(16, 2, 8, 8), (1, 6)),
    'negated_columns': lambda: np.concatenate([int_matrix(12, 5, 7, 9), -int_matrix(12, 5, 7, 9)], axis=1),
    'binary_pm1': lambda: np.sign(int_matrix(24, 24, 8, 10) + 0.5).astype(np.float32),
}


@pytest.mark.parametrize('name', sorted(EDGE_CASES))
def test_edge_case_matrices(cuda_binary, name):
    mod, _ = oracle.best()
    W = np.ascontiguousarray(EDGE_CASES[name](), dtype=np.float32)
    for kw in (dict(), dict(hard_dc=1, adder_size=2, carry_size=4), dict(method0='mc', method1='mc', search_all_decompose_dc=False, decompose_dc=1, hard_dc=3)):
        raw = cuda_binary.solve_raw(W, **kw)
        want = mod.solve(W, **kw)
        for i, (a, b) in enumerate(zip(raw.stages, want, strict=True)):
            assert_stage_equal(a, b, f'{name} {kw} stage{i} ')
        assert np.array_equal(raw.to_pipeline().kernel, W)


def test_job_sharing_is_result_neutral(cuda_binary):
    """Candidates whose decomposition gives byte-identical stage matrices are solved once (host_solve.cuh); with the
    sharing switched off every candidate is solved separately, as the reference does.  Same graphs either way."""
    W = int_matrix(40, 33, 8, 12)
    base = cuda_binary.solve_raw(W)
    assert base.profile['jobs_run'] <= base.profile['jobs_total']
    cuda_binary.set_job_sharing(False)
    try:
        alt = cuda_binary.solve_raw(W)
    finally:
        cuda_binary.set_job_sharing(True)
    assert alt.profile['jobs_run'] == alt.profile['jobs_total'] == base.profile['jobs_total']
    for a, b in zip(base.stages, alt.stages, strict=True):
        assert_stage_equal(a, b)


def test_dense_stack_batch_vs_checker(cuda_binary):
    """BASELINE config 5 stand-in: the reference tree holds no JEDI-linear weights or shapes, so a synthetic stack of
    quantized dense layers (shapes stated here) is compiled in one batched call with the CLI's default delay
    constraint (hard_dc=2, reference _cli/convert.py:212) and compared layer by layer with the CPU checker."""
    mod, _ = oracle.best()
    shapes = [(16, 64), (64, 64), (64, 32), (32, 32), (32, 5)]
    layers = [int_matrix(a, b, 6, 40 + i) for i, (a, b) in enumerate(shapes)]
    got = cuda_binary.solve_batch_raw(layers, hard_dc=2)
    for W, r in zip(layers, got, strict=True):
        want = mod.solve(W, hard_dc=2)
        for i, (a, b) in enumerate(zip(r.stages, want, strict=True)):
            assert_stage_equal(a, b, f'{W.shape} stage{i} ')
        assert np.array_equal(r.to_pipeline().kernel, W)


def test_release_and_regrow(cuda_binary):
    W = int_matrix(20, 20, 8, 30)
    a = cuda_binary.solve_raw(W)
    cuda_binary.release()
    b = cuda_binary.solve_raw(W)
    for x, y in zip(a.stages, b.stages, strict=True):
        assert_stage_equal(x, y)


def test_group_sizes_and_full_solves_match_checker(cuda_binary):
    """Single stages at group sizes from one CTA to the whole GPU, and full solves of a few shapes, against the checker."""
    mod, _ = oracle.best()
    try:
        for n_in, n_out, bits, seed in [(8, 8, 4, 0), (16, 12, 6, 1), (32, 32, 8, 2), (64, 64, 8, 3), (24, 130, 6, 4)]:
            W = int_matrix(n_in, n_out, bits, seed)
            raw = cuda_binary.solve_raw(W)
            for i, (a, b) in enumerate(zip(raw.stages, mod.solve(W), strict=True)):
                assert_stage_equal(a, b, f'{n_in}x{n_out} stage{i} ')
        W = int_matrix(48, 40, 8, 9)
        want = mod.solve_single(W, 'wmc')
        for G in (1, 2, 7, 40, 132):
            cuda_binary.set_group_size(G)
            raw, _ = cuda_binary.solve_single_raw(W, 'wmc')
            assert_stage_equal(raw.stages[0], want, f'G={G} ')
    finally:
        cuda_binary.set_group_size(0)
