"""The independent restatement (oracle/port) against the reference's own object code on a broad random family of
inputs: ragged shapes, sparse / scaled / wide matrices, heterogeneous intervals and latencies, every selector.  This is
what lets the port stand in as the checker where the reference is absent.  The reference's answers for these inputs are
stored in tests/golden/reference_checks.json.gz (tests/golden/make_golden_refchecks.py).  No GPU."""
import numpy as np
import pytest
from conftest import GOLDEN, assert_stage_equal

from oracle import port

METHODS = ['mc', 'wmc', 'mc-dc', 'mc-pdc', 'wmc-dc', 'wmc-pdc']


def random_matrix(rng, n_in, n_out):
    kind = rng.choice(['dense', 'sparse', 'holes', 'fraction', 'wide', 'constant', 'diag'])
    bits = int(rng.integers(2, 9))
    W = rng.integers(-(2 ** (bits - 1)), 2 ** (bits - 1), size=(n_in, n_out)).astype(np.float64)
    if kind == 'sparse':
        W *= rng.random((n_in, n_out)) < 0.3
    elif kind == 'holes':  # whole rows / columns of zeros
        W[rng.random(n_in) < 0.3, :] = 0
        W[:, rng.random(n_out) < 0.3] = 0
    elif kind == 'fraction':
        W *= 2.0 ** -int(rng.integers(1, 6))
    elif kind == 'wide':
        W = rng.integers(-(2**11), 2**11, size=(n_in, n_out)).astype(np.float64)
    elif kind == 'constant':
        W[:] = float(rng.integers(-7, 8))
    elif kind == 'diag':
        W = np.eye(n_in, n_out) * float(rng.integers(1, 100))
    return np.ascontiguousarray(W, dtype=np.float32), kind


def random_intervals(rng, n_in):
    mode = rng.choice(['none', 'hetero', 'unsigned', 'some_zero'])
    if mode == 'none':
        return None
    q = np.zeros((n_in, 3), np.float32)
    for i in range(n_in):
        step = 2.0 ** int(rng.integers(-3, 3))
        lo, hi = sorted(int(v) for v in rng.integers(-200, 200, size=2))
        if mode == 'unsigned':
            lo = 0
            hi = abs(hi) + 1
        q[i] = (lo * step, hi * step, step)
        if mode == 'some_zero' and rng.random() < 0.3:
            q[i] = (0.0, 0.0, 1.0)
    return [tuple(float(v) for v in r) for r in q]


def random_latencies(rng, n_in):
    if rng.random() < 0.5:
        return None
    return [float(v) for v in rng.integers(0, 4, size=n_in)]


def shapes(rng):
    pick = rng.integers(0, 6)
    if pick == 0:
        return 1, int(rng.integers(1, 12))
    if pick == 1:
        return int(rng.integers(1, 12)), 1
    return int(rng.integers(2, 22)), int(rng.integers(2, 22))


def single_case(seed):
    rng = np.random.default_rng(7000 + seed)
    n_in, n_out = shapes(rng)
    W, kind = random_matrix(rng, n_in, n_out)
    kw = dict(
        method=str(rng.choice(METHODS + ['dummy'])),
        qintervals=random_intervals(rng, n_in),
        latencies=random_latencies(rng, n_in),
        adder_size=int(rng.choice([-1, 1, 3, 8])),
        carry_size=int(rng.choice([-1, 1, 4])),
    )
    return W, kind, kw


def full_case(seed):
    rng = np.random.default_rng(9000 + seed)
    n_in, n_out = shapes(rng)
    W, kind = random_matrix(rng, n_in, n_out)
    kw = dict(
        method0=str(rng.choice(METHODS)),
        method1=str(rng.choice(['auto'] + METHODS)),
        hard_dc=int(rng.choice([-1, 0, 1, 2, 5])),
        decompose_dc=int(rng.choice([-2, -1, 0, 1, 3])),
        qintervals=random_intervals(rng, n_in),
        latencies=random_latencies(rng, n_in),
        adder_size=int(rng.choice([-1, 2])),
        carry_size=int(rng.choice([-1, 3])),
        search_all_decompose_dc=bool(rng.integers(0, 2)),
    )
    return W, kind, kw


def helper_case(seed):
    """(W, int32 values for int_arr_to_csd, integer-grid matrix for kernel_decompose)"""
    rng = np.random.default_rng(11000 + seed)
    n_in, n_out = shapes(rng)
    W, _ = random_matrix(rng, n_in, n_out)
    ints = rng.integers(-(2**20), 2**20, size=(int(rng.integers(1, 40)),)).astype(np.int32)
    Wi = np.round(W * 64).astype(np.float32)  # kernel_decompose works on the integer grid
    return W, ints, Wi


HELPER_DCS = (-2, -1, 0, 1, 2)


def load_stored(name):
    """A file written by tests/golden/make_golden_refchecks.py: name -> array (or digest string)."""
    import gzip
    import json

    with gzip.open(GOLDEN / name, 'rt') as f:
        return {k: v if isinstance(v, str) else np.asarray(v[2], dtype=v[0]).reshape(v[1]) for k, v in json.load(f).items()}


@pytest.fixture(scope='module')
def want():
    return load_stored('reference_checks.json.gz')


def stored_stage(z, prefix):
    return {k: z[f'{prefix}_{k}'] for k in ('inp_shifts', 'out_idxs', 'out_shifts', 'out_negs', 'ops_i', 'ops_f')}


@pytest.mark.parametrize('seed', range(60))
def test_single_stage_random_family(want, seed):
    W, kind, kw = single_case(seed)
    assert_stage_equal(port.solve_single(W, **kw), stored_stage(want, f'cross_single{seed}'), f'{kind} {W.shape} {kw["method"]} ')


@pytest.mark.parametrize('seed', range(40))
def test_full_solve_random_family(want, seed):
    W, kind, kw = full_case(seed)
    b = port.solve(W, **kw)
    assert len(b) == 2
    for i, y in enumerate(b):
        assert_stage_equal(y, stored_stage(want, f'cross_full{seed}_s{i}'), f'{kind} {W.shape} {kw} stage{i} ')


@pytest.mark.parametrize('seed', range(20))
def test_helpers_random_family(want, seed):
    W, ints, Wi = helper_case(seed)
    p = f'cross_helpers{seed}'
    for center in (True, False):
        b = port.csd_decompose(W, center)
        for j, y in enumerate(b):
            x = want[f'{p}_csd{int(center)}_{j}']
            assert x.shape == y.shape and np.array_equal(x, y)
    assert np.array_equal(want[f'{p}_ints_csd'], port.int_arr_to_csd(ints))
    for dc in HELPER_DCS:
        b = port.kernel_decompose(Wi, dc)
        a = (want[f'{p}_kd{dc}_0'], want[f'{p}_kd{dc}_1'])
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]), dc
        assert np.array_equal(a[0].astype(np.float64) @ a[1].astype(np.float64), Wi)
