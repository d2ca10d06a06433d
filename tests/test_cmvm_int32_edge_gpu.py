"""The CUDA path against the reference's stored answers where CSD digits reach the int32 limit (tests/cmvm_int32_cases.py,
tests/golden/cmvm_int32_edge.json.gz), and on the stored random family of tests/test_oracle_cross.py.  -m gpu.

At 32 digits the reference's digit loop wraps in int32, and a centred value out of the int32 range or NaN converts to
INT_MIN (x86 ``cvttss2si``) where a plain device cast would saturate.  Every solve entry point and every helper runs on
the device and must give the reference's answer bit for bit."""
import numpy as np
import pytest
from cmvm_int32_cases import KD_DCS, METHODS, SOLVES, ints, matrices
from conftest import assert_stage_equal, int_matrix
from test_oracle_cross import HELPER_DCS, full_case, helper_case, load_stored, single_case, stored_stage

pytestmark = pytest.mark.gpu

CASES = matrices()
INTS = ints()


@pytest.fixture(scope='module')
def want():
    return load_stored('cmvm_int32_edge.json.gz')


@pytest.fixture(scope='module')
def cross():
    return load_stored('reference_checks.json.gz')


def solve_key(dc, search_all):
    return f'solve{dc}{"a" if search_all else ""}'


def assert_float_equal(x, y, tag):
    """Bit for bit, except that a NaN only has to be a NaN: the GPU's float units return the canonical NaN 0x7fffffff,
    where x86 passes the input's sign and payload through (kernel_decompose of a matrix that holds a NaN)."""
    x, y = np.asarray(x, np.float32), np.asarray(y, np.float32)
    assert x.shape == y.shape, tag
    nan = np.isnan(x)
    assert np.array_equal(nan, np.isnan(y)) and np.array_equal(x[~nan].view(np.uint32), y[~nan].view(np.uint32)), tag


@pytest.mark.parametrize('name', list(CASES))
def test_solve_single(cuda_binary, want, name):
    for m in METHODS:
        raw, _ = cuda_binary.solve_single_raw(CASES[name], m)
        assert len(raw.stages) == 1
        assert_stage_equal(raw.stages[0], stored_stage(want, f'{name}_single_{m}'), f'{name} {m} ')


@pytest.mark.parametrize('name', list(CASES))
def test_solve(cuda_binary, want, name):
    for dc, search_all in SOLVES:
        raw = cuda_binary.solve_raw(CASES[name], decompose_dc=dc, search_all_decompose_dc=search_all)
        assert len(raw.stages) == 2
        for i, st in enumerate(raw.stages):
            key = f'{name}_{solve_key(dc, search_all)}_s{i}'
            assert_stage_equal(st, stored_stage(want, key), f'{key} ')


def test_solve_batch_whole_family(cuda_binary, want):
    """The whole family in one batch, next to ordinary matrices whose answers are those of their own solves."""
    names = list(CASES)
    plain = [int_matrix(6, 5, 6, 1), int_matrix(12, 9, 8, 2), int_matrix(3, 4, 3, 3)]
    mats = plain[:2] + [CASES[n] for n in names] + plain[2:]
    for dc, search_all in SOLVES:
        got = cuda_binary.solve_batch_raw(mats, decompose_dc=dc, search_all_decompose_dc=search_all)
        assert len(got) == len(mats)
        for name, raw in zip(names, got[2:-1]):
            for i, st in enumerate(raw.stages):
                key = f'{name}_{solve_key(dc, search_all)}_s{i}'
                assert_stage_equal(st, stored_stage(want, key), f'batched {key} ')
        for W, raw in zip(plain, got[:2] + got[-1:]):
            alone = cuda_binary.solve_raw(W, decompose_dc=dc, search_all_decompose_dc=search_all)
            for a, b in zip(raw.stages, alone.stages, strict=True):
                assert_stage_equal(a, b, f'plain {W.shape} dc={dc} ')


@pytest.mark.parametrize('name', list(CASES))
def test_helpers(cuda_binary, want, name):
    W = CASES[name]
    for center in (True, False):
        for j, y in enumerate(cuda_binary.csd_decompose(W, center)):
            x = want[f'{name}_csd{int(center)}_{j}']
            assert x.shape == y.shape and np.array_equal(x, y), f'csd_decompose center={center} output {j}'
    for dc in KD_DCS:
        m0, m1 = cuda_binary.kernel_decompose(W, dc)
        assert_float_equal(want[f'{name}_kd{dc}_0'], m0, f'kernel_decompose dc={dc} m0')
        assert_float_equal(want[f'{name}_kd{dc}_1'], m1, f'kernel_decompose dc={dc} m1')


@pytest.mark.parametrize('name', list(INTS))
def test_int_arr_to_csd(cuda_binary, want, name):
    y = cuda_binary.int_arr_to_csd(INTS[name])
    x = want[f'ints_{name}']
    assert x.shape == y.shape and np.array_equal(x, y)


# ---- the stored random family of test_oracle_cross.py, so far checked against the port only


@pytest.mark.parametrize('seed', range(60))
def test_cross_single_stage_family(cuda_binary, cross, seed):
    W, kind, kw = single_case(seed)
    raw, _ = cuda_binary.solve_single_raw(W, **kw)
    assert_stage_equal(raw.stages[0], stored_stage(cross, f'cross_single{seed}'), f'{kind} {W.shape} {kw["method"]} ')


@pytest.mark.parametrize('seed', range(40))
def test_cross_full_solve_family(cuda_binary, cross, seed):
    W, kind, kw = full_case(seed)
    raw = cuda_binary.solve_raw(W, **kw)
    assert len(raw.stages) == 2
    for i, st in enumerate(raw.stages):
        assert_stage_equal(st, stored_stage(cross, f'cross_full{seed}_s{i}'), f'{kind} {W.shape} {kw} stage{i} ')


@pytest.mark.parametrize('seed', range(20))
def test_cross_helpers_family(cuda_binary, cross, seed):
    W, ints_, Wi = helper_case(seed)
    p = f'cross_helpers{seed}'
    for center in (True, False):
        for j, y in enumerate(cuda_binary.csd_decompose(W, center)):
            x = cross[f'{p}_csd{int(center)}_{j}']
            assert x.shape == y.shape and np.array_equal(x, y), f'csd_decompose center={center} output {j}'
    assert np.array_equal(cross[f'{p}_ints_csd'], cuda_binary.int_arr_to_csd(ints_))
    for dc in HELPER_DCS:
        m0, m1 = cuda_binary.kernel_decompose(Wi, dc)
        assert_float_equal(cross[f'{p}_kd{dc}_0'], m0, f'kernel_decompose dc={dc} m0')
        assert_float_equal(cross[f'{p}_kd{dc}_1'], m1, f'kernel_decompose dc={dc} m1')
