"""CMVM solves whose centred values reach the int32 limit of the CSD step (tests/cmvm_int32_cases.py), checked against
the reference's stored answers (tests/golden/cmvm_int32_edge.json.gz, tests/golden/make_golden_int32_edge.py).

At 32 CSD digits the reference's digit loop wraps in int32 (the threshold ``2^31 * 2 / 3`` is 0), and a centred value
outside the int32 range, or NaN, converts to INT_MIN as x86 ``cvttss2si`` gives it.  The port must keep both to stay a
valid checker here, and the simulated kernels show that the device sources reproduce them.  No GPU."""
import numpy as np
import pytest
from cmvm_int32_cases import KD_DCS, METHODS, SOLVES, ints, matrices
from conftest import assert_stage_equal
from test_oracle_cross import load_stored, stored_stage

import simt
from oracle import port

CASES = matrices()
INTS = ints()


@pytest.fixture(scope='module')
def want():
    return load_stored('cmvm_int32_edge.json.gz')


def solve_key(dc, search_all):
    return f'solve{dc}{"a" if search_all else ""}'


@pytest.mark.parametrize('name', list(CASES))
def test_port_solve_single(want, name):
    W = CASES[name]
    for m in METHODS:
        assert_stage_equal(port.solve_single(W, m), stored_stage(want, f'{name}_single_{m}'), f'{name} {m} ')


@pytest.mark.parametrize('name', list(CASES))
def test_port_solve(want, name):
    W = CASES[name]
    for dc, search_all in SOLVES:
        stages = port.solve(W, decompose_dc=dc, search_all_decompose_dc=search_all)
        assert len(stages) == 2
        for i, st in enumerate(stages):
            key = f'{name}_{solve_key(dc, search_all)}_s{i}'
            assert_stage_equal(st, stored_stage(want, key), f'{key} ')


def assert_helpers_equal(want, name, csd_decompose, kernel_decompose):
    W = CASES[name]
    for center in (True, False):
        for j, y in enumerate(csd_decompose(W, center)):
            x = want[f'{name}_csd{int(center)}_{j}']
            assert x.shape == y.shape and np.array_equal(x, y), f'csd_decompose center={center} output {j}'
    for dc in KD_DCS:
        m0, m1 = kernel_decompose(W, dc)
        for j, y in enumerate((m0, m1)):
            x = want[f'{name}_kd{dc}_{j}']
            assert x.shape == y.shape and np.array_equal(x.view(np.uint32), y.view(np.uint32)), f'kernel_decompose dc={dc} m{j}'


@pytest.mark.parametrize('name', list(CASES))
def test_port_helpers(want, name):
    assert_helpers_equal(want, name, port.csd_decompose, port.kernel_decompose)


@pytest.mark.parametrize('name', list(INTS))
def test_port_int_arr_to_csd(want, name):
    x = INTS[name]
    y = port.int_arr_to_csd(x)
    assert np.array_equal(want[f'ints_{name}'], y)
    # the digits sum back to the value modulo 2^32 at every width; INT_MIN takes no part in choosing the width
    w = (y.astype(np.int64) * (np.int64(1) << np.arange(y.shape[-1], dtype=np.int64))).sum(-1)
    keep = x != np.int32(-(2**31))
    assert np.array_equal(w.astype(np.uint32)[keep], x.view(np.uint32)[keep])


@pytest.mark.parametrize('name', list(CASES))
def test_simulated_kernel_solve_single(want, name):
    W = CASES[name]
    for i, m in enumerate(METHODS):
        got, _ = simt.solve_single(W, m, ctas=1 + i % 3, cta_threads=64)
        assert_stage_equal(got, stored_stage(want, f'{name}_single_{m}'), f'{name} {m} ')


@pytest.mark.parametrize('name', list(CASES))
def test_simulated_kernel_decompose(want, name):
    W = CASES[name]
    for dc in KD_DCS:
        m0, m1 = simt.kernel_decompose(W, dc)
        for j, y in enumerate((m0, m1)):
            x = want[f'{name}_kd{dc}_{j}']
            assert np.array_equal(x.view(np.uint32), y.view(np.uint32)), f'{name} kernel_decompose dc={dc} m{j}'
