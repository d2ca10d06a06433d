"""chain_front with activations on the GPU: the real solve_sweep_batch and price_pipelined against the reference's own traces
of whole models (tests/golden/chain_traced.json.gz), every design against solve under its reference call, and the
cheapest point's whole-chain split against the same kernels under the SIMT shim.  -m gpu."""
import numpy as np
import pytest

import da4ml_b200._binary as B

from golden.make_golden_chain_traced import digest
from simt import pipeline_split as SIM
from test_chain_traced import check_front_against_golden, model_args, traced_golden
from test_pipeline_split_gpu import _assert_stages_equal

pytestmark = pytest.mark.gpu


def _solve_stages(W, **call):
    return B.solve_raw(np.asarray(W, np.float32), **call).stages


@pytest.mark.parametrize('c', [3.0, 5.0])
def test_front_matches_the_tracer(cuda_binary, c):
    g = traced_golden()
    for m in g['models']:
        kernels, qs, acts, cost_model = model_args(m)
        cf = B.chain_front(kernels, g['sets'], qintervals=qs, latency_cutoff=c, activations=acts, **cost_model)
        check_front_against_golden(cf, m, g['sets'], c, _solve_stages)
        for p in range(len(cf)):
            for k, W in enumerate(kernels):
                assert digest(B.solve_raw(W, **cf.reference_calls(p)[k]).stages) == digest(cf.raw(p, k).stages), (m['name'], c, p, k)


@pytest.mark.parametrize('c', [0.0, 3.0])
def test_every_design_is_its_reference_solve(cuda_binary, c):
    rng = np.random.default_rng(5)
    kernels = [rng.integers(-32, 32, size=(12, 16)).astype(np.float32), rng.integers(-16, 16, size=(16, 10)).astype(np.float32),
               rng.integers(-16, 16, size=(10, 6)).astype(np.float32)]  # fmt: skip
    sets = [dict(method0='wmc'), dict(method0='wmc', hard_dc=2), dict(method0='mc', decompose_dc=1), dict(method0='wmc-dc', hard_dc=1)]
    acts = [('relu', (0, 9, 0)), ('quantize', [(1, 8, 0) if j % 3 else (0, 6, 1) for j in range(10)])]
    cf = B.chain_front(kernels, sets, qintervals=[[(-32.0, 31.0, 1.0)] * 12, None, None], latency_cutoff=c, activations=acts, adder_size=-1, carry_size=12)
    assert len(cf) >= 1
    for p in range(len(cf)):
        calls = cf.reference_calls(p)
        for k, W in enumerate(kernels):
            assert digest(B.solve_raw(W, **calls[k]).stages) == digest(cf.raw(p, k).stages), (c, p, k)


@pytest.mark.parametrize('c', [3.0, 5.0])
def test_best_point_split(cuda_binary, c):
    g = traced_golden()
    kernels, qs, acts, cost_model = model_args(g['models'][1])
    cf = B.chain_front(kernels, g['sets'], qintervals=qs, latency_cutoff=c, activations=acts, **cost_model)
    p = int(np.argmin(cf.cost))  # (the cheapest point)
    d = cf.design(p)
    assert any(np.isin(st['ops_i'][:, 2], (2, 3)).any() for st in d.stages)
    for rt in (False, True):
        got = B.price_pipelined([d], [c, 2 * c], retiming=rt, keep_split=True)
        want = SIM.split([d], [c, 2 * c], retiming=rt, threads=128)
        for key in ('status', 'stages', 'reg_bits'):
            assert np.array_equal(getattr(got, key), getattr(want, key)), (c, rt, key)
        assert np.array_equal(got.latency_max.view(np.uint64), want.latency_max.view(np.uint64)), (c, rt)
        for j in range(2):
            if int(got.status[0, j]) == 0:
                _assert_stages_equal(got.split(0, j), want.split(0, j), (c, rt, j))
