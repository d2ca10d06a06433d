"""Chain designs priced and split as one pipeline on the GPU: ``price_pipelined(chain_design(...), ..., keep_split=True)``
against the reference's own traces of the whole chain (tests/golden/chain_pipeline.json.gz), the best points of a
pipelined ``chain_front`` against the same kernels under the SIMT shim, and a chain whose activations change nothing
against the layers priced one after another."""
import numpy as np
import pytest

import da4ml_b200._binary as B
from da4ml_b200.cmvm import chain_design

from simt import pipeline_split as SIM
from test_chain_pipeline import check_chains_against_golden
from test_pipeline_split_gpu import _assert_stages_equal

pytestmark = pytest.mark.gpu


def test_chain_split_equals_reference():
    check_chains_against_golden(lambda ds, cuts, lats, rt: B.price_pipelined(ds, cuts, lats, rt, keep_split=True))


def _front(c):
    rng = np.random.default_rng(23)
    kernels = [rng.integers(-32, 32, size=(12, 12)).astype(np.float32), rng.integers(-16, 16, size=(12, 10)).astype(np.float32),
               rng.integers(-16, 16, size=(10, 6)).astype(np.float32)]  # fmt: skip
    sets = [dict(method0='wmc'), dict(method0='wmc', hard_dc=2), dict(method0='mc', decompose_dc=1)]
    return B.chain_front(kernels, sets, latencies=[0.0] * 12, latency_cutoff=c, adder_size=-1, carry_size=12)


@pytest.mark.parametrize('c', [2.0, 3.0, 5.0])
def test_chain_front_best_point_split(c):
    front = _front(c)
    p = int(np.argmin(front.cost))  # (the cheapest point)
    acts = [('relu', (0, 9, 0)), ('quantize', [(1, 8, 0) if j % 3 else (0, 6, 1) for j in range(10)])]
    d = front.design(p, acts)
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


@pytest.mark.parametrize('c', [3.0, 5.0])
def test_chain_without_activations_is_the_concatenation(c):
    """Quantizers wider than every value change nothing: the chain design prices and splits as the layers' stages one
    after another."""
    front = _front(c)
    for p in range(min(len(front), 4)):
        d = front.design(p, [('quantize', (1, 40, 40)), ('quantize', (1, 40, 40))])
        plain = B.RawPipeline.from_stages([st for k in range(3) for st in front.raw(p, k).stages])
        assert len(d.stages) == len(plain.stages) + 2
        for rt in (False, True):
            a = B.price_pipelined([d], [c, 2 * c], retiming=rt, keep_split=True)
            b = B.price_pipelined([plain], [c, 2 * c], retiming=rt, keep_split=True)
            for key in ('status', 'stages', 'reg_bits', 'latency_max', 'cutoff'):
                assert np.array_equal(getattr(a, key), getattr(b, key), equal_nan=True), (p, rt, key)
            for j in range(2):
                if int(a.status[0, j]) == 0:
                    _assert_stages_equal(a.split(0, j), b.split(0, j), (p, rt, j))
