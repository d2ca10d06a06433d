"""Chains with biases on the GPU: the real solve_sweep_batch and price_pipelined against the reference's own traces of
whole models (tests/golden/chain_bias.json.gz), every design against solve under its reference call, the cheapest
point's whole-chain split against the same kernels under the SIMT shim and the golden, and the chain design's stages run
by the DAIS interpreter on the golden's input rows against the traced model's outputs.  -m gpu."""
import numpy as np
import pytest

import da4ml_b200._binary as B
from da4ml_b200.dais import DaisProgram

from golden.make_golden_chain_traced import digest
from simt import pipeline_split as SIM
from test_chain_bias import OK_MODELS, model, model_args, stated_cost, trace_designs
from test_pipeline_split import assert_split_equal
from test_pipeline_split_gpu import _assert_stages_equal

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('name', OK_MODELS)
@pytest.mark.parametrize('c', [3.0, 5.0])
def test_front_matches_the_tracer(cuda_binary, name, c):
    g, m = model(name)
    kernels, qs, acts, biases, cm = model_args(m)
    cf = B.chain_front(kernels, g['sets'], qintervals=qs, latency_cutoff=c, activations=acts, biases=biases, **cm)
    traces = {(tuple(t['choice']), t['cutoff']): t for t in m['traces']}
    for p in range(len(cf)):
        calls = cf.reference_calls(p)
        choice = tuple(next(s for s, o in enumerate(g['sets']) if all(call[key] == v for key, v in o.items())) for call in calls)
        t = traces[choice, c]
        for k, (W, gc) in enumerate(zip(kernels, t['calls'])):
            assert digest(cf.raw(p, k).stages) == gc['digest'], (name, c, p, k)
            assert digest(B.solve_raw(W, **calls[k]).stages) == gc['digest'], (name, c, p, k)
        designs = [cf.raw(p, k).stages for k in range(len(kernels))]
        assert cf.cost[p].view(np.uint32) == stated_cost(cf.design(p), m, designs, [gc['cost'] for gc in t['calls']]).view(np.uint32), (name, c, p)
        assert float(cf.latency[p]) == max(t['out_latency']), (name, c, p)


@pytest.mark.parametrize('name', OK_MODELS)
@pytest.mark.parametrize('c', [3.0, 5.0])
def test_best_point_split(cuda_binary, name, c):
    g, m = model(name)
    kernels, qs, acts, biases, cm = model_args(m)
    cf = B.chain_front(kernels, g['sets'], qintervals=qs, latency_cutoff=c, activations=acts, biases=biases, **cm)
    p = int(np.argmin(cf.cost))
    d = cf.design(p)
    assert any((st['ops_i'][:, 2] == 4).any() for st in d.stages)
    calls = cf.reference_calls(p)
    choice = [next(s for s, o in enumerate(g['sets']) if all(call[key] == v for key, v in o.items())) for call in calls]
    t = next(t for t in m['traces'] if t['choice'] == choice and t['cutoff'] == c)
    for rt, key in ((False, 'split'), (True, 'retimed')):
        got = B.price_pipelined([d], c, retiming=rt, keep_split=True)
        want = SIM.split([d], c, retiming=rt, threads=128)
        for k in ('status', 'stages', 'reg_bits'):
            assert np.array_equal(getattr(got, k), getattr(want, k)), (name, c, rt, k)
        assert np.array_equal(got.latency_max.view(np.uint64), want.latency_max.view(np.uint64)), (name, c, rt)
        _assert_stages_equal(got.split(0, 0), want.split(0, 0), (name, c, rt))
        assert (int(got.stages[0, 0]), int(got.reg_bits[0, 0])) == (t[key]['stages'], t[key]['reg_bits']), (name, c, rt)
        assert_split_equal(got.split(0, 0), t[key], (name, c, rt))


@pytest.mark.parametrize('name', OK_MODELS)
def test_split_computes_the_traced_model(cuda_binary, name):
    """``price_pipelined(keep_split=True)`` of the chain design of option set 0 at cutoff 5, each register stage run by the
    DAIS interpreter on the GPU, gives the traced model's outputs on the golden's input rows exactly.  (The chain
    design's own stages keep each layer's solver intervals, which need not bound the traced values inside a multi-stage
    layer design; the split carries the tracer's.)"""
    _, m = model(name)
    _, _, acts, biases, _ = model_args(m)
    t = next(t for t in m['traces'] if t['choice'] == [0] * len(m['kernels']) and t['cutoff'] == 5.0)
    d = B.chain_design(trace_designs(m, t), acts, biases)
    for rt in (False, True):
        pr = B.price_pipelined([d], 5.0, retiming=rt, keep_split=True)
        sp = pr.split(0, 0)
        assert any((st['ops_i'][:, 2] == 4).any() for st in sp)
        x = np.asarray(m['rows'], np.float64)
        for st in sp:
            with DaisProgram(B.RawPipeline.from_stages([st]).to_binary()[0]) as prog:
                x = np.asarray(prog(x), np.float64)
        assert x.tolist() == m['outputs'], (name, rt)
