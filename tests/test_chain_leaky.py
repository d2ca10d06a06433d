"""Chains with leaky ReLU activations (``('leaky_relu', alpha)``, alone or in a sequence) without a GPU: ``chain_design``'s
condition adders and MSB muxes and its cost column, ``chain_front`` with stand-in sweeps, and the pricing and split
kernels under the SIMT shim, against the reference's own traces of whole models (tests/golden/chain_leaky.json.gz); the
emitters' text of the splits; the argument checks and pickling."""
import gzip
import json
import pickle
from pathlib import Path

import numpy as np
import pytest

from da4ml_b200 import emit
from da4ml_b200.cmvm import chain_design

from simt import pipeline_split as SPLIT
from test_chain_bias import trace_designs
from test_chain_lookup import emitted, tables_of
from test_pipeline_split import assert_split_equal

GOLDEN = Path(__file__).resolve().parent / 'golden' / 'chain_leaky.json.gz'
FNS = {'tanh': np.tanh}


def golden():
    return json.loads(gzip.decompress(GOLDEN.read_bytes()))


MODELS = [m['name'] for m in golden()['models']]


def model(name):
    return next(m for m in golden()['models'] if m['name'] == name)


def acts_of(m):
    def one(a):
        if a[0] == 'apply':
            return ('apply', FNS[a[1]], np.asarray(a[2], np.int64), *a[3:])
        if a[0] == 'leaky_relu':
            return tuple(a)
        return (a[0], np.asarray(a[1], np.int64))

    return [[one(a) for a in seq] for seq in m['activations']]


def stated_cost(d, m, designs, layer_costs):
    """The float32 sum in stage order of the chain design's cost column, each layer's cost taken as one value: a layer's
    stages, then its bias / activation stages (one, and one more per leaky ReLU)."""
    cost, pos = np.float32(0.0), 0
    for k, c in enumerate(layer_costs):
        cost = np.float32(cost + np.float32(c))
        pos += len(designs[k])
        seq = m['activations'][k] if k < len(m['activations']) else []
        n_act = (1 + sum(a[0] == 'leaky_relu' for a in seq)) if seq or (m['biases'][k] is not None) else 0
        for st in d.stages[pos : pos + n_act]:
            for v in np.asarray(st['ops_f'], np.float32)[:, 4]:
                cost = np.float32(cost + v)
        pos += n_act
    return cost


def hand_design():
    """The golden file's hand-made design with MSB muxes on a condition of their own (opcodes 6 and -6)."""
    stages = []
    for st in golden()['hand_muxes']['stages']:
        x = {k: np.asarray(st[k], np.int64) for k in ('inp_shifts', 'out_idxs', 'out_shifts', 'out_negs')}
        x['ops_i'] = np.asarray(st['ops_i'], np.int64).reshape(-1, 4)
        x['ops_f'] = np.asarray(st['ops_f_bits'], np.uint32).view(np.float32).reshape(-1, 5)
        x.update(adder_size=st['adder_size'], carry_size=st['carry_size'], shape=(len(x['inp_shifts']), len(x['out_idxs'])))
        stages.append(x)
    return stages


def check_hand_muxes(run):
    """``run(design, cutoff, latencies, retiming)`` -> a ``PipelinePrice`` with kept splits, against every task of the
    hand-made muxes: the split (its copies' row order in the muxes' stage follows each mux's events: operand 0, operand
    1, the condition), reg_bits and the emitters' text; retimed splits where every input is in the first stage."""
    d = hand_design()
    n = 0
    for t in golden()['hand_muxes']['tasks']:
        for rt in (False, True):
            pr = run(d, t['cutoff'], t['latencies'], rt)
            tag = (t['latencies'], t['cutoff'], rt)
            assert int(pr.status[0, 0]) == 0, tag
            rec = t['retimed'] if rt else t['split']
            if rt and not all(v < t['cutoff'] for v in (t['latencies'] or [0.0])):
                continue
            got = pr.split(0, 0)
            assert_split_equal(got, rec, tag)
            assert int(pr.reg_bits[0, 0]) == rec['reg_bits'], tag
            assert emitted(got)[0] == rec['text'], tag
            assert {int(v) for st in got for v in np.asarray(st['ops_i'])[:, 2] if abs(v) == 6} == set(t['opcodes']), tag
            n += 1
    return n


def ok_traces(m):
    return [t for t in m['traces'] if not t['raised']]


@pytest.mark.parametrize('name', MODELS)
def test_chain_design_muxes_equal_the_tracer(name):
    """Every condition adder and MSB mux of the chain design (interval, cost) is the one the tracer created, in value
    order; the muxes read the condition through ``data`` and carry ``max_of``'s interval."""
    m = model(name)
    n = 0
    for t in ok_traces(m):
        d = chain_design(trace_designs(m, t), acts_of(m), m['biases'])
        got_c, got_m = [], []
        for st, nx in zip(d.stages, d.stages[1:] + [None]):
            oi, of = np.asarray(st['ops_i']), np.asarray(st['ops_f'], np.float64)
            for r in np.flatnonzero(oi[:, 2] == 6).tolist():
                c = int(oi[r, 3]) & 0xFFFFFFFF
                assert oi[c, 2] == -1 and oi[r, 3] >> 32 == 0
                got_m.append(float(np.float32(of[r, 4])))
            if nx is not None and (np.asarray(nx['ops_i'])[:, 2] == 6).any():  # (the stage of the condition adders)
                for r in np.flatnonzero((oi[:, 2] == 1) & (oi[:, 0] == oi[:, 1])).tolist():
                    got_c.append([*of[r, :3].tolist(), float(np.float32(of[r, 4]))])
        want = [x for layer in t['muxes'] for x in layer]
        assert got_c == [[*x[0][:3], float(np.float32(x[0][3]))] for x in want], (name, t['choice'], t['cutoff'])
        assert got_m == [float(np.float32(x[1][3])) for x in want], (name, t['choice'], t['cutoff'])
        n += len(want)
    assert n > 0


def test_golden_covers_every_leaky_case():
    """The models reach every shortcut of ``max_of``: x itself, the view alpha * x, the constant 0, and the mux; and the
    hand-made design has both mux opcodes."""
    g = golden()
    cases = {c for m in g['models'] for t in ok_traces(m) for layer in t['leaky_cases'] for c in layer}
    assert cases == {'x', 'view', 'zero', 'mux'}
    assert all(t['opcodes'] == [-6, 6] for t in g['hand_muxes']['tasks'])


def test_hand_muxes_split_equal_the_tracer():
    assert check_hand_muxes(lambda d, c, lats, rt: SPLIT.split([d], c, None if lats is None else [lats], retiming=rt)) >= 16


@pytest.mark.parametrize('name', MODELS)
@pytest.mark.parametrize('retiming', [False, True])
def test_split_equals_the_tracer(name, retiming):
    """The chain design priced and split under the SIMT shim: the reference's split (ops, tables, reg_bits) and the
    emitters' text."""
    m = model(name)
    n = 0
    for t in ok_traces(m):
        rec = t['retimed'] if retiming else t['split']
        if rec is None or isinstance(rec, str):
            continue
        d = chain_design(trace_designs(m, t), acts_of(m), m['biases'])
        pr = SPLIT.split([d], t['cutoff'], retiming=retiming)
        assert int(pr.status[0, 0]) == 0
        got = pr.split(0, 0)
        tag = (name, t['choice'], t['cutoff'], retiming)
        assert_split_equal(got, rec, tag)
        assert tables_of(got) == rec['tables'], tag
        assert int(pr.reg_bits[0, 0]) == rec['reg_bits'], tag
        assert emitted(got) == (rec['text'], rec['mem']), tag
        n += 1
    assert n > 0


def test_split_binary_runs_the_traced_model():
    """The unretimed split of option set 0 at cutoff 5, stage by stage through the reference's DAIS interpreter, gives
    the traced model's outputs."""
    from oracle import dais_ref

    from da4ml_b200.types import stage_to_binary

    for name in MODELS:
        m = model(name)
        t = next(t for t in m['traces'] if t['choice'] == [0] * len(m['kernels']) and t['cutoff'] == 5.0)
        d = chain_design(trace_designs(m, t), acts_of(m), m['biases'])
        x = np.asarray(m['rows'], np.float64)
        for st in SPLIT.split([d], 5.0, retiming=False).split(0, 0):
            x = dais_ref.run(stage_to_binary(st), x)
        np.testing.assert_array_equal(x, np.asarray(m['outputs'], np.float64), err_msg=name)


def test_argument_errors():
    m = model('leaky_quantize_5x6x3')
    ds = trace_designs(m, ok_traces(m)[0])
    for bad in [0.3, 1.0, 2.0, 0.0, -0.5, float('nan'), float('inf'), True, '0.5', None]:
        with pytest.raises(ValueError, match=r"activation 0: \('leaky_relu', alpha\) needs alpha .*got"):
            chain_design(ds, [('leaky_relu', bad)])
    for act in [('leaky_relu',), ('leaky_relu', 0.125, (1, 2, 3)), ('leaky_relu', (1, 2, 3))]:
        with pytest.raises(ValueError, match='activation 0'):
            chain_design(ds, [act])
    with pytest.raises(ValueError, match='activation 0'):
        chain_design(ds, [[('quantize', (1, 6, 2)), ('leaky_relu', 0.3)]])


def test_emit_retrace_refuses_the_mux():
    m = model('leaky_negated_3x4x2')
    t = ok_traces(m)[0]
    d = chain_design(trace_designs(m, t), acts_of(m), m['biases'])
    st = next(s for s in d.stages if (np.asarray(s['ops_i'])[:, 2] == 6).any())
    with pytest.raises(ValueError, match='opcode 6'):
        emit._adder_graph(emit.as_stage(st))


@pytest.mark.parametrize('name', ['leaky_quantize_5x6x3', 'leaky_negated_3x4x2', 'bias_leaky_4x4x2', 'leaky_noop_2x4x2', 'leaky_noop_relu_2x4x2'])
@pytest.mark.parametrize('c', [0.0, 2.0, 3.0, 5.0])
def test_front_equals_the_tracer(name, c):
    """``chain_front`` with the oracle stand-in: every point is the tracer's trace of its choice of option sets -- its
    designs, reference calls (latencies through the condition adder and the mux, qintervals the muxes' traced
    intervals), cost (the float32 sum of the chain design's cost column) and, under a cutoff, its traced latency."""
    from da4ml_b200.cmvm import chain_front
    from golden.make_golden_chain_traced import digest
    from test_chain_traced import OracleSolver, simt_pricer

    g = golden()
    m = model(name)
    ks = [np.asarray(W, np.float32) for W in m['kernels']]
    kw = dict(latency_cutoff=c, pricer=simt_pricer) if c else {}
    f = chain_front(ks, g['sets'], qintervals=[[tuple(q) for q in m['qintervals']], None], solver=OracleSolver(), activations=acts_of(m), biases=m['biases'],
                    adder_size=m['adder_size'], carry_size=m['carry_size'], **kw)  # fmt: skip
    traces = {tuple(t['choice']): t for t in m['traces'] if t['cutoff'] == (c or 5.0)}
    assert len(f) > 0
    for p in range(len(f)):
        t = traces[tuple(int(v) for v in f.choice[p])]
        calls = f.reference_calls(p)
        if c:
            assert [call['latencies'] for call in calls] == [call['latencies'] for call in t['calls']]
        assert [[list(q) for q in call['qintervals']] for call in calls] == [call['qintervals'] for call in t['calls']]
        designs = [f.raw(p, k).stages for k in range(len(ks))]
        assert [digest(d) for d in designs] == [call['digest'] for call in t['calls']]
        assert f.cost[p] == stated_cost(f.design(p), m, designs, [call['cost'] for call in t['calls']])
        if c:
            assert float(f.latency[p]) == max(t['out_latency'])


def test_front_pickles_and_compares_alpha():
    from da4ml_b200.cmvm import chain_front
    from test_chain_traced import OracleSolver

    g = golden()
    m = model('leaky_quantize_5x6x3')
    ks = [np.asarray(W, np.float32) for W in m['kernels']]
    f = chain_front(ks, g['sets'], qintervals=[[tuple(q) for q in m['qintervals']], None], solver=OracleSolver(), activations=acts_of(m))
    f2 = pickle.loads(pickle.dumps(f))
    a, b = f.design(0), f2.design(0)
    assert [np.asarray(x).tolist() for x in a.to_binary()] == [np.asarray(x).tolist() for x in b.to_binary()]
    assert [np.asarray(x).tolist() for x in f.design(0, [[('leaky_relu', 0.125), ('quantize', (1, 6, 2))]]).to_binary()] == [np.asarray(x).tolist() for x in a.to_binary()]
    with pytest.raises(ValueError, match='differ'):
        f.design(0, [[('leaky_relu', 0.25), ('quantize', (1, 6, 2))]])
