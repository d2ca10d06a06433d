"""Chains with lookup-table activations (``('apply', fn, kif[, round_mode[, overflow_mode]])``, alone or in a sequence)
without a GPU: ``chain_design``'s lookup ops and tables, and the split kernels under the SIMT shim with their tables,
against the reference's own traces of whole models (tests/golden/chain_lookup.json.gz); the DAIS binary of a split;
the argument checks, the constant refusal, and that a one-element list is the single activation."""
import gzip
import hashlib
import json
import pickle
from pathlib import Path

import numpy as np
import pytest

from da4ml_b200 import emit
from da4ml_b200.cmvm import chain_design

import chain_lookup_fns as F
from golden.make_golden_chain_pipeline import text_digests
from simt import pipeline_split as SPLIT
from test_chain_bias import trace_designs
from test_pipeline_split import assert_split_equal

GOLDEN = Path(__file__).resolve().parent / 'golden' / 'chain_lookup.json.gz'
FNS = {'tanh': np.tanh, 'sigmoid': F.sigmoid, 'odd_cube': F.odd_cube}
OK_MODELS = ['quantize_tanh_6x5x3', 'bias_relu_sigmoid_5x4x3', 'odd_narrow_3x4x2', 'wide_tanh_5x4x2']


def golden():
    return json.loads(gzip.decompress(GOLDEN.read_bytes()))


def model(name):
    return next(m for m in golden()['models'] if m['name'] == name)


def acts_of(m):
    return [[('apply', FNS[a[1]], np.asarray(a[2], np.int64), *a[3:]) if a[0] == 'apply' else (a[0], np.asarray(a[1], np.int64)) for a in seq]
            for seq in m['activations']]  # fmt: skip


def sha(t):
    return hashlib.sha256(np.asarray(t, np.int32).tobytes()).hexdigest()


def emitted(stages):
    """(sha256 of the Verilog / VHDL / HLS text, sha256 of every .mem file by name) of a split."""
    text = text_digests(emit.verilog_pipeline_logic_gen(stages, 'chain', print_latency=True), emit.vhdl_pipeline_logic_gen(stages, 'chain'),
                        [emit.hls_logic_and_bridge_gen(s, f'chain{k}', 'vitis', print_latency=True) for k, s in enumerate(stages)])  # fmt: skip
    return text, {k: hashlib.sha256(v.encode()).hexdigest() for k, v in sorted(emit.table_mem_gen(stages).items())}


def tables_of(stages):
    return [[[sha(t['table']), [float(v) for v in t['out_qint']]] for t in st.get('lookup_tables', [])] for st in stages]


@pytest.mark.parametrize('name', OK_MODELS)
def test_chain_design_lookups_equal_the_tracer(name):
    """Every lookup op of the chain design (interval, cost, table) is the one the tracer created, in value order."""
    m = model(name)
    for t in m['traces']:
        d = chain_design(trace_designs(m, t), acts_of(m), m['biases'])
        got = []
        for st in d.stages:
            oi, of = np.asarray(st['ops_i']), np.asarray(st['ops_f'], np.float64)
            for r in np.flatnonzero(oi[:, 2] == 8).tolist():
                got.append([*of[r, :3].tolist(), float(np.float32(of[r, 4])), sha(st['lookup_tables'][oi[r, 3]]['table'])])
        want = [[*x[:3], float(np.float32(x[3])), x[5]] for layer in t['lookups'] for x in layer]
        assert got == want, (name, t['choice'], t['cutoff'])


@pytest.mark.parametrize('name', OK_MODELS)
@pytest.mark.parametrize('retiming', [False, True])
def test_split_equals_the_tracer(name, retiming):
    """The chain design priced and split under the SIMT shim: the reference's split (ops, tables, reg_bits) and output
    latencies."""
    m = model(name)
    n = 0
    for t in m['traces']:
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

    for name in OK_MODELS:
        m = model(name)
        t = next(t for t in m['traces'] if t['choice'] == [0] * len(m['kernels']) and t['cutoff'] == 5.0)
        d = chain_design(trace_designs(m, t), acts_of(m), m['biases'])
        pr = SPLIT.split([d], 5.0, retiming=False)
        from da4ml_b200.types import stage_to_binary

        x = np.asarray(m['rows'], np.float64)
        for st in pr.split(0, 0):
            x = dais_ref.run(stage_to_binary(st), x)
        np.testing.assert_array_equal(x, np.asarray(m['outputs'], np.float64), err_msg=name)


def test_dead_column_into_sigmoid_is_refused():
    m = model('dead_sigmoid_4x3x2')
    with pytest.raises(ValueError, match='constant 0.5'):
        chain_design(trace_designs(m, m['traces'][0]), acts_of(m), m['biases'])


def test_one_element_list_is_the_single_activation():
    m = model('odd_narrow_3x4x2')
    t = m['traces'][0]
    ds = trace_designs(m, t)
    a = chain_design(ds, [acts_of(m)[0][0]])
    b = chain_design(ds, [[acts_of(m)[0][0]]])
    for x, y in zip(a.stages, b.stages):
        assert pickle.dumps({k: v for k, v in x.items()}) == pickle.dumps({k: v for k, v in y.items()})
    assert [np.asarray(p).tolist() for p in a.to_binary()] == [np.asarray(p).tolist() for p in b.to_binary()]
    with pytest.raises(ValueError, match='opcode 8'):
        a.to_pipeline()
    with pytest.raises(ValueError, match='opcode 8'):
        a.to_json()


def test_argument_errors():
    m = model('quantize_tanh_6x5x3')
    ds = trace_designs(m, m['traces'][0])
    for act, msg in [(('apply', 3.0, (1, 0, 6)), 'callable'), (('apply', np.tanh), "expected .*'apply', fn, kif"), (('apply', np.tanh, (1, 0)), 'kif'), (('apply', np.tanh, (1, 0, 6), 'RND_CONV'), 'rounding mode'),
                     (('apply', np.tanh, (1, 0, 6), 'TRN', 'WRAP_SM'), 'overflow mode'), ([], 'non-empty'), (('tanh', (1, 0, 6)), "'tanh' is not")]:
        with pytest.raises(ValueError, match=msg):
            chain_design(ds, [act])
    with pytest.raises(ValueError, match='rounding mode'):  # (relu / quantize keep TRN / WRAP only)
        chain_design(ds, [[('quantize', (1, 2, 3), 'RND'), ('apply', np.tanh, (1, 0, 6))]])


@pytest.mark.parametrize('name', ['quantize_tanh_6x5x3', 'wide_tanh_5x4x2', 'bias_relu_sigmoid_5x4x3'])
@pytest.mark.parametrize('c', [0.0, 3.0, 5.0])
def test_front_equals_the_tracer(name, c):
    """``chain_front`` with the oracle stand-in: every point is the tracer's trace of its choice of option sets -- its
    designs, reference calls (latencies including each lookup's increment, qintervals the table outputs' traced
    intervals), cost (the float32 sum of the chain design's cost column) and, under a cutoff, its traced latency."""
    from da4ml_b200.cmvm import chain_front
    from golden.make_golden_chain_traced import digest
    from test_chain_bias import stated_cost
    from test_chain_traced import OracleSolver, simt_pricer

    g = golden()
    m = model(name)
    ks = [np.asarray(W, np.float32) for W in m['kernels']]
    kw = dict(latency_cutoff=c, pricer=simt_pricer) if c else {}
    f = chain_front(ks, g['sets'], qintervals=[[tuple(q) for q in m['qintervals']], None], solver=OracleSolver(), activations=acts_of(m), biases=m['biases'],
                    adder_size=m['adder_size'], carry_size=m['carry_size'], **kw)  # fmt: skip
    assert [layer['dropped_constant'] for layer in f.profile['layers']] == [0, 0]
    traces = {tuple(t['choice']): t for t in m['traces'] if t['cutoff'] == (c or 5.0)}
    assert len(f) > 0
    for p in range(len(f)):
        t = traces[tuple(int(v) for v in f.choice[p])]
        calls = f.reference_calls(p)
        assert [call['latencies'] for call in calls] == [call['latencies'] for call in t['calls']]
        assert [[list(q) for q in call['qintervals']] for call in calls] == [call['qintervals'] for call in t['calls']]
        designs = [f.raw(p, k).stages for k in range(len(ks))]
        assert [digest(d) for d in designs] == [call['digest'] for call in t['calls']]
        assert f.cost[p] == stated_cost(f.design(p), m, designs, [call['cost'] for call in t['calls']])
        if c:
            assert float(f.latency[p]) == max(t['out_latency'])


def test_front_drops_a_dead_column_into_sigmoid():
    """Every candidate of layer 0 has the dead column, which sigmoid makes the constant 0.5: all are dropped."""
    from da4ml_b200.cmvm import chain_front
    from test_chain_traced import OracleSolver

    m = model('dead_sigmoid_4x3x2')
    with pytest.raises(ValueError, match='^layer 0: .*non-zero constant'):
        chain_front([np.asarray(W, np.float32) for W in m['kernels']], golden()['sets'], qintervals=[[tuple(q) for q in m['qintervals']], None],
                    solver=OracleSolver(), activations=acts_of(m))  # fmt: skip


def test_front_pickles_and_checks_its_activations():
    """A front using a module-level ``fn`` pickles and gives the same design; other activations are refused, also
    when an ``apply`` before them is given as another function object with the same tables."""
    from da4ml_b200.cmvm import chain_front
    from test_chain_traced import OracleSolver

    g = golden()
    m = model('quantize_tanh_6x5x3')
    ks = [np.asarray(W, np.float32) for W in m['kernels']]
    f = chain_front(ks, g['sets'], qintervals=[[tuple(q) for q in m['qintervals']], None], solver=OracleSolver(), activations=acts_of(m))
    f2 = pickle.loads(pickle.dumps(f))
    a, b = f.design(0), f2.design(0)
    assert [np.asarray(x).tolist() for x in a.to_binary()] == [np.asarray(x).tolist() for x in b.to_binary()]
    same = [[('quantize', (1, 2, 3)), ('apply', lambda x: np.tanh(x), (1, 0, 6))]]
    assert [np.asarray(x).tolist() for x in f.design(0, same).to_binary()] == [np.asarray(x).tolist() for x in a.to_binary()]
    with pytest.raises(ValueError, match='differ'):
        f.design(0, [[('quantize', (1, 2, 3)), ('apply', F.odd_cube, (1, 0, 6))]])
    with pytest.raises(ValueError, match='differ'):
        f.design(0, [[('quantize', (1, 2, 3)), ('apply', lambda x: np.tanh(x), (1, 0, 6)), ('relu', (0, 2, 6))]])
