"""Chain designs (``chain_design``: solver designs with relu / quantize stages between the layers) priced and split as one
pipeline without a GPU: the pricing and split kernels and their host code under the SIMT shim against the reference's
own traces of the whole chain (tests/golden/chain_pipeline.json.gz), ``chain_design``'s op fields against what the tracer
records, and the argument checks."""
import gzip
import json
from pathlib import Path

import numpy as np
import pytest

import da4ml_b200._binary as B
from da4ml_b200 import emit
from da4ml_b200.cmvm import chain_design

from golden.make_golden_chain_pipeline import text_digests
from simt import pipeline_split as SIM
from test_pipeline_split import assert_split_equal

GOLDEN = Path(__file__).resolve().parent / 'golden' / 'chain_pipeline.json.gz'


def chain_golden():
    return json.loads(gzip.decompress(GOLDEN.read_bytes()))


def _layer(stages):
    out = []
    for st in stages:
        x = {k: np.asarray(st[k], np.int64) for k in ('inp_shifts', 'out_idxs', 'out_shifts', 'out_negs')}
        x['ops_i'] = np.asarray(st['ops_i'], np.int64).reshape(-1, 4)
        x['ops_f'] = np.asarray(st['ops_f_bits'], np.uint32).view(np.float32).reshape(-1, 5)
        x.update(adder_size=st['adder_size'], carry_size=st['carry_size'], shape=(len(x['inp_shifts']), len(x['out_idxs'])))
        out.append(x)
    return out


def chain_designs():
    """(chain design, fixture record) of every chain of the fixture."""
    g = chain_golden()
    return [(chain_design([_layer(s) for s in c['layers']], [(kind, np.asarray(kif)) for kind, kif in c['activations']]), c) for c in g['chains']]


def check_chains_against_golden(run):
    """``run(designs, cutoffs, latencies, retiming)`` -> a ``PipelinePrice`` with kept splits.  Every task of the fixture:
    status, traced output latencies (where the run reports them), stages and register bits, and the split array for
    array; retimed splits where every input is in the first stage (the reference re-traces a split with its inputs at
    latency 0)."""
    designs = chain_designs()
    groups = {}
    for t in chain_golden()['tasks']:
        groups.setdefault((t['chain'], json.dumps(t['latencies'])), []).append(t)
    n_checked = n_retimed = 0
    for (c, _), ts in groups.items():
        cuts = sorted({t['cutoff'] for t in ts})
        lats = None if ts[0]['latencies'] is None else [ts[0]['latencies']]
        for rt in (False, True):
            pr = run([designs[c][0]], cuts, lats, rt)
            for t in ts:
                j = cuts.index(t['cutoff'])
                tag = (designs[c][1]['name'], t['latencies'], t['cutoff'], rt)
                assert int(pr.status[0, j]) == t['status'], tag
                if t['status'] != 0:
                    continue
                if pr._out_lat[0] is not None:
                    assert pr.out_latency(0, j).tolist() == t['out_latency'], tag
                if t['split'] is None:
                    with pytest.raises(ValueError, match='KeyError'):
                        pr.split(0, j)
                    continue
                if not rt:
                    assert (int(pr.stages[0, j]), int(pr.reg_bits[0, j])) == (t['split']['stages'], t['split']['reg_bits']), tag
                    assert_split_equal(pr.split(0, j), t['split'], tag)
                elif all(v < t['cutoff'] for v in (t['latencies'] or [0.0])):
                    r = t['retimed']
                    assert (int(pr.stages[0, j]), int(pr.reg_bits[0, j]), float(pr.cutoff[0, j])) == (r['stages'], r['reg_bits'], r['cutoff']), tag
                    assert_split_equal(pr.split(0, j), r, tag)
                    n_retimed += 1
                n_checked += 1
    assert n_checked > 120 and n_retimed > 30


@pytest.mark.parametrize('threads', [32, 128])
def test_simulated_chain_split_equals_reference(threads):
    check_chains_against_golden(lambda ds, cuts, lats, rt: SIM.split(ds, cuts, lats, rt, threads=threads))


def test_golden_covers_the_cases():
    designs = chain_designs()
    ok = [t for t in chain_golden()['tasks'] if t['status'] == 0]
    ops = lambda d: np.concatenate([st['ops_i'] for st in d.stages])  # noqa: E731
    assert any(np.isin(ops(d)[:, 2], (2,)).any() for d, _ in designs) and any(np.isin(ops(d)[:, 2], (3,)).any() for d, _ in designs)
    splits = [st for t in ok if t['split'] and 'full' in t['split'] for st in t['split']['full']]
    opc = {o[2] for st in splits for o in st['ops_i']}
    assert {2, 3} <= opc and ({-2, -3} & opc)  # relu / quantize of negated values too
    assert any(rec == 'self' for _, c in designs for recs in c['traced_ops'] for rec in recs)  # an activation that changes nothing
    assert any(isinstance(rec, list) and rec[0] == 'const' for _, c in designs for recs in c['traced_ops'] for rec in recs)  # a dead column
    assert any(t['split']['stages'] > 3 for t in ok if t['split'])
    assert any(t['latencies'] and max(t['latencies']) > 0 for t in ok)
    # a stage boundary between an activation and the op reading it, and one between an activation and its operand
    cross = False
    for t in ok:
        for a, b in zip((t['split'] or {}).get('full', [])[:-1], (t['split'] or {}).get('full', [])[1:]):
            outs = set(a['out_idxs'])
            cross |= any(a['ops_i'][i][2] in (2, -2, 3, -3) for i in outs)
    assert cross


def test_chain_design_fields_match_the_tracer():
    for d, c in chain_designs():
        n_layers = len(c['layers'])
        sizes = [len(layer) for layer in c['layers']]
        pos = np.cumsum([s + 1 for s in sizes])[:-1] - 1  # index of each activation stage
        assert len(d.stages) == sum(sizes) + n_layers - 1
        for k, recs in enumerate(c['traced_ops']):
            st = d.stages[pos[k]]
            n = len(recs)
            assert st['shape'] == (n, n) and st['ops_i'][:n].tolist() == [[j, -1, -1, 0] for j in range(n)]
            for j, rec in enumerate(recs):
                o = int(st['out_idxs'][j])
                if rec == 'self':
                    assert o == j, (c['name'], k, j)
                elif rec[0] == 'const':
                    assert rec[1] == 0.0 and o == -1, (c['name'], k, j)
                else:
                    opcode, data, q, _, cost = rec
                    assert st['ops_i'][o].tolist() == [j, -1, opcode, data], (c['name'], k, j)
                    # (the latency is the value's as its layer's design records it: a layer is solved as if its inputs were at 0)
                    assert st['ops_f'][o].tolist() == np.asarray([*q, st['ops_f'][j, 3], cost], np.float32).tolist(), (c['name'], k, j)


def test_chain_with_unchanged_values_is_the_concatenation():
    """Quantizers wider than every value change nothing: a three-layer chain design prices and splits as its layers'
    stages one after another."""
    d, c = chain_designs()[0]
    layers = [_layer(s) for s in c['layers']]
    wide = chain_design(layers, [('quantize', (1, 40, 40))] * 2)
    plain = B.RawPipeline.from_stages([st for layer in layers for st in layer])
    assert len(wide.stages) == len(plain.stages) + 2
    for rt in (False, True):
        a, b = SIM.split([wide], [2.0, 5.0], retiming=rt), SIM.split([plain], [2.0, 5.0], retiming=rt)
        for key in ('status', 'stages', 'reg_bits'):
            assert np.array_equal(getattr(a, key), getattr(b, key)), (rt, key)
        for j in range(2):
            if int(a.status[0, j]) == 0:
                x, y = a.split(0, j), b.split(0, j)
                assert len(x) == len(y) and all(np.array_equal(s[k], t[k]) for s, t in zip(x, y) for k in ('ops_i', 'ops_f', 'out_idxs')), (rt, j)


def _identity(qs, adder_size=-1, carry_size=-1):
    n = len(qs)
    return [dict(shape=(n, n), inp_shifts=np.zeros(n, np.int64), out_idxs=np.arange(n), out_shifts=np.zeros(n, np.int64), out_negs=np.zeros(n, np.int64),
                 ops_i=np.asarray([[j, -1, -1, 0] for j in range(n)], np.int64).reshape(-1, 4),
                 ops_f=np.asarray([[*q, 0.0, 0.0] for q in qs], np.float32).reshape(-1, 5), adder_size=adder_size, carry_size=carry_size)]  # fmt: skip


@pytest.mark.parametrize('kind', ['relu', 'quantize'])
def test_host_replay_agrees_with_chain_design(kind):
    """chain_design (Python) and pp_prepare (C++) apply the same relu / quantize rules: the activation ops the split
    writes carry chain_design's intervals, on edge cases (negative bounds with WRAP, formats with no bits left, dropped
    fractional and integer bits, values left unchanged)."""
    qs = [(-37.5, 21.25, 0.25), (-8.0, 7.75, 0.25), (0.0, 15.0, 1.0), (-1.0, 0.5, 0.5), (-100.0, -3.0, 1.0), (3.0, 200.0, 1.0), (-0.75, 0.25, 0.25), (-64.0, 63.0, 1.0)]
    kifs = [(0, 4, 1), (0, 2, 0), (0, 3, -1), (0, 0, 0), (0, 5, 2), (0, 6, 0), (0, 0, 1), (0, 7, 3)] if kind == 'relu' else \
        [(1, 3, 1), (0, 2, 0), (1, 1, -1), (0, -1, 0), (1, 5, 2), (0, 6, -2), (1, 0, 1), (1, 4, 3)]  # fmt: skip
    d = chain_design([_identity(qs), _identity([(0.0, 0.0, 1.0)] * len(qs))], [(kind, np.asarray(kifs))])
    act = d.stages[1]
    assert np.isin(act['ops_i'][:, 2], (2, 3)).sum() >= 4
    pr = SIM.split([d], 1000.0, retiming=False)
    (st,) = pr.split(0, 0)
    for j, o in enumerate(act['out_idxs'].tolist()):
        r = int(st['out_idxs'][j])
        if o < 0:  # the constant 0
            assert st['ops_i'][r, 2] == 5 and st['ops_f'][r, 0] == st['ops_f'][r, 1] == 0.0, j
        elif o == j:  # unchanged
            assert st['ops_i'][r, 2] == -1 and st['ops_i'][r, 0] == j, j
        else:
            assert st['ops_i'][r, 2] == act['ops_i'][o, 2], j
            assert st['ops_f'][r, :3].tolist() == act['ops_f'][o, :3].astype(np.float64).tolist() and st['ops_f'][r, 4] == act['ops_f'][o, 4], j


def test_chain_design_argument_errors():
    _, c = chain_designs()[0]
    l0, l1, l2 = (_layer(s) for s in c['layers'])
    with pytest.raises(ValueError, match='need 2 activations'):
        chain_design([l0, l1, l2], [('relu', (0, 4, 0))])
    with pytest.raises(ValueError, match='layer 0 has 5 outputs but layer 1 has 4 inputs'):
        chain_design([l0, l2], [('relu', (0, 4, 0))])
    with pytest.raises(ValueError, match="'tanh' is not"):
        chain_design([l0, l1], [('tanh', (0, 4, 0))])
    with pytest.raises(ValueError, match='rounding mode'):
        chain_design([l0, l1], [('quantize', (1, 4, 0), 'RND')])
    with pytest.raises(ValueError, match='overflow mode'):
        chain_design([l0, l1], [('quantize', (1, 4, 0), 'TRN', 'SAT')])
    with pytest.raises(ValueError, match=r'\[5, 3\]'):
        chain_design([l0, l1], [('quantize', np.zeros((4, 3), np.int64))])
    with pytest.raises(ValueError, match='0 for .relu'):
        chain_design([l0, l1], [('relu', (1, 4, 0))])
    with pytest.raises(ValueError, match='k must be 0 or 1'):
        chain_design([l0, l1], [('quantize', (2, 4, 0))])
    with pytest.raises(ValueError, match='integers'):
        chain_design([l0, l1], [('quantize', (1, 4.5, 0))])
    other = [dict(st, adder_size=3) for st in l1]
    with pytest.raises(ValueError, match='share adder_size'):
        chain_design([l0, other], [('relu', (0, 4, 0))])


def test_activation_ops_are_checked_on_the_host():
    d, _ = chain_designs()[0]
    stages = [dict(st) for st in d.stages]
    k = next(i for i, st in enumerate(stages) if np.isin(st['ops_i'][:, 2], (2, 3)).any())
    st = stages[k] = dict(stages[k])
    r = int(np.flatnonzero(np.isin(st['ops_i'][:, 2], (2, 3)))[0])
    st['ops_i'] = st['ops_i'].copy()
    st['ops_i'][r, 1] = 0  # relu / quantize read one operand
    with pytest.raises(ValueError, match='not an adder-graph op'):
        SIM.split([stages], 2.0)
    st['ops_i'][r, 1] = -1
    st['ops_f'] = st['ops_f'].copy()
    st['ops_f'][r, 2] = 0.3  # not a power-of-two step
    with pytest.raises(ValueError, match='not a quantized interval'):
        SIM.split([stages], 2.0)
    st['ops_f'][r, 2] = 1.0
    st['ops_i'][r, 2] = 4  # a constant addition: not covered
    with pytest.raises(ValueError, match='opcode 4'):
        SIM.split([stages], 2.0)


def test_emitted_text_equals_reference():
    """The Verilog, VHDL and HLS text of every split of the fixture (relu / quantize ops, negated operands and outputs
    included) against the sha256 of the reference emitters' text."""
    designs = chain_designs()
    groups = {}
    for t in chain_golden()['tasks']:
        groups.setdefault((t['chain'], json.dumps(t['latencies'])), []).append(t)
    n = 0
    for (c, _), ts in groups.items():
        cuts = sorted({t['cutoff'] for t in ts})
        lats = None if ts[0]['latencies'] is None else [ts[0]['latencies']]
        for rt, key in ((False, 'split'), (True, 'retimed')):
            pr = SIM.split([designs[c][0]], cuts, lats, rt, threads=128)
            for t in ts:
                rec = t.get(key) if t['status'] == 0 and t.get('split') else None
                if rec is None or rec.get('text') is None or (rt and not all(v < t['cutoff'] for v in (t['latencies'] or [0.0]))):
                    continue
                sp = pr.split(0, cuts.index(t['cutoff']))
                got = text_digests(emit.verilog_pipeline_logic_gen(sp, 'chain', print_latency=True), emit.vhdl_pipeline_logic_gen(sp, 'chain'),
                                   [emit.hls_logic_and_bridge_gen(s, f'chain{k}', 'vitis', print_latency=True) for k, s in enumerate(sp)])  # fmt: skip
                assert got == rec['text'], (designs[c][1]['name'], t['latencies'], t['cutoff'], rt)
                n += 1
    assert n > 100


def test_retrace_refuses_activations():
    d, _ = chain_designs()[0]
    with pytest.raises(ValueError, match='relu / quantize'):
        emit.retime_pipeline(d.stages)


def test_no_device_error():
    if B.device_info()['cuda_devices'] > 0:
        pytest.skip('a CUDA device is present')
    d, _ = chain_designs()[0]
    with pytest.raises(RuntimeError, match='no CUDA device'):
        B.price_pipelined([d], 2.0, keep_split=True)
