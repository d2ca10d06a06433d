"""Register stages of solver designs (``price_pipelined(..., keep_split=True).split(d, j)``) without a GPU: the split kernels
and their host code under the SIMT shim against the reference's own splits (tests/golden/pipeline_split.json.gz) and
against ``emit``'s Python re-trace / split / retiming, ``split()``'s errors, and the argument checks of the new path."""
import gzip
import hashlib
import json
from pathlib import Path

import numpy as np
import pytest

import da4ml_b200._binary as B
from da4ml_b200 import emit

from golden.make_golden_pipeline_split import split_bytes
from simt import pipeline_price as PRICE_SIM
from simt import pipeline_split as SIM
from test_pipeline_price import _emit_split_numbers, golden

GOLDEN = Path(__file__).resolve().parent / 'golden' / 'pipeline_split.json.gz'


def split_golden():
    return json.loads(gzip.decompress(GOLDEN.read_bytes()))['tasks']


def split_designs():
    """The designs the fixture's tasks number: pipeline_price.json.gz's, then the fixture's own hand-made ones."""
    designs, _ = golden()
    for d in json.loads(gzip.decompress(GOLDEN.read_bytes()))['designs']:
        stages = []
        for st in d['stages']:
            x = {k: np.asarray(st[k], np.int64) for k in ('inp_shifts', 'out_idxs', 'out_shifts', 'out_negs')}
            x['ops_i'] = np.asarray(st['ops_i'], np.int64).reshape(-1, 4)
            x['ops_f'] = np.asarray(st['ops_f_bits'], np.uint32).view(np.float32).reshape(-1, 5)
            x.update(adder_size=st['adder_size'], carry_size=st['carry_size'], shape=(len(x['inp_shifts']), len(x['out_idxs'])))
            stages.append(x)
        designs.append(stages)
    return designs


def assert_split_equal(got, rec, tag):
    """A split (stage dicts) against a golden record: stage count, per-stage shapes, digest, and the full arrays where
    the record has them."""
    assert len(got) == rec['stages'], tag
    assert [[int(s['shape'][0]), int(s['shape'][1]), len(s['ops_i'])] for s in got] == rec['meta'], tag
    for st, full in zip(got, rec.get('full') or []):
        for k in ('inp_shifts', 'out_idxs', 'out_shifts', 'out_negs', 'ops_i'):
            assert np.asarray(st[k], np.int64).tolist() == full[k], (tag, k)
        assert np.asarray(st['ops_f'], np.float64).view(np.uint64).tolist() == full['ops_f_bits'], tag
    assert hashlib.sha256(split_bytes(got)).hexdigest() == rec['sha256'], tag


def check_splits_against_golden(run):
    """``run(designs, cutoffs, latencies, retiming)`` -> a ``PipelinePrice`` with kept splits; every task of the fixture
    is checked.  Retimed splits are compared where every input is in the first stage (the reference re-traces a split
    with its inputs at latency 0)."""
    designs = split_designs()
    tasks = split_golden()
    groups = {}
    for t in tasks:
        groups.setdefault((t['design'], json.dumps(t['latencies'])), []).append(t)
    n_checked = n_full = 0
    for (d, _), ts in groups.items():
        cuts = sorted({t['cutoff'] for t in ts})
        lats = None if ts[0]['latencies'] is None else [ts[0]['latencies']]
        for rt in (False, True):
            pr = run([designs[d]], cuts, lats, rt)
            for t in ts:
                j = cuts.index(t['cutoff'])
                tag = (t['design'], t['latencies'], t['cutoff'], rt)
                assert int(pr.status[0, j]) == t['status'], tag
                if t['status'] != 0:
                    with pytest.raises(ValueError, match='is not ok'):
                        pr.split(0, j)
                    continue
                if t['split'] is None:
                    with pytest.raises(ValueError, match='KeyError'):
                        pr.split(0, j)
                    continue
                if not rt:
                    assert_split_equal(pr.split(0, j), t['split'], tag)
                    n_full += 'full' in t['split']
                elif all(v < t['cutoff'] for v in (t['latencies'] or [0.0])):
                    assert_split_equal(pr.split(0, j), t['retimed'], tag)
                n_checked += 1
    assert n_checked > 300 and n_full > 20


@pytest.mark.parametrize('threads', [32, 128])
def test_simulated_split_equals_reference(threads):
    check_splits_against_golden(lambda ds, cuts, lats, rt: SIM.split(ds, cuts, lats, rt, threads=threads))


def test_golden_covers_the_cases():
    designs = split_designs()
    tasks = split_golden()
    ok = [t for t in tasks if t['status'] == 0]
    assert any(t['interleaved'] and t['split'] for t in ok)  # an op order that is not the (latency, position) order
    assert any(t['split'] is None for t in ok)  # the reference's KeyError
    assert any(t['split'] and t['split']['stages'] > 2 for t in ok)
    assert any(t['split'] and t['latencies'] and max(t['latencies']) >= t['cutoff'] for t in ok)  # inputs past stage 0
    assert any((np.asarray(designs[t['design']][-1]['out_idxs']) < 0).any() and t['split'] for t in ok)  # a dead column
    dead_op = [d for d, ds in enumerate(designs) if len(ds[0]['ops_i']) and ds[0]['ops_i'][-1, 2] == 0 and ds[0]['ops_i'][-1, 0] == len(ds[0]['ops_i']) - 2]
    assert any(t['design'] in dead_op and t['split'] for t in ok)  # a dead stage-0 op
    assert any(t['split'] and 'full' in t['split'] and len(t['split']['full']) > 1 for t in ok)
    # an output that is an input, at latency 0, next to late inputs nothing reads: the input kept by
    # dead_statement_elimination lands after the output stage (KeyError), or in a split of its own row
    n_base = len(golden()[0])
    late_unread = [t for t in ok if t['design'] == n_base and t['latencies'] and t['latencies'][2] == 0.0]
    assert any(t['split'] is None for t in late_unread) and any(t['split'] and t['split']['meta'][0][2] > 1 for t in late_unread)


def test_split_keeps_the_prices():
    """The status, stages, register-bit and cutoff arrays with kept splits are the pricing kernel's."""
    designs, _ = golden()
    cuts = [1.0, 2.5, 4.0, 12.0]
    for rt in (False, True):
        a = PRICE_SIM.price(designs, cuts, retiming=rt, threads=64)
        b = SIM.split(designs, cuts, retiming=rt, threads=64)
        for k in ('status', 'stages', 'reg_bits'):
            assert np.array_equal(a[k], getattr(b, k)), k
        for k in ('cutoff', 'latency_max'):
            assert np.array_equal(a[k], getattr(b, k), equal_nan=True), k
        assert b.profile['launches'] == a['launches'] + 2


@pytest.mark.parametrize('seed', range(4))
def test_simulated_split_equals_emit(seed):
    from oracle import oracle_solve

    rng = np.random.default_rng(100 + seed)
    W = rng.integers(-64, 64, size=(int(rng.integers(6, 16)), int(rng.integers(4, 14)))).astype(np.float32)
    if seed == 1:
        W[:, 0] = 0
    st, _ = oracle_solve(W, adder_size=int(rng.integers(1, 8)), carry_size=int(rng.integers(1, 4)))
    stages = [emit.as_stage(s) for s in st]
    cuts = [2.0, 3.0, 5.0, 8.0]
    for rt in (False, True):
        pr = SIM.split([stages], cuts, retiming=rt, threads=64)
        for j, c in enumerate(cuts):
            try:
                comb = emit._retrace(stages, c, B.cost_add)
            except AssertionError:
                assert pr.status[0, j] == 1
                continue
            want = emit.to_pipeline(comb, c, retiming=rt)
            got = pr.split(0, j)
            assert len(got) == len(want) == int(pr.stages[0, j]) and _emit_split_numbers(got)[1] == int(pr.reg_bits[0, j]), (seed, c, rt)
            for a, b in zip(got, want):
                assert a['shape'] == b['shape']
                for k in ('inp_shifts', 'out_idxs', 'out_shifts', 'out_negs', 'ops_i', 'ops_f'):
                    assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), (seed, c, rt, k)
                assert a['ops_f'].dtype == np.float64 and a['out_negs'].dtype == bool


def test_split_errors():
    designs, _ = golden()
    tasks = split_golden()
    t_slow = next(t for t in tasks if t['status'] == 1 and t['latencies'] is None)
    t_key = next(t for t in tasks if t['status'] == 0 and t['split'] is None)
    pr = SIM.split([designs[t_slow['design']]], [t_slow['cutoff']], retiming=False)
    with pytest.raises(ValueError, match='is not ok'):
        pr.split(0, 0)
    pr = SIM.split([designs[t_key['design']]], [t_key['cutoff']], [t_key['latencies']], retiming=True)
    with pytest.raises(ValueError, match="to_pipeline raises KeyError"):
        pr.split(0, 0)
    ok = next(t for t in tasks if t['status'] == 0 and t['split'] and t['latencies'] is None)
    pr = SIM.split([designs[ok['design']]], [ok['cutoff']], retiming=False)
    s1 = pr.split(0, 0)
    s1[0]['ops_i'][:] = -7  # (a fresh copy every call)
    assert_split_equal(pr.split(0, 0), ok['split'], 'copy')
    no = B.PipelinePrice(pr.status, pr.stages, pr.reg_bits, pr.latency_max, pr.cutoff, pr.cutoffs, [None], {})
    with pytest.raises(ValueError, match='was not kept'):
        no.split(0, 0)
    sc = pr._scatter([1], 3)  # (SweepResult.pipelined: rows of candidates that were not priced)
    assert_split_equal(sc.split(1, 0), ok['split'], 'scatter')
    with pytest.raises(ValueError, match='was not kept'):
        sc.split(0, 0)


def _design(n_in=3):
    rng = np.random.default_rng(0)
    from oracle import oracle_solve

    return [emit.as_stage(s) for s in oracle_solve(rng.integers(-8, 8, size=(n_in, 3)).astype(np.float32))[0]]


def test_argument_errors():
    d = _design()
    with pytest.raises(ValueError, match='cutoff 0 is'):
        B.price_pipelined([d], 0.0, keep_split=True)
    with pytest.raises(ValueError, match='expected 3 latencies'):
        B.price_pipelined([d], 2.0, latencies=[[0.0, 1.0]], keep_split=True)
    bad = [dict(s) for s in d]
    bad[0]['ops_i'] = bad[0]['ops_i'].copy()
    bad[0]['ops_i'][-1, 0] = len(bad[0]['ops_i'])
    with pytest.raises(ValueError, match='not an adder-graph op'):
        B.price_pipelined([bad], 2.0, keep_split=True)
    with pytest.raises(ValueError, match='input latency 1 is not'):
        B.price_pipelined([d], 2.0, latencies=[[0.0, -1.0, 0.0]], keep_split=True)
    q = np.zeros(4, np.int64)
    with pytest.raises(ValueError, match='split_info: the handle or the output array is null'):
        B._check(B._L.da4ml_split_info(None, 0, q.ctypes.data_as(B._i64p)))
    with pytest.raises(ValueError, match='split_copy: the handle is null'):
        B._check(B._L.da4ml_split_copy(None, 0, *[None] * 6))
    with pytest.raises(ValueError, match='handle pointer is null'):
        B._check(B._L.da4ml_pipeline_split(1, *[None] * 10, 1, 0, *[None] * 7, None))


def test_no_device_error():
    if B.device_info()['cuda_devices'] > 0:
        pytest.skip('a CUDA device is present')
    with pytest.raises(RuntimeError, match='no CUDA device'):
        B.price_pipelined([_design()], 2.0, keep_split=True)


def test_sweep_pipelined_passes_keep_split():
    seen = []

    def pricer(designs, c, latencies=None, retiming=True, **kw):
        seen.append(kw)
        return SIM.split(designs, c, latencies, retiming)

    class Sweep:  # the two attributes SweepResult.pipelined reads, around one design
        candidates = dict(kept=np.asarray([False, True]))
        _call = dict(latencies=None)

        def __len__(self):
            return 2

        def raw(self, i):
            return B.RawPipeline.from_stages(_design())

    pr = B.SweepResult.pipelined(Sweep(), [3.0], pricer=pricer, keep_split=True)
    assert seen == [dict(keep_split=True)]
    assert len(pr.split(1, 0)) == int(pr.stages[1, 0])
    with pytest.raises(ValueError, match='was not kept'):
        pr.split(0, 0)
    B.SweepResult.pipelined(Sweep(), [3.0], pricer=pricer)
    assert seen[-1] == {}
