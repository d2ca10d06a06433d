"""Pipelined pricing (``price_pipelined``) without a GPU: the kernel source under the SIMT shim against the reference tracer's
answers (tests/golden/pipeline_price.json.gz), the retiming bisection against ``emit.retime_pipeline``, argument checks,
and ``chain_front(latency_cutoff=c)`` with stand-in solver and pricer against brute force."""
import gzip
import itertools
import json
from pathlib import Path

import numpy as np
import pytest

import da4ml_b200._binary as B
from da4ml_b200 import emit
from da4ml_b200.types import minimal_kif_array

from simt import pipeline_price as SIM

GOLDEN = Path(__file__).resolve().parent / 'golden' / 'pipeline_price.json.gz'


def golden():
    g = json.loads(gzip.decompress(GOLDEN.read_bytes()))
    designs = []
    for d in g['designs']:
        stages = []
        for st in d['stages']:
            s = {k: np.asarray(st[k], np.int64) for k in ('inp_shifts', 'out_idxs', 'out_shifts', 'out_negs')}
            s['ops_i'] = np.asarray(st['ops_i'], np.int64).reshape(-1, 4)
            s['ops_f'] = np.asarray(st['ops_f_bits'], np.uint32).view(np.float32).reshape(-1, 5)
            s.update(adder_size=st['adder_size'], carry_size=st['carry_size'], shape=(len(s['inp_shifts']), len(s['out_idxs'])))
            stages.append(s)
        designs.append(stages)
    return designs, g['tasks']


def check_against_golden(price):
    """``price(designs, cutoffs, latencies, retiming)`` -> dict / PipelinePrice-like answers, checked task by task."""
    designs, tasks = golden()
    groups = {}
    for t in tasks:
        groups.setdefault((t['design'], json.dumps(t['latencies'])), []).append(t)
    # one call per latency set: every design under every cutoff of its tasks
    by_lat = {}
    for (d, lk), ts in groups.items():
        by_lat.setdefault(lk, []).append((d, ts))
    n_checked = 0
    for lk, items in by_lat.items():
        cuts = sorted({t['cutoff'] for _, ts in items for t in ts})
        ds = [designs[d] for d, _ in items]
        lats = None if json.loads(lk) is None else [json.loads(lk)] * len(ds)
        if lats is not None:  # (a latency set belongs to one design: its length is the design's input count)
            for (d, ts), dd in zip(items, ds):
                r = price([dd], cuts, [ts[0]['latencies']], False)
                r2 = price([dd], cuts, [ts[0]['latencies']], True)
                n_checked += _check_tasks(ts, cuts, r, r2, 0)
            continue
        r = price(ds, cuts, None, False)
        r2 = price(ds, cuts, None, True)
        for k, (d, ts) in enumerate(items):
            n_checked += _check_tasks(ts, cuts, r, r2, k)
    assert n_checked == len(tasks)


def _get(r, key):
    return r[key] if isinstance(r, dict) else getattr(r, key)


def _olat(r, k, j):
    return _get(r, 'out_latency')[k][j] if isinstance(r, dict) else r.out_latency(k, j)


def _check_tasks(ts, cuts, r, r2, k):
    for t in ts:
        j = cuts.index(t['cutoff'])
        tag = (t['design'], t['latencies'], t['cutoff'])
        assert int(_get(r, 'status')[k, j]) == t['status'], tag
        assert int(_get(r2, 'status')[k, j]) == t['status'], tag
        if t['status'] != 0:
            assert int(_get(r, 'stages')[k, j]) == -1 and np.isnan(_get(r, 'latency_max')[k, j])
            continue
        assert list(_olat(r, k, j)) == t['out_latency'], tag
        assert float(_get(r, 'latency_max')[k, j]) == max(t['out_latency']), tag
        assert float(_get(r, 'cutoff')[k, j]) == t['cutoff']
        if t['split'] is None:  # (the reference's splitter fails on a design whose first stage would be empty)
            continue
        assert (int(_get(r, 'stages')[k, j]), int(_get(r, 'reg_bits')[k, j])) == (t['split']['stages'], t['split']['reg_bits']), tag
        if all(v < t['cutoff'] for v in (t['latencies'] or [0.0])):  # (every input in the first stage: the re-trace the reference does)
            got = (int(_get(r2, 'stages')[k, j]), int(_get(r2, 'reg_bits')[k, j]), float(_get(r2, 'cutoff')[k, j]))
            assert got == (t['retimed']['stages'], t['retimed']['reg_bits'], t['retimed']['cutoff']), tag
    return len(ts)


@pytest.mark.parametrize('threads', [32, 128])
def test_simulated_kernel_equals_reference_tracer(threads):
    check_against_golden(lambda ds, cuts, lats, rt: SIM.price(ds, cuts, lats, rt, threads=threads))


def test_golden_covers_the_cases():
    designs, tasks = golden()
    st = np.bincount([t['status'] for t in tasks], minlength=3)
    assert st[0] > 100 and st[1] > 50  # ok tasks and tasks with an adder slower than the cutoff
    assert any(t['latencies'] is not None and len(set(t['latencies'])) > 1 and t['status'] == 0 for t in tasks)
    assert any(len(d) == 1 for d in designs) and any(len(d) == 2 for d in designs)
    assert any((np.asarray(d[-1]['out_idxs']) < 0).any() for d in designs)  # an all-zero column
    ok = [t for t in tasks if t['status'] == 0 and t['split']]
    assert any(t['retimed']['cutoff'] != t['cutoff'] for t in ok) and any(t['split']['stages'] > 2 for t in ok)


def _emit_split_numbers(split):
    qi, _ = emit._qint_io(split[0])
    bits = int(minimal_kif_array(qi).sum()) + sum(int(minimal_kif_array(emit._qint_io(s)[1]).sum()) for s in split)
    return len(split), bits


@pytest.mark.parametrize('seed', range(6))
def test_bisection_equals_emit_retime(seed):
    from oracle import oracle_solve

    rng = np.random.default_rng(seed)
    W = rng.integers(-64, 64, size=(int(rng.integers(6, 16)), int(rng.integers(4, 14)))).astype(np.float32)
    st, _ = oracle_solve(W, adder_size=int(rng.integers(1, 8)), carry_size=int(rng.integers(1, 4)))
    stages = [emit.as_stage(s) for s in st]
    cuts = [3.0, 6.0, 10.0, 25.0]
    r = SIM.price([stages], cuts, retiming=True, threads=64)
    for j, c in enumerate(cuts):
        try:
            comb = emit._retrace(stages, c, B.cost_add)
        except AssertionError:
            assert r['status'][0, j] == 1
            continue
        split = emit.to_pipeline(comb, c, retiming=True)
        assert (int(r['stages'][0, j]), int(r['reg_bits'][0, j])) == _emit_split_numbers(split), (seed, c)


def _design(n_in=3):
    rng = np.random.default_rng(0)
    from oracle import oracle_solve

    return [emit.as_stage(s) for s in oracle_solve(rng.integers(-8, 8, size=(n_in, 3)).astype(np.float32))[0]]


def test_argument_errors():
    d = _design()
    with pytest.raises(ValueError, match='cutoff 0 is'):
        B.price_pipelined([d], 0.0)
    with pytest.raises(ValueError, match='positive'):
        B.price_pipelined([d], [2.0, -1.0])
    with pytest.raises(ValueError, match='at least one design'):
        B.price_pipelined([], 2.0)
    with pytest.raises(ValueError, match='expected 3 latencies'):
        B.price_pipelined([d], 2.0, latencies=[[0.0, 1.0]])
    bad = [dict(s) for s in d]
    bad[0]['ops_i'] = bad[0]['ops_i'].copy()
    bad[0]['ops_i'][-1, 2] = 5  # a constant op: not a solver result
    with pytest.raises(ValueError, match='opcode 5'):
        B.price_pipelined([bad], 2.0)
    bad[0]['ops_i'][-1, 2] = 0
    bad[0]['ops_i'][-1, 0] = len(bad[0]['ops_i'])  # an operand that is not an earlier op
    with pytest.raises(ValueError, match='not an adder-graph op'):
        B.price_pipelined([bad], 2.0)
    with pytest.raises(ValueError, match='opcode 7'):
        bad[0]['ops_i'][-1, 2] = 7
        B.price_pipelined([bad], 2.0)


def test_no_device_error():
    if B.device_info()['cuda_devices'] > 0:
        pytest.skip('a CUDA device is present')
    with pytest.raises(RuntimeError, match='no CUDA device'):
        B.price_pipelined([_design()], 2.0)


# ---- chain_front with a latency cutoff, on stand-ins ------------------------------------------------------------------


class FakeSweep:
    """A sweep of hand-made candidates: each is a one-stage design whose graph depends on the input latencies it was
    'solved' under, so that the pricer's traced latencies matter."""

    def __init__(self, designs, cost, lats):
        self._designs, self._lats = designs, lats
        n = len(designs)
        self.candidates = dict(cost=np.asarray(cost, np.float32), latency_max=np.zeros(n, np.float32), kept=np.ones(n, bool), set=np.zeros(n, np.int64),
                               hard_dc=np.full(n, -1), decompose_dc_start=np.full(n, -2))  # fmt: skip
        self.front = np.arange(n)
        self.option_sets = [{}]
        self.profile = dict(launches=1, device_ms=0.0, jobs_run=n, jobs_total=n)

    def raw(self, i):
        return B.RawPipeline.from_stages(self._designs[i])

    def reference_call(self, i):
        return dict(method0='wmc', method1='auto', hard_dc=-1, decompose_dc=-2, search_all_decompose_dc=False, qintervals=None, latencies=self._lats, adder_size=2,
                    carry_size=2, cand=int(i))  # fmt: skip


def _chain_solver(seed):
    from oracle import oracle_solve

    def solver(kernels, option_sets, qintervals=None, latencies=None, adder_size=-1, carry_size=-1):
        out = []
        for W, l in zip(kernels, latencies):
            h = int(abs(hash((seed, tuple(np.asarray(l).round(6)))) % 1000))
            rng = np.random.default_rng(h)
            ds, cs = [], []
            for k in range(3):
                Wk = (W * rng.choice([1, 1, 3], size=W.shape)).astype(np.float32)
                ds.append([emit.as_stage(s) for s in oracle_solve(Wk, latencies=list(l))[0]][:1])
                cs.append(float(rng.integers(5, 40)))
            out.append(FakeSweep(ds, cs, list(l)))
        return out

    return solver


def _tracer_pricer(calls):
    """price_pipelined restated by emit's re-trace (the tracer's rule), for the CPU: latencies and stage count only."""

    def pricer(designs, latency_cutoff, latencies=None, retiming=True):
        assert not retiming
        calls.append(len(designs))
        c = float(latency_cutoff)
        st, lm, ol = [], [], []
        for d, l in zip(designs, latencies):
            stages = emit._stages_of(d)
            try:
                comb = _retrace_at(stages, c, l)
            except AssertionError:
                st.append(1), lm.append(np.nan), ol.append(None)
                continue
            o = np.asarray([float(comb['ops_f'][i, 3]) if i >= 0 else 0.0 for i in comb['out_idxs']])
            st.append(0), lm.append(o.max()), ol.append(o[None, :])
        n = len(designs)
        return B.PipelinePrice(np.asarray(st, np.int32)[:, None], np.full((n, 1), -1), np.full((n, 1), -1), np.asarray(lm)[:, None], np.full((n, 1), c), np.asarray([c]), ol,
                               dict(device_ms=0.0, launches=1))  # fmt: skip

    return pricer


def _retrace_at(stages, c, lats):
    """emit._retrace with the inputs at ``lats`` instead of 0."""
    orig = emit._Node.__init__

    def init(self, uid, frm, latency, cost, inp=-1):
        orig(self, uid, frm, float(lats[inp]) if inp >= 0 and not frm else latency, cost, inp)

    emit._Node.__init__ = init
    try:
        return emit._retrace(stages, c, B.cost_add)
    finally:
        emit._Node.__init__ = orig


def _brute(kernels, solver, pricer, c):
    """Every chain of candidates, each layer solved under the traced output latencies of the design before it."""
    pts = []

    def rec(k, lats, cost, choice):
        if k == len(kernels):
            pts.append((cost, lats.max(), tuple(choice)))
            return
        sw = solver([kernels[k]], [{}], latencies=[list(map(float, lats))])[0]
        for i in sw.front:
            r = pricer([sw.raw(int(i))], c, latencies=[list(map(float, lats))], retiming=False)
            if r.status[0, 0] != 0:
                continue
            rec(k + 1, r.out_latency(0, 0), np.float32(cost + sw.candidates['cost'][i]), choice + [int(i)])

    rec(0, np.zeros(kernels[0].shape[0]), np.float32(0), [])
    cost = np.asarray([p[0] for p in pts], np.float32)
    lat = np.asarray([p[1] for p in pts])
    keep = B.sweep_front(cost, lat.astype(np.float32))
    return {(float(cost[i]), float(lat[i])) for i in keep}


@pytest.mark.parametrize('seed', range(4))
@pytest.mark.parametrize('c', [3.0, 5.0])
def test_chain_front_cutoff_against_brute_force(seed, c):
    rng = np.random.default_rng(seed)
    kernels = [rng.integers(-6, 6, size=(4, 4)).astype(np.float32) for _ in range(3)]
    calls = []
    front = B.chain_front(kernels, [{}], latency_cutoff=c, solver=_chain_solver(seed), pricer=_tracer_pricer(calls))
    assert len(calls) == 3  # one pricer call per layer
    got = {(float(a), float(b)) for a, b in zip(front.cost, front.latency)}
    want = _brute(kernels, _chain_solver(seed), _tracer_pricer([]), c)
    assert got <= want and min(want) in got  # every point is exact; the cheapest chain survives the pruning
    assert np.array_equal(front.stages, np.floor(front.latency.astype(np.float64) / (c + 1e-9)).astype(np.int64) + 1)
    for n in sorted(set(front.stages.tolist())):
        p = front.best_stages(n)
        ok = front.stages <= n
        assert p.cost == float(front.cost[ok].min())
    for p in range(len(front)):  # the reference calls carry the traced latencies of the design before
        calls_p = front.reference_calls(p)
        lats = [0.0] * 4
        for k, call in enumerate(calls_p):
            assert call['latencies'] == [float(v) for v in lats]
            r = _tracer_pricer([])([front.raw(p, k)], c, latencies=[lats], retiming=False)
            lats = [float(v) for v in r.out_latency(0, 0)]
        assert max(lats) == float(front.latency[p])


def test_chain_front_cutoff_zero_is_unchanged():
    rng = np.random.default_rng(3)
    kernels = [rng.integers(-6, 6, size=(4, 4)).astype(np.float32) for _ in range(3)]
    a = B.chain_front(kernels, [{}], solver=_chain_solver(1))
    b = B.chain_front(kernels, [{}], latency_cutoff=0.0, solver=_chain_solver(1), pricer=lambda *x, **k: pytest.fail('no pricing at cutoff 0'))
    assert np.array_equal(a.cost, b.cost) and np.array_equal(a.latency, b.latency) and np.array_equal(a.choice, b.choice)
    assert a.latency.dtype == b.latency.dtype == np.float32
    assert [a.reference_calls(p) for p in range(len(a))] == [b.reference_calls(p) for p in range(len(b))]
    assert list(itertools.chain(*[[r['states'], r['points']] for r in a.profile['layers']])) == list(itertools.chain(*[[r['states'], r['points']] for r in b.profile['layers']]))
