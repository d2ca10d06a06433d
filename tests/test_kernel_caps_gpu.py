"""The solve kernel's capacity paths on the device: owner-list rows spilled to global memory, pair counting in several
passes of a small hash table, 12-byte list rows, histogram-segment compaction, the capacity statuses and the host's retry
with larger capacities.  The planner sizes the full-size problems of the rest of the suite so that none of these paths
runs; ``capacity_override`` squeezes the capacities so that they do, and every result must still be the checker's graph
bit for bit.  Each forced path also checks a counter that shows it ran, so that a squeeze that stops biting fails."""
import contextlib

import numpy as np
import pytest
from conftest import assert_stage_equal, golden_cases, int_matrix, load_golden
from test_cmvm_gpu import digest

from oracle import port

ALL = golden_cases(full_only=False)
SOLVE_CASES = sorted(k for k, v in ALL.items() if v['full'] and not v.get('single'))


@pytest.fixture
def B(cuda_binary):
    yield cuda_binary
    cuda_binary.set_group_size(0)
    cuda_binary.set_accounting(False)


@contextlib.contextmanager
def group_size(B, G):
    B.set_group_size(G)
    try:
        yield
    finally:
        B.set_group_size(0)


def hetero(n_in, seed):
    rng = np.random.default_rng(seed)
    q = [(-float(2 ** rng.integers(2, 8)), float(2 ** rng.integers(2, 8)) - 1.0, 1.0) for _ in range(n_in)]
    return q, [float(v) for v in rng.integers(0, 4, n_in)]


# single stages: (shape, method, non-trivial intervals and latencies)
LAYOUT_CASES = [((48, 40), 'wmc', False), ((48, 40), 'wmc-dc', False), ((48, 40), 'mc', True),
                ((64, 64), 'wmc', False), ((64, 64), 'wmc-dc', False), ((64, 64), 'mc', True)]  # fmt: skip
LAYOUTS = [dict(list_rows=0), dict(list_rows=4), dict(wide_rows=True), dict(hash_log=8), dict(hash_log=9)]


def single_case(shape, method, hetero_q):
    W = int_matrix(*shape, 8, shape[0] * 100 + shape[1])
    kw = dict(zip(('qintervals', 'latencies'), hetero(shape[0], 5))) if hetero_q else {}
    return W, kw


def solve_single(B, W, method, **kw):
    raw, _ = B.solve_single_raw(W, method, kw.get('qintervals'), kw.get('latencies'))
    return raw


def test_override_arguments_are_checked():
    """Checked on the host before anything is set (no device needed)."""
    import da4ml_b200._binary as B

    with pytest.raises(TypeError, match='unknown capacity knobs'):
        with B.capacity_override(rows=3):
            pass
    for bad in (dict(hash_log=7), dict(hash_log=14), dict(segment_entries=0), dict(expr_cap=0), dict(cell_pool=0)):
        with pytest.raises(ValueError, match='capacity override'):
            with B.capacity_override(**bad):
                pass


@pytest.mark.gpu
def test_natural_spills_at_full_size_one_cta(B):
    """With one CTA per problem and no squeeze, the shared memory cannot hold every row of the 128x128 int8 matrix's
    longest column list: the list spills to global memory, and the graph is still the pinned one.  (The int6 matrices
    of the same shape have fewer digits and do not spill.)"""
    meta = ALL['128x128_int8_dc-1']
    W = int_matrix(*meta['spec'][1:])
    with group_size(B, 1):
        raw = B.solve_raw(W, **meta['kwargs'])
    c = raw.counters[0]
    assert c['group_ctas'] == 1
    assert c['list_max'] > c['smem_list_cap'], (c['list_max'], c['smem_list_cap'])
    assert raw.profile['solve_retries'] == 0
    assert digest(raw.stages) == meta['sha256']


@pytest.mark.gpu
@pytest.mark.parametrize('shape,method,hetero_q', LAYOUT_CASES)
def test_forced_list_layouts(B, shape, method, hetero_q):
    """Owner lists entirely / beyond the fourth row in global memory, 12-byte rows, and pair-counter tables of 256 and
    512 slots (many counting passes per step), at group sizes 1, 2, 7 and the planner's."""
    W, kw = single_case(shape, method, hetero_q)
    want = port.solve_single(W, method, **kw)
    for G in (1, 2, 7, 0):
        with group_size(B, G):
            for caps in LAYOUTS:
                tag = f'{shape} {method} G={G} {caps} '
                with B.capacity_override(**caps):
                    raw = solve_single(B, W, method, **kw)
                c = raw.counters[0]
                assert_stage_equal(raw.stages[0], want, tag)
                assert raw.profile['solve_retries'] == 0, tag
                if 'list_rows' in caps:
                    assert c['smem_list_cap'] == caps['list_rows'], tag
                    assert c['list_max'] > c['smem_list_cap'], tag
                if G:
                    assert c['group_ctas'] == G, tag
    # the planner's tables are larger than the squeezed ones
    c = raw.counters[0]
    p = B.plan([dict(n_in=shape[0], n_out=shape[1], nbits=c['n_bits'], digits=c['D0'])], group_override=1)
    assert p['log2_pair_counters'] >= 11 and p['narrow_rows'] == 1


@pytest.mark.gpu
def test_small_hash_table_counts_the_reference_work(B):
    """Counting in many passes of a 256-slot table, in accounting mode: the work counters are the reference's."""
    W = int_matrix(48, 40, 8, 4840)
    want, cnt = port.solve_single(W, 'wmc'), port.partial(W, 'wmc')
    B.set_accounting(True)
    for G in (1, 2, 0):
        with group_size(B, G), B.capacity_override(hash_log=8):
            raw = solve_single(B, W, 'wmc')
        c = raw.counters[0]
        assert_stage_equal(raw.stages[0], want, f'G={G} ')
        assert (c['T'], c['sum_F'], c['sum_R'], c['F0'], c['R0']) == (cnt['iters'], cnt['sum_F'], cnt['sum_R'], cnt['F0'], cnt['R0']), G


@pytest.mark.gpu
@pytest.mark.parametrize('G', [2, 0])
def test_segment_compaction_and_overflow_retries(B, G):
    """Histogram segments from the planner's size down to a few pages: a segment that only compacts, one that overflows
    once (ST_FSEG_OVERFLOW, relaunched with 4x the segment) and one that overflows twice all give the checker's graph."""
    W = int_matrix(48, 40, 8, 4840)
    want = port.solve_single(W, 'wmc')
    seen = {}
    for k in range(40, 14, -1):  # 2^20 ... 2^7.5 entries, in steps of sqrt(2)
        cap = int(2 ** (k / 2))
        with group_size(B, G), B.capacity_override(segment_entries=cap):
            raw = solve_single(B, W, 'wmc')
        c, r = raw.counters[0], raw.profile['solve_retries']
        assert_stage_equal(raw.stages[0], want, f'segment {cap} ')
        assert raw.profile['solve_kernel_launches'] == 1 + r
        key = 'compacted' if r == 0 and c['compactions'] >= 1 else r
        seen.setdefault(key, cap)
        if r >= 3:
            break
    assert {'compacted', 1, 2} <= set(seen), seen


@pytest.mark.gpu
@pytest.mark.parametrize('caps,exact', [(dict(list_rows=4, spill_rows=16), None), (dict(cell_pool=1024), None), (dict(expr_cap=16), 1)])
def test_list_pool_and_expression_overflow_retries(B, caps, exact):
    """Owner lists with no room to spill, a small cell pool, a small expression table: the kernel reports the status,
    the host relaunches the job with the larger capacity, and the graph is the checker's.  (At the planner's group size
    each CTA owns one or two inputs, and these caps do not bite.)"""
    for shape, method, hetero_q in LAYOUT_CASES[:3]:
        W, kw = single_case(shape, method, hetero_q)
        want = port.solve_single(W, method, **kw)
        for G in (1, 2):
            with group_size(B, G), B.capacity_override(**caps):
                raw = solve_single(B, W, method, **kw)
            r = raw.profile['solve_retries']
            assert_stage_equal(raw.stages[0], want, f'{caps} {method} G={G} ')
            assert r == exact if exact else r >= 1, (caps, method, G, r)
            assert raw.profile['solve_kernel_launches'] == 1 + r


SQUEEZE = dict(list_rows=4, hash_log=9, segment_entries=4096)


@pytest.mark.gpu
def test_mixed_rounds(B):
    """A batch in which one job overflows and the others finish: only that job is relaunched, and every result is its
    own solve.  A sweep and a 3-layer chain under the squeeze are the un-squeezed calls."""
    kw = dict(decompose_dc=-1, search_all_decompose_dc=False)
    mats = [int_matrix(48, 40, 8, 11), int_matrix(8, 8, 4, 12), int_matrix(10, 12, 5, 13), int_matrix(6, 9, 6, 14)]
    plain = [B.solve_raw(W, **kw) for W in mats]
    with B.capacity_override(expr_cap=60):
        got = B.solve_batch_raw(mats, **kw)
    assert got[0].profile['solve_retries'] == 1  # (the jobs relaunched: only the 48x40 stage)
    for i, (a, b) in enumerate(zip(got, plain)):
        assert digest(a.stages) == digest(b.stages), i

    from test_chain_gpu import SETS, chain3
    from test_sweep_batch_gpu import assert_same_sweep

    W = int_matrix(24, 20, 7, 33)
    want = B.solve_sweep(W, SETS, keep_all=True)
    with B.capacity_override(**SQUEEZE):
        sw = B.solve_sweep(W, SETS, keep_all=True)
    assert_same_sweep(sw, want, 'squeezed sweep ')
    Ws, qs, l0 = chain3()
    want = B.chain_front(Ws, SETS, qintervals=qs, latencies=l0)
    with B.capacity_override(**SQUEEZE):
        cf = B.chain_front(Ws, SETS, qintervals=qs, latencies=l0)
    assert np.array_equal(cf.choice, want.choice) and np.array_equal(cf.cost, want.cost) and np.array_equal(cf.latency, want.latency)
    for p in range(len(cf)):
        for k in range(len(Ws)):
            assert digest(cf.raw(p, k).stages) == digest(want.raw(p, k).stages), (p, k)


@pytest.mark.gpu
def test_poisoned_buffers(B):
    """Every buffer the driver does not clear holds 0xA5 before the launch: a batch, and a single solve whose lists
    spill, are the plain runs."""
    mats = [int_matrix(14, 11, 6, 3), np.zeros((4, 5), np.float32), int_matrix(6, 40, 5, 31), int_matrix(48, 40, 8, 4840)]
    plain = B.solve_batch_raw(mats)
    W, kw = single_case((64, 64), 'wmc-dc', False)
    want = solve_single(B, W, 'wmc-dc')
    with B.capacity_override(poison=True):
        got = B.solve_batch_raw(mats)
    with group_size(B, 2), B.capacity_override(poison=True, list_rows=2):
        single = solve_single(B, W, 'wmc-dc')
    for i, (a, b) in enumerate(zip(got, plain)):
        assert digest(a.stages) == digest(b.stages), i
    assert single.counters[0]['list_max'] > single.counters[0]['smem_list_cap'] == 2
    assert digest(single.stages) == digest(want.stages)


@pytest.mark.gpu
def test_seeded_solves_under_a_squeeze(B):
    import seeded

    W = int_matrix(48, 40, 8, 4840)
    for seed, method in ((3, 'wmc'), (11, 'wmc-dc')):
        with group_size(B, 2), B.capacity_override(hash_log=8, segment_entries=256):
            raw, _ = B.solve_single_raw(W, method, seed=seed)
        assert raw.profile['solve_retries'] >= 1, seed
        assert_stage_equal(raw.stages[0], seeded.solve_single(W, method, seed=seed), f'seed {seed} ')


@pytest.mark.gpu
def test_goldens_under_a_combined_squeeze(B):
    """The pinned full solves and the cheapest large digests, with 4 shared rows per owner list, a 512-slot pair
    table and a histogram segment that has to be regrown."""
    for name in SOLVE_CASES:
        extra, stages = load_golden(name)
        with B.capacity_override(**SQUEEZE):
            raw = B.solve_raw(extra['kernel'], **ALL[name]['kwargs'])
        for i, (a, b) in enumerate(zip(raw.stages, stages, strict=True)):
            assert_stage_equal(a, b, f'{name} stage{i} ')
    for name in ('c2_64x64_int8_dc-1', 'c2_64x64_int8_default'):
        meta = ALL[name]
        W = int_matrix(*meta['spec'][1:])
        with B.capacity_override(**SQUEEZE):
            raw = B.solve_raw(W, **meta['kwargs'])
        assert raw.profile['solve_retries'] >= 1, name
        assert max(c['list_max'] - c['smem_list_cap'] for c in raw.counters) > 0, name
        assert digest(raw.stages) == meta['sha256'], name
