"""The page pool of the histogram segment (solve_histogram.cuh hot_grow / hot_free, the page lists of solve_common.cuh),
run by the simulated kernels of tests/simt and compared with the oracle.  A CTA's segment is a pool of pages: the common
log fills it from the bottom, the hot logs (one per early owned expression) take single pages from the top, and a
rewritten hot expression returns its pages to a free stack, from which the next pages are taken."""
import numpy as np
import pytest
from conftest import assert_stage_equal, int_matrix

import simt
from oracle import port


@pytest.mark.parametrize('ctas,threads,schedule', [(2, 64, 0), (1, 32, 0), (3, 128, 2)])
def test_hot_pages_are_freed_and_reused(ctas, threads, schedule):
    """22 x 20 int8 over 184 greedy steps: the inputs a CTA owns get hot logs, each log keeps a page of room ahead, and
    every rewrite of a hot input sends all but its first page back to the free stack, to be handed to the next log that
    fills up -- many times per solve.  Accounting mode re-reads every page in use every step and counts the live entries:
    a freed page still listed as in use, or a reused page read past its new fill, would change the reference's work
    counters; a page handed to two logs would change the graph."""
    W = int_matrix(22, 20, 8, 21)
    want = port.solve_single(W, 'wmc')
    cnt = port.partial(W, 'wmc')
    simt.set_schedule(schedule)
    try:
        got, meta = simt.solve_single(W, 'wmc', ctas=ctas, cta_threads=threads, accounting=True)
        plain, _ = simt.solve_single(W, 'wmc', ctas=ctas, cta_threads=threads)
    finally:
        simt.set_schedule(0)
    assert_stage_equal(got, want, f'{ctas}x{threads} accounting ')
    assert_stage_equal(plain, want, f'{ctas}x{threads} ')
    assert (meta[2], meta[3], meta[4], meta[5], meta[6]) == (cnt['iters'], cnt['sum_F'], cnt['sum_R'], cnt['F0'], cnt['R0'])


def test_pool_that_runs_out_is_retried_larger_with_the_same_result():
    """A pool of 4000 entries per CTA runs out (capacity status 2, which the host driver answers with a retry at four
    times the capacity); the retry compacts along the way and gives the reference graph, as does the planner's pool."""
    W = int_matrix(22, 20, 8, 21)
    want = port.solve_single(W, 'wmc')
    try:
        simt.set_segment_cap(4000)
        with pytest.raises(RuntimeError, match='capacity status 2'):
            simt.solve_single(W, 'wmc', ctas=2, cta_threads=64)
        simt.set_segment_cap(16000)
        got, meta = simt.solve_single(W, 'wmc', ctas=2, cta_threads=64)
        assert meta[9] >= 1  # compacted
        assert_stage_equal(got, want, 'retried ')
    finally:
        simt.set_segment_cap(0)
    got, meta = simt.solve_single(W, 'wmc', ctas=2, cta_threads=64)
    assert_stage_equal(got, want, 'planner pool ')
    assert meta[9] == 0
