"""Launch planner of the persistent solve kernel (da4ml_b200/csrc/host_plan.cuh) through ``da4ml_cmvm_plan``.
Pure host arithmetic: runs without a GPU."""
import numpy as np
import pytest

from da4ml_b200 import _binary as B


def job(n_in, n_out, nbits, density=0.36, **kw):
    """Shape of a uniform random intN matrix: about 0.36 * nbits CSD digits per element."""
    digits = int(n_in * n_out * nbits * density)
    return dict(n_in=n_in, n_out=n_out, nbits=nbits, digits=digits, **kw)


def check_invariants(p, jobs, coop):
    G, groups = p['ctas_per_problem'], p['concurrent_groups']
    assert 1 <= G <= coop and 1 <= groups <= len(jobs)
    assert G * groups <= coop  # the cooperative launch must be co-resident
    assert p['columns_per_cta'] * G >= max(j['n_out'] for j in jobs)
    assert p['shared_bytes'] <= p['shared_budget']
    assert (p['segment_entries_per_cta'] >> p['log2_chunk']) + 2 == p['chunk_slots']
    assert 11 <= p['log2_pair_counters'] <= 13
    assert p['list_rows_smem'] % 2 == 0  # the 32-bit plane arrays of 6-byte rows stay aligned
    assert p['list_rows_smem'] + p['spill_rows'] >= 1


def test_lone_problem_gets_the_whole_gpu():
    p = B.plan([job(256, 256, 8)])
    check_invariants(p, [job(256, 256, 8)], 132)
    assert p['ctas_per_problem'] == 132 and p['concurrent_groups'] == 1
    assert p['columns_per_cta'] == 2 and p['list_rows_smem'] > 0 and p['narrow_rows'] == 1
    tiny = B.plan([job(8, 8, 4)])
    assert tiny['ctas_per_problem'] == 1  # 100 digits cannot keep more than one CTA busy
    wide = B.plan([job(16, 16, 20)])
    assert wide['narrow_rows'] == 0  # 20-bit planes need three words per row


def test_candidates_of_one_call_share_the_gpu_in_one_wave():
    jobs = [job(256, 256, 8) for _ in range(10)]  # the ten decompose_dc candidates of the bench workload (before identical ones are shared)
    p = B.plan(jobs)
    check_invariants(p, jobs, 132)
    assert p['ctas_per_problem'] == 13 and p['concurrent_groups'] == 10
    assert p['list_rows_smem'] >= 20 + 10 + 8 and p['log2_pair_counters'] == 13  # an owner's share of a column with slack, next to the large table
    six = B.plan(jobs[:6])
    assert six['ctas_per_problem'] == 22 and six['concurrent_groups'] == 6


def test_more_jobs_than_groups_run_in_equal_waves():
    jobs = [job(128, 128, 6) for _ in range(64)]
    p = B.plan(jobs)
    check_invariants(p, jobs, 132)
    G, groups = p['ctas_per_problem'], p['concurrent_groups']
    waves = -(-len(jobs) // groups)
    assert waves * groups < len(jobs) + groups  # no nearly-empty last wave
    assert p['list_rows_smem'] >= (128 // G) * 3 // 2 and p['log2_pair_counters'] >= 12  # lists fit next to >= 4096 counters


def test_several_waves_pick_the_group_size_that_wastes_least_of_the_last_wave():
    # BASELINE config 4 on one H100 (132 SMs): 64 matrices x 6 distinct stage-0 jobs.  2 CTAs per job are 6 waves on 66
    # groups (0.970 of the CTA-time busy), no larger group does better (3: 9 waves on 44 groups, 0.970; 7: 22 waves on 18
    # groups, 0.926), and ties go to the smaller group; a job's time is ~ 1 / G in this range.
    jobs = [job(128, 128, 6) for _ in range(384)]
    p = B.plan(jobs)
    check_invariants(p, jobs, 132)
    G, groups = p['ctas_per_problem'], p['concurrent_groups']
    assert (G, groups) == (2, 66)
    waves = -(-len(jobs) // groups)
    assert len(jobs) * G / (waves * 132) > 0.95
    # ... with 148 co-resident CTAs 2 CTAs per job would be 6 waves on 74 groups (0.865), 3 CTAs 8 waves on 49 groups (0.973)
    p148 = B.plan(jobs, co_resident_ctas=148)
    check_invariants(p148, jobs, 148)
    assert (p148['ctas_per_problem'], p148['concurrent_groups']) == (3, 49)
    # a single wave is left alone (the default solve: 6 jobs x 22 CTAs), and so is a pinned group size
    assert B.plan([job(256, 256, 8)] * 6)['ctas_per_problem'] == 22
    assert B.plan(jobs, group_override=2)['ctas_per_problem'] == 2


def test_group_grows_until_the_lists_fit_shared_memory():
    # 132 jobs would get one CTA each, but 512 columns x ~780 rows x 6 B do not fit one CTA
    jobs = [job(512, 512, 8) for _ in range(132)]
    p = B.plan(jobs)
    check_invariants(p, jobs, 132)
    assert p['ctas_per_problem'] > 1 and p['list_rows_smem'] >= (512 // p['ctas_per_problem']) * 3 // 2
    # a retry that asks for longer lists gets more spill rows
    longer = B.plan([dict(j, list_mul=8) for j in jobs])
    assert longer['list_rows_smem'] + longer['spill_rows'] > p['list_rows_smem'] + p['spill_rows']


def test_override_and_bad_arguments():
    p = B.plan([job(64, 64, 8)], group_override=7)
    assert p['ctas_per_problem'] == 7
    assert B.plan([job(64, 64, 8)], group_override=1000)['ctas_per_problem'] == 132
    with pytest.raises(ValueError):
        B.plan([dict(n_in=0, n_out=4, nbits=4, digits=1)])


def test_random_job_mixes_keep_the_invariants():
    rng = np.random.default_rng(0)
    for _ in range(200):
        n = int(rng.integers(1, 200))
        jobs = [job(int(rng.integers(1, 400)), int(rng.integers(1, 400)), int(rng.integers(2, 12))) for _ in range(n)]
        for j in jobs:
            j['digits'] = max(j['digits'], 1)
        coop = int(rng.choice([148, 296, 132]))
        check_invariants(B.plan(jobs, co_resident_ctas=coop), jobs, coop)
