"""The refresh team (team R) joins the first counting pass of every recount once its refresh is done (own_recount_help):
its warps claim chunks of (column, row) items next to team C.  Under the CPU SIMT shim, with a pair-counter table so
small that first passes run out of slots while team R counts: the graphs and the exact work counters of accounting mode
must equal the reference's, and team R must have claimed chunks, some of them in passes that were abandoned."""
import ctypes as C
import shutil
import subprocess

import pytest
from conftest import assert_stage_equal, int_matrix

import simt
from oracle import port


@pytest.fixture(scope='module')
def counted_lib(tmp_path_factory):
    """The simulator harness with the solve kernel wrapped to read team R's counters (simt/recount_help_harness.cc), with
    the signatures of the shared harness functions taken over from simt.lib()."""
    gxx = '/usr/bin/g++' if shutil.which('/usr/bin/g++') else 'g++'
    so = tmp_path_factory.mktemp('recount_help') / 'librecount_help.so'
    subprocess.run([gxx, '-O2', '-std=c++17', '-ffp-contract=off', '-fPIC', '-shared', '-w', str(simt.HERE / 'recount_help_harness.cc'), '-o', str(so)], check=True)
    lib, ref = C.CDLL(str(so)), simt.lib()
    for name in ('sim_last_error', 'sim_solve_single', 'sim_set_schedule', 'sim_set_own_caps', 'sim_set_list_cap'):
        getattr(lib, name).argtypes = getattr(ref, name).argtypes
        getattr(lib, name).restype = getattr(ref, name).restype
    lib.sim_helped.argtypes = [C.POINTER(C.c_longlong)]
    return lib


@pytest.mark.parametrize('schedule', [0, 2])
def test_refresh_team_counts_first_passes_that_overflow(counted_lib, monkeypatch, schedule):
    W = int_matrix(24, 40, 8, 5)
    want = port.solve_single(W, 'wmc')
    cnt = port.partial(W, 'wmc')
    monkeypatch.setattr(simt, '_lib', counted_lib)
    simt.set_own_caps(hash_log=8)  # 160 usable slots per pass: first passes overflow and are split
    simt.set_schedule(schedule)
    got, meta = simt.solve_single(W, 'wmc', ctas=2, cta_threads=128, accounting=True)  # 4 warps: team R is the last
    helped = (C.c_longlong * 2)()
    counted_lib.sim_helped(helped)
    chunks, abandoned = helped
    assert_stage_equal(got, want, f'schedule {schedule} ')
    assert (meta[2], meta[3], meta[4], meta[5], meta[6]) == (cnt['iters'], cnt['sum_F'], cnt['sum_R'], cnt['F0'], cnt['R0'])
    assert chunks > 0, 'team R never claimed a chunk of a first pass'
    assert abandoned > 0, 'no first pass overflowed while team R was counting'
