"""The DAIS interpreter for every opcode (da4ml_b200.dais) without a GPU: the op evaluator of dais_replay.cuh, compiled
with g++ behind a sequential driver (tests/simt/dais_eval.py), reproduces the reference interpreter's stored answers bit
for bit, error messages included; every host check of the library rejects its malformed program before any device call.
The answers are in tests/golden/dais_programs.json.gz (tests/golden/make_golden_dais_programs.py)."""
import hashlib
import re

import dais_programs as G
import numpy as np
import pytest
from test_dais_replay import run_key


@pytest.fixture(scope='module')
def stored():
    from test_oracle_cross import load_stored

    return load_stored('dais_programs.json.gz')


def named_programs(z):
    return {k.split('/', 1)[1]: v.astype(np.int32) for k, v in z.items() if k.startswith('words/')}


def check_answer(want, fn, prog, x, tag):
    """``fn(prog, x)`` gives what the reference gave: the same float64 bits, digest, or RuntimeError message."""
    if isinstance(want, str) and want.startswith('error:'):
        with pytest.raises(RuntimeError) as e:
            fn(prog, x)
        assert str(e.value) == want[len('error:') :], tag
        return
    got = fn(prog, x)
    bits = np.ascontiguousarray(got, dtype=np.float64).view(np.uint64)
    if isinstance(want, str):
        assert 'sha256:' + hashlib.sha256(np.ascontiguousarray(got).tobytes()).hexdigest() == want, tag
    else:
        assert bits.shape == want.shape and np.array_equal(bits, want), tag


def test_random_programs_are_the_stored_ones(stored):
    for seed in G.RANDOM_SEEDS:
        assert hashlib.sha256(G.random_case(seed)[0].tobytes()).hexdigest() == stored[f'words_sha256/random{seed}'], seed
    assert hashlib.sha256(G.random_program(**G.MULTI_CHUNK).tobytes()).hexdigest() == stored['words_sha256/multi_chunk']
    assert hashlib.sha256(G.lookup_oob_program(0, pad=G.OOB_PAD).tobytes()).hexdigest() == stored['words_sha256/lookup_oob_padded']


def test_random_programs_cover_every_opcode():
    seen = set()
    for seed in G.RANDOM_SEEDS:
        p = G.random_case(seed)[0]
        n_in, n_out, n_ops = int(p[2]), int(p[3]), int(p[4])
        o = 6 + n_in + 3 * n_out
        seen |= set(p[o : o + 8 * n_ops].reshape(-1, 8)[:, 0].tolist())
    assert seen == {-9, -6, -3, -2, -1, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10}


def test_evaluator_reproduces_named_programs(stored):
    from simt import dais_eval

    for name, prog in named_programs(stored).items():
        for tag, x in G.stored_inputs(name, prog):
            check_answer(stored[run_key(prog, x)], dais_eval.run, prog, x, f'{name}/{tag}')


@pytest.mark.parametrize('seed', G.RANDOM_SEEDS)
def test_evaluator_reproduces_random_programs(stored, seed):
    from simt import dais_eval

    prog, x = G.random_case(seed)
    check_answer(stored[run_key(prog, x)], dais_eval.run, prog, x, seed)


def test_evaluator_reproduces_a_large_program(stored):
    from simt import dais_eval

    prog, x = G.random_program(**G.MULTI_CHUNK), G.multi_chunk_inputs()
    assert not stored[run_key(prog, x)].startswith('error:')
    check_answer(stored[run_key(prog, x)], dais_eval.run, prog, x, 'multi_chunk')
    prog, x = G.lookup_oob_program(0, pad=G.OOB_PAD), G.late_lookup_failure_inputs()
    check_answer(stored[run_key(prog, x)], dais_eval.run, prog, x, 'late lookup failure')
    dais_eval.run(prog, x[: G.OOB_FIRST_FAILING])  # nothing fails before that sample


def test_shift_counts_follow_x86_masking(stored):
    """The documented cases: quantize from f=0 to f=1 maps 5 -> 0 and -5 -> -0.5; a 33-bit signed wrap has int_min -1."""
    from simt import dais_eval

    p = named_programs(stored)['shift_quantize_f0_f1']
    assert dais_eval.run(p, np.array([[5.0], [-5.0]]))[:, 1].tolist() == [0.0, -0.5]
    p = named_programs(stored)['shift_wide_wrap']
    assert dais_eval.run(p, np.array([[-1.0, 0.0]]))[0, 0] == -1.0


def _mutations():
    """(words, expected message) of malformed programs; built from a valid program with a table and a mux."""
    n_in, n_out = 2, 2
    ops = [
        [-1, 0, -1, 0, 0, 1, 3, 0],
        [-1, 1, -1, 0, 0, 1, 3, 0],
        [0, 0, 1, 0, 0, 1, 4, 0],
        [6, 0, 1, 2, 0, 1, 3, 0],
        [8, 0, -1, 0, 0, 0, 8, 0],
        [9, 3, -1, 1, 0, 0, 1, 0],
        [10, 0, 1, 0, 1 << 24, 1, 3, 0],
    ]
    table = list(range(16))

    def words(ops=ops, tables=(table,), header=None):
        hdr = header or [1, 0, n_in, n_out, len(ops), len(tables)]
        w = hdr + [0, 0, 4, 6, 0, 0, 0, 1]
        for op in ops:
            w += op
        w += [len(t) for t in tables]
        for t in tables:
            w += list(t)
        return np.array(w, np.int32)

    def op_set(i, field, value):
        o = [list(op) for op in ops]
        o[i][field] = value
        return words(o)

    good = words()
    yield good, None
    yield good[:5], 'Binary data too small to contain valid DAIS model file'
    yield np.concatenate([[3], good[1:]]).astype(np.int32), 'DAIS version mismatch: expected version 1, got version 3'
    yield good[:-1], f'Binary data size mismatch: expected {4 * good.size} bytes , got {4 * (good.size - 1)} bytes'
    yield words(header=[1, 0, n_in, n_out, len(ops), -1]), 'negative count'
    yield words(tables=([0] * 3,))[:-3], 'size mismatch'
    w = good.copy()
    w[6 + n_in + 3 * n_out + 8 * len(ops)] = -16
    yield w, 'Lookup table 0 has a negative size (-16)'
    yield op_set(2, 1, 2), 'Operation 2 has id0=2violating causality'
    yield op_set(2, 2, 5), 'Operation 2 has id1=5 violating causality'
    yield op_set(3, 3, 3), 'Operation 3 has cond_idx=3 violating causality'
    yield op_set(3, 3, -1), 'Operation 3 has cond_idx=-1 violating causality'
    yield op_set(2, 0, 11), 'Unknown opcode: 11 at index 2'
    yield op_set(2, 0, -4), 'Unknown opcode: -4 at index 2'
    yield op_set(0, 1, 2), 'input index out of range at operation 0'
    yield op_set(2, 1, -3), 'Operation 2 has id0=-3 out of range'
    yield op_set(2, 2, -1), 'Operation 2 has id1=-1 out of range'
    yield op_set(3, 7, 1), 'Unsupported msb_mux shift configuration: shift0=1, shift1=1'
    yield op_set(4, 3, 1), 'Operation 4 has table index 1 out of range (1 tables)'
    yield op_set(4, 3, -1), 'Operation 4 has table index -1 out of range (1 tables)'
    yield op_set(5, 3, 3), 'Unknown bit unary operation with data_low=3'
    yield op_set(6, 4, 3 << 24), 'Unknown bit binary operation with data_low=0'
    w = good.copy()
    w[6 + n_in] = 7
    yield w, 'output index out of range at output 0'
    w = good.copy()
    w[6] = 2000
    yield w, 'input shift out of range at input 0'
    w = good.copy()
    w[6 + n_in + n_out + 1] = -1024
    yield w, 'output shift out of range at output 1'


def test_host_checks_reject_malformed_programs_before_touching_the_device():
    """Every data-independent check runs on the host at load: no GPU is needed to be told a program is bad, the
    evaluator's g++ build agrees on every message, and the library keeps working afterwards."""
    from simt import dais_eval

    from da4ml_b200.dais import DaisProgram

    for words, msg in _mutations():
        if msg is None:
            with DaisProgram(words) as p:
                assert (p.n_in, p.n_out, p.n_ops, p.n_tables) == (2, 2, 7, 1)
                assert p.n_levels == 4 and p.max_width == 8
            dais_eval.run(words, np.array([[1.0, -2.0]]))
            continue
        with pytest.raises(RuntimeError, match=re.escape(msg)):
            DaisProgram(words)
        with pytest.raises(RuntimeError, match=re.escape(msg)):
            dais_eval.run(words, np.zeros((1, 2)))
    with DaisProgram(next(_mutations())[0]) as p:
        assert p.n_ops == 7


def test_run_interp_header_errors_without_a_device():
    from da4ml_b200.dais import run_interp

    with pytest.raises(RuntimeError, match='Invalid binary logic data'):
        run_interp(np.array([1, 0, 1], np.int32), np.zeros(1))
    with pytest.raises(RuntimeError, match='DAIS version mismatch: expected version 1, got version 2'):
        run_interp(np.array([2, 0, 1, 1, 0, 0], np.int32), np.zeros(1))
    assert run_interp(np.array([1, 0, 1, 3, 0, 0], np.int32), np.zeros(0)).shape == (0, 3)
