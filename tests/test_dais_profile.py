"""Profiling DAIS programs (``DaisProgram.dump`` / ``profile``, ``OpProfile``) without a GPU.

The evaluator of dais_replay.cuh, compiled with g++ behind the sequential driver of tests/simt/dais_profile_harness.cc
(``dp_dump`` / ``dp_profile``), reproduces the reference interpreter's value of every op, stored in
tests/golden/dais_op_values.json.gz (tests/golden/make_golden_dais_op_values.py).  The ``OpProfile`` derivations are
checked on hand-built cases and against ``types.minimal_kif_array``; the argument checks of the C ABI refuse bad calls
before any device call."""
import ctypes as C
import gzip
import hashlib
import json
from pathlib import Path

import dais_programs as G
import numpy as np
import pytest

GOLDEN = Path(__file__).resolve().parent / 'golden'
I64_MAX, I64_MIN = (1 << 63) - 1, -(1 << 63)
PROFILE_SEEDS = range(0, 80, 4)  # as tests/golden/make_golden_dais_op_values.py


# ---- the g++ build of the evaluator (tests/simt/dais_profile_harness.cc) -----------------------------------------------
def harness_stats(prog, x) -> np.ndarray:
    """[n_ops, 3] int64 {min, max, OR} of the op codes, sample by sample on the CPU."""
    from simt import dais_profile

    return dais_profile.stats(prog, x)


def harness_profile(prog, x):
    from da4ml_b200.dais import OpProfile

    st = harness_stats(prog, x)
    n = np.asarray(x, dtype=np.float64).size // max(int(np.asarray(prog)[2]), 1)
    return OpProfile(n, st[:, 0], st[:, 1], st[:, 2], kif_of(prog))


def harness_dump(prog, x, ops=None) -> np.ndarray:
    from simt import dais_profile

    return dais_profile.dump(prog, x, ops)


# ---- the stored reference values ---------------------------------------------------------------------------------------
def kif_of(prog) -> np.ndarray:
    w = np.asarray(prog, np.int32)
    n_in, n_out, n_ops = int(w[2]), int(w[3]), int(w[4])
    o = 6 + n_in + 3 * n_out
    return w[o : o + 8 * n_ops].reshape(n_ops, 8)[:, 5:8].astype(np.int64)


def load_op_values() -> dict:
    with gzip.open(GOLDEN / 'dais_op_values.json.gz', 'rt') as f:
        return json.load(f)


def case_program(case: str):
    """(program words, inputs) of a stored case: "<name>/<tag>" of dais_programs.json.gz or "random<seed>"."""
    if case.startswith('random'):
        return G.random_case(int(case[len('random') :]))
    from test_dais_interp import named_programs
    from test_oracle_cross import load_stored

    name, tag = case.split('/')
    prog = named_programs(load_stored('dais_programs.json.gz'))[name]
    return prog, dict(G.stored_inputs(name, prog))[tag]


def as_outputs(codes, prog, ops=None) -> np.ndarray:
    """Codes converted as the interpreter converts an output (``dais_output``, shift 0, not negated):
    ``double(code) * 2^-f``."""
    f = kif_of(prog)[:, 2] if ops is None else kif_of(prog)[np.asarray(ops), 2]
    return np.asarray(codes, np.int64).astype(np.float64) * np.ldexp(1.0, -f)[None, :]


def check_against_stored(want: dict, codes, stats, prog, tag):
    """All-ops ``codes`` [n, n_ops] and ``stats`` [n_ops, 3] equal the reference's stored values."""
    y = np.ascontiguousarray(as_outputs(codes, prog))
    assert hashlib.sha256(y.tobytes()).hexdigest() == want['sha256'], tag
    ops = np.asarray(want['ops'], np.int64)
    assert np.array_equal(stats[ops, 0], want['min']), tag
    assert np.array_equal(stats[ops, 1], want['max']), tag
    assert np.array_equal(stats[ops, 2], want['or']), tag


@pytest.fixture(scope='module')
def op_values():
    return load_op_values()


def test_stored_cases_are_the_named_programs_and_seeds(op_values):
    from test_dais_interp import named_programs
    from test_oracle_cross import load_stored

    names = named_programs(load_stored('dais_programs.json.gz'))
    want = {f'{n}/{t}' for n, p in names.items() for t, _ in G.stored_inputs(n, p)} | {f'random{s}' for s in PROFILE_SEEDS}
    assert set(op_values) == want
    assert sum('error' in v for v in op_values.values()) >= 1  # the lookup failure


def test_harness_reproduces_the_reference_values(op_values):
    for case, want in op_values.items():
        prog, x = case_program(case)
        if 'error' in want:
            for fn in (harness_stats, harness_dump):
                with pytest.raises(RuntimeError) as e:
                    fn(prog, x)
                assert str(e.value) == want['error'], case
            continue
        codes, stats = harness_dump(prog, x), harness_stats(prog, x)
        check_against_stored(want, codes, stats, prog, case)
        # the statistics of every op, the wide ones too, are those of the dump
        if len(codes):
            assert np.array_equal(stats, np.stack([codes.min(0), codes.max(0), np.bitwise_or.reduce(codes, axis=0)], 1)), case


def test_observed_kif_is_minimal_kif_of_the_observed_range(op_values):
    from da4ml_b200.types import minimal_kif_array

    checked = 0
    for case, want in op_values.items():
        if 'error' in want:
            continue
        prog, x = case_program(case)
        p = harness_profile(prog, x)
        f = p.kif[:, 2]
        small = (np.abs(p.min.astype(object)) < 2**53) & (np.abs(p.max.astype(object)) < 2**53)
        small = small.astype(bool) & (np.abs(f) < 900)
        t = np.array([(int(b) & -int(b)).bit_length() - 1 if b else 0 for b in p.bits_or])
        q = np.stack([np.ldexp(p.min.astype(np.float64), -f), np.ldexp(p.max.astype(np.float64), -f), np.ldexp(1.0, t - f)], 1)
        assert np.array_equal(p.observed_kif[small], minimal_kif_array(q[small]).astype(np.int64)), case
        checked += int(small.sum())
    assert checked > 2000


def test_merge_of_batches_is_the_profile_of_the_whole(op_values):
    for case in ('traced_mlp/mixed', 'traced_lookup/mixed', 'random8', 'random12', 'shift_wide_wrap/edge'):
        prog, x = case_program(case)
        whole = harness_profile(prog, x)
        parts = [harness_profile(prog, x[a:b]) for a, b in ((0, 1), (1, 100), (100, 100), (100, len(x)))]
        m = parts[0]
        for q in parts[1:]:
            m = m.merge(q)
        assert m.n_samples == whole.n_samples == len(x)
        for k in ('min', 'max', 'bits_or'):
            assert np.array_equal(getattr(m, k), getattr(whole, k)), (case, k)
        assert np.array_equal(m.observed_kif, whole.observed_kif) and np.array_equal(m.overflow, whole.overflow)


def _profile(rows, kif):
    from da4ml_b200.dais import OpProfile

    rows = np.asarray(rows, dtype=object)
    return OpProfile(1, rows[:, 0].astype(np.int64), rows[:, 1].astype(np.int64), rows[:, 2].astype(np.int64), kif)


def test_observed_kif_and_overflow_on_hand_built_cases():
    cases = [
        # (min, max, or), declared (k, i, f) -> observed (k, i, f), overflow
        ((0, 0, 0), (1, 3, 2), (0, 0, 0), False),  # always zero
        ((-8, -1, -1), (1, 3, 0), (1, 3, 0), False),  # negative only: [-8, -1] needs 3 bits + sign
        ((-9, -1, -1), (1, 3, 0), (1, 4, 0), True),  # one past the signed minimum
        ((-12, 20, 0b11100 | -16), (1, 5, 2), (1, 3, 0), False),  # t = 2: codes are multiples of 4
        ((4, 12, 12), (0, 2, 2), (0, 2, 0), False),  # t = 2, unsigned
        ((0, 15, 15), (0, 4, 0), (0, 4, 0), False),  # unsigned [0, 2^w - 1]: the top of the range
        ((0, 16, 16), (0, 4, 0), (0, 5, -4), True),  # one past it (t = 4)
        ((-1, 0, -1), (0, 4, 0), (1, 0, 0), True),  # a negative code in an unsigned type
        ((-8, 7, -1), (1, 3, 0), (1, 3, 0), False),  # signed boundaries exactly
        ((-8, 8, -1), (1, 3, 0), (1, 4, 0), True),
        ((0, 0, 0), (0, -2, 1), (0, 0, 0), False),  # w <= 0: the range is {0}
        ((0, 2, 2), (0, -2, 1), (0, 1, 0), True),
        ((-2, 0, -2), (1, -3, 1), (1, 0, 0), True),
        ((I64_MIN, I64_MAX, -1), (1, 63, 0), (1, 63, 0), False),  # the whole int64 range
        ((I64_MIN, I64_MIN, I64_MIN), (1, 63, 0), (1, 63, -63), False),  # t = 63
        ((I64_MIN, -1, -1), (1, 62, 0), (1, 63, 0), True),
        ((0, I64_MAX, I64_MAX), (0, 62, 0), (0, 63, 0), True),
        ((0, I64_MAX, I64_MAX), (0, 63, 0), (0, 63, 0), False),
        ((1 << 62, 1 << 62, 1 << 62), (0, 40, 30), (0, 33, -32), False),  # t = 62 with f = 30
        ((-(1 << 62), 0, -(1 << 62)), (1, 100, 0), (1, 62, -62), False),  # a declared width above 64 bits
    ]
    p = _profile([c[0] for c in cases], np.array([c[1] for c in cases]))
    for j, (st, kif, obs, ovf) in enumerate(cases):
        assert tuple(p.observed_kif[j]) == obs, (j, st)
        assert bool(p.overflow[j]) == ovf, (j, st)


def test_empty_profile_is_the_identity_and_merges_away():
    from da4ml_b200.dais import DaisProgram

    prog, x = case_program('traced_product/mixed')
    with DaisProgram(prog) as dp:
        empty = dp.profile(np.zeros((0, dp.n_in)))  # no samples: no device call
        assert empty.n_samples == 0
        assert (empty.min == I64_MAX).all() and (empty.max == I64_MIN).all() and (empty.bits_or == 0).all()
        assert not empty.overflow.any() and not empty.observed_kif.any()
        assert dp.dump(np.zeros((0, dp.n_in)), [0, 3, 3]).shape == (0, 3)
        assert np.array_equal(dp.kif, kif_of(prog)) and dp.kif.shape == (dp.n_ops, 3)
    whole = harness_profile(prog, x)
    m = empty.merge(whole)
    for k in ('min', 'max', 'bits_or'):
        assert np.array_equal(getattr(m, k), getattr(whole, k))
    with pytest.raises(ValueError, match='different programs'):
        whole.merge(harness_profile(*case_program('traced_bits/mixed')))


def test_arguments_are_refused_before_any_device_call():
    import da4ml_b200._binary as B
    from da4ml_b200.dais import DaisProgram

    L = B._L
    prog, _ = case_program('traced_product/mixed')
    x = np.zeros((4, int(prog[2])))
    with DaisProgram(prog) as dp:
        n = dp.n_ops
        for ops in ([0, n], [-1], [1 << 40]):
            with pytest.raises(ValueError, match='out of range'):
                dp.dump(x, ops)
        with pytest.raises(TypeError, match='float64 CUDA tensor'):
            import torch

            dp.profile(torch.zeros(4, int(prog[2]), dtype=torch.float32))
        h = dp._handle()
        vals = np.zeros((4, 2), np.int64)
        ids = np.array([0, n], np.int32)
        stats = np.zeros((n, 3), np.int64)

        def refused(rc, msg):
            assert rc == 1 and msg in L.da4ml_cmvm_last_error().decode(), L.da4ml_cmvm_last_error()

        refused(L.da4ml_dais_program_dump(h, x.ctypes.data, 4, ids.ctypes.data, 2, vals.ctypes.data, 0, None), f'op id {n} at position 1 is out of range [0, {n})')
        ids[1] = -3
        refused(L.da4ml_dais_program_dump(h, x.ctypes.data, 4, ids.ctypes.data, 2, vals.ctypes.data, 0, None), 'op id -3 at position 1')
        ids[1] = 0
        refused(L.da4ml_dais_program_dump(h, x.ctypes.data, 4, ids.ctypes.data, -1, vals.ctypes.data, 0, None), 'n_sel is negative')
        refused(L.da4ml_dais_program_dump(h, x.ctypes.data, 4, None, 2, vals.ctypes.data, 0, None), 'op_ids is null')
        refused(L.da4ml_dais_program_dump(h, x.ctypes.data, 4, ids.ctypes.data, 2, None, 0, None), 'values is null')
        refused(L.da4ml_dais_program_dump(h, None, 4, ids.ctypes.data, 2, vals.ctypes.data, 0, None), 'inputs is null')
        refused(L.da4ml_dais_program_dump(h, x.ctypes.data, -4, ids.ctypes.data, 2, vals.ctypes.data, 0, None), 'n_samples is negative')
        refused(L.da4ml_dais_program_dump(None, x.ctypes.data, 4, ids.ctypes.data, 2, vals.ctypes.data, 0, None), 'handle is null')
        refused(L.da4ml_dais_program_profile(h, x.ctypes.data, 4, 0, None, None), 'stats is null')
        refused(L.da4ml_dais_program_profile(h, None, 4, 0, None, stats.ctypes.data), 'inputs is null')
        refused(L.da4ml_dais_program_profile(h, x.ctypes.data, -1, 0, None, stats.ctypes.data), 'n_samples is negative')
        refused(L.da4ml_dais_program_profile(None, x.ctypes.data, 4, 0, None, stats.ctypes.data), 'handle is null')
        assert not stats.any() and not vals.any()


def test_profiling_symbols_are_exported_and_declared():
    import da4ml_b200._binary as B
    from test_abi import declared_symbols

    for s in ('da4ml_dais_program_profile', 'da4ml_dais_program_dump'):
        assert hasattr(C.CDLL(str(B.lib_path())), s) and s in declared_symbols() and s in B.EXPORTED_SYMBOLS
