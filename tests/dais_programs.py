"""Seeded random DAIS programs for the interpreter tests (TEST INFRASTRUCTURE).

Every opcode of the reference interpreter and its negated form, signed and unsigned dtypes of widths 1-63, lookup
tables with non-zero ``data_high`` offsets, both legal MSB-mux shift configurations, 64-bit constants, and shift counts
outside [0, 64) where the reference's compiled code masks them (quantize to more fractional bits, constant add to fewer,
33-bit and wider signed wraps).  Program words follow ``CombLogic.to_binary`` (reference types.py:500-541)."""
from __future__ import annotations

import hashlib

import numpy as np

UNARY = [2, -2, 3, -3, 4, 8, 9, -9]
BINARY = [0, 1, 6, -6, 7, 10]


def _dtype(rng, max_width=63, frac=(-6, 10)):
    signed = int(rng.integers(0, 2))
    w = int(rng.integers(1, max_width + 1))
    if signed and w < 2 and rng.random() < 0.5:
        w = 2
    f = int(rng.integers(frac[0], frac[1] + 1))
    return signed, w - f - signed, f


def _width(d):
    return d[0] + d[1] + d[2]


def _set_f(d, f):
    """Move the binary point of dtype ``d`` (a list) to ``f`` fractional bits, keeping its width."""
    d[1] = _width(d) - d[0] - f
    d[2] = f


def random_program(seed: int, n_in: int = 6, n_ops: int = 48, n_out: int = 8, lookups: bool = True, narrow: bool = False,
                   lookup_on_inputs: bool = False):
    """Words of one random program.  ``narrow`` keeps widths small (values stay far from 64 bits, so the outputs are
    mostly distinct finite numbers); otherwise widths run up to 63 bits and shifts leave [0, 64).  ``lookup_on_inputs``
    makes every table look up an input op, so that no lookup goes out of range unless an input is NaN or huge."""
    rng = np.random.default_rng(seed)
    max_w = 14 if narrow else 63
    ops = []  # [opcode, id0, id1, data_low, data_high, signed, integers, fractionals]
    wraps = []  # ops whose value is wrapped into their dtype's range (the only safe lookup operands)
    tables = []
    for i in range(n_in):
        d = _dtype(rng, max_w)
        ops.append([-1, i, -1, 0, 0, *d])
        wraps.append(i)
    while len(ops) < n_ops:
        i = len(ops)
        r = rng.random()
        if r < 0.06:  # 64-bit constant
            lo, hi = (int(v) for v in rng.integers(-(2**31), 2**31, size=2))
            if narrow:
                hi = -1 if lo < 0 else 0
            ops.append([5, -1, -1, lo, hi, *_dtype(rng, max_w)])
            continue
        opc = int(rng.choice(UNARY + BINARY))
        a = int(rng.integers(0, i))
        b = int(rng.integers(0, i))
        d = list(_dtype(rng, max_w))
        da, db = ops[a][5:], ops[b][5:]
        dl, dh = 0, 0
        if opc in (0, 1):
            dl = int(rng.integers(-4, 5))
            if narrow:
                _set_f(d, min(da[2], db[2] - dl))  # no global shift: the sum keeps its precision
        elif opc in (2, -2, 3, -3):
            if not narrow and rng.random() < 0.3:
                _set_f(d, da[2] + int(rng.integers(1, 4)))  # more fractional bits: the shift count is negative
        elif opc == 4:
            lo = int(rng.integers(-(2**31), 2**31))
            dl, dh = lo, (int(rng.integers(-(2**31), 2**31)) if not narrow and rng.random() < 0.5 else (-1 if lo < 0 else 0))
            if not narrow and rng.random() < 0.3:
                _set_f(d, da[2] - int(rng.integers(1, 4)))  # fewer fractional bits: the shift count is negative
        elif opc in (6, -6):
            c = int(rng.integers(0, i))
            dl = c
            if rng.random() < 0.5:  # shift0 == 0: the output keeps operand 0's fractionals
                _set_f(d, da[2])
                dh = int(rng.integers(-3, 4))
            else:  # shift1 == 0
                dh = db[2] - d[2]
        elif opc == 8:
            cand = [k for k in (range(n_in) if lookup_on_inputs else wraps) if 1 <= _width(ops[k][5:]) <= 8]
            if not cand or not lookups:
                continue
            a = int(rng.choice(cand))
            w0 = _width(ops[a][5:])
            off = int(rng.integers(-3, 1))  # index = v0 - zero - data_high, v0 - zero in [0, 2^w0)
            size = (1 << w0) - off
            tables.append(rng.integers(-(2**31), 2**31, size=size).astype(np.int64) if not narrow else rng.integers(-5000, 5000, size=size))
            dl, dh = len(tables) - 1, off
        elif opc in (9, -9):
            dl = int(rng.integers(0, 3))
        elif opc == 10:
            dl = int(rng.integers(-3, 4))
            dh = (int(rng.integers(0, 3)) << 24) | int(rng.integers(0, 4))
        if opc not in (0, 1, 4, 6, -6, 7, 10):
            b = -1
        if opc in (8,):
            b = -1
        ops.append([opc, a, b, dl, dh, *d])
        if opc in (2, -2, 3, -3, 6, -6):
            wraps.append(i)
    out_idxs = [int(v) for v in rng.integers(-1, n_ops, size=n_out)]
    inp_shifts = [int(v) for v in rng.integers(-3, 4, size=n_in)]
    out_shifts = [int(v) for v in rng.integers(-4, 5, size=n_out)]
    out_negs = [int(v) for v in rng.integers(0, 2, size=n_out)]
    words = [1, 0, n_in, n_out, n_ops, len(tables), *inp_shifts, *out_idxs, *out_shifts, *out_negs]
    for op in ops:
        words += op
    words += [len(t) for t in tables]
    for t in tables:
        words += [int(v) for v in t]
    return np.array(words, dtype=np.int64).astype(np.int32)


def lookup_oob_program(seed: int, pad: int = 0):
    """A program whose table is too short for part of its operand's range: some samples look up out of bounds.
    ``pad`` appends that many shift-adds of the first two inputs that no output reads (a program with many ops is run in
    small chunks of samples)."""
    rng = np.random.default_rng(seed)
    n_in = 3
    ops = [[-1, i, -1, 0, 0, 1, 4, 0] for i in range(n_in)]  # signed 5-bit integers
    ops.append([0, 0, 1, 0, 0, 1, 5, 0])  # 6-bit sum
    ops.append([3, 3, -1, 0, 0, 1, 4, 0])  # wrapped back to 5 bits
    ops.append([8, 4, -1, 0, 2, 0, 16, 0])  # table 0 at offset 2: v0 = -16, -15 give negative indices
    ops.append([8, 2, -1, 1, -1, 0, 16, 0])  # table 1 at offset -1: always in range
    ops += [[0, 0, 1, k % 3, 0, 1, 8, 0] for k in range(pad)]
    table0 = rng.integers(-(2**31), 2**31, size=30)
    table1 = rng.integers(-100, 100, size=33)
    n_out = 3
    words = [1, 0, n_in, n_out, len(ops), 2, 0, 0, 0, 5, 6, 4, 0, 1, -2, 0, 1, 0]
    for op in ops:
        words += op
    words += [30, 33, *table0.tolist(), *table1.tolist()]
    return np.array(words, dtype=np.int64).astype(np.int32)


def random_inputs(seed: int, n: int, n_in: int, special: bool = True):
    """Samples over several scales: in-range integers, fractions, out-of-range magnitudes and (``special``) NaN / +-inf."""
    rng = np.random.default_rng(seed)
    x = rng.integers(-40, 40, size=(n, n_in)).astype(np.float64)
    m = rng.random((n, n_in))
    x = np.where(m < 0.25, rng.normal(0, 8, size=(n, n_in)), x)
    x = np.where((m >= 0.25) & (m < 0.3), rng.normal(0, 1, size=(n, n_in)) * 2.0 ** rng.integers(10, 70, size=(n, n_in)), x)
    if special:
        x = np.where((m >= 0.3) & (m < 0.31), np.nan, x)
        x = np.where((m >= 0.31) & (m < 0.32), np.inf, x)
        x = np.where((m >= 0.32) & (m < 0.33), -np.inf, x)
    return np.ascontiguousarray(x)


# ---- the cases whose reference answers are stored in tests/golden/dais_programs.json.gz ---------------------------
RANDOM_SEEDS = range(80)
MULTI_CHUNK = dict(seed=1000, n_in=8, n_ops=65536, n_out=16, narrow=True, lookup_on_inputs=True)  # 2048 samples per chunk on the device
MULTI_CHUNK_SAMPLES = 5000
MILLION = 1_000_000


def multi_chunk_inputs():
    """Finite inputs of moderate size: every lookup of the multi-chunk program stays in range."""
    return np.clip(random_inputs(7, MULTI_CHUNK_SAMPLES, MULTI_CHUNK['n_in'], special=False), -1000.0, 1000.0)


OOB_PAD = 65536  # filler ops of the padded lookup_oob program: 2048 samples per chunk on the device
OOB_FIRST_FAILING = 4100  # in the third chunk


def late_lookup_failure_inputs():
    """Inputs of ``lookup_oob_program(0, pad=OOB_PAD)``: every lookup stays in range before sample OOB_FIRST_FAILING,
    there x0 + x1 = -15 and after it -16 make the lookup of op 5 fail (index -1, then -2)."""
    rng = np.random.default_rng(17)
    x = np.stack([rng.integers(-7, 8, MULTI_CHUNK_SAMPLES), rng.integers(-7, 8, MULTI_CHUNK_SAMPLES), rng.integers(-16, 16, MULTI_CHUNK_SAMPLES)], axis=1)
    x[OOB_FIRST_FAILING:, :2] = -8
    x[OOB_FIRST_FAILING, 1] = -7
    return x.astype(np.float64)


def random_case(seed):
    """(program words, inputs) of random case ``seed``."""
    prog = random_program(seed, narrow=seed % 3 == 0)
    return prog, random_inputs(seed, 64, int(prog[2]))


def stored_inputs(name: str, prog):
    """The inputs the stored answers of program ``name`` were computed on: [(tag, data)]."""
    n_in = int(prog[2])
    seed = int(hashlib.sha256(name.encode()).hexdigest()[:8], 16)
    runs = [('mixed', random_inputs(seed, 257, n_in))]
    if name.startswith('shift_'):
        runs.append(('edge', np.array([5.0, -5.0, -1.0, 0.5, -0.5, 2.0**40, -(2.0**33), 2.0**32 - 1, np.nan, np.inf, -np.inf, 1e300] * 2)[: 12 * n_in].reshape(-1, n_in)))
    if name == 'lookup_oob':
        runs = [('mixed', random_inputs(5, 50, n_in, special=False)), ('in_range', np.array([[3.0, -2.0, 7.0], [0.0, 0.0, -16.0]]))]
    return runs
