"""Reference values of every op of a DAIS program, for the profiling tests (tests/test_dais_profile.py,
tests/test_dais_profile_gpu.py).

  dais_op_values.json.gz
    {"<case>": {"sha256": ..., "ops": [...], "min": [...], "max": [...], "or": [...]}} or {"<case>": {"error": <message>}}

Cases are the named programs of dais_programs.json.gz on each of their stored inputs ("<name>/<tag>") and the seeded
random programs of PROFILE_SEEDS ("random<seed>"), as tests/dais_programs.py regenerates them.  Each program is
rewritten into its all-ops-as-outputs variant (n_out = n_ops, out_idxs = 0..n_ops-1, out shifts 0, not negated) and run
through the reference interpreter (oracle/_ref/libdais_ref.so), which then returns ``double(code) * 2^-f`` for every op:
  sha256      of those [n_samples, n_ops] float64 bytes;
  ops         the ops whose codes are all below 2^53 in magnitude, so that they are recovered exactly from the outputs;
  min/max/or  per listed op, the min, max and bitwise OR of the recovered codes;
  error       the reference's message, when it raised.

Needs oracle/_ref built from the reference sources (``make -C oracle REF=<reference checkout>``):

    python tests/golden/make_golden_dais_op_values.py
"""

import gzip
import hashlib
import json
import sys
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
ROOT = HERE.parents[1]
sys.path[:0] = [str(ROOT), str(ROOT / 'tests')]

import dais_programs as G  # noqa: E402

from oracle import dais_ref  # noqa: E402

OUT = 'dais_op_values.json.gz'
PROFILE_SEEDS = range(0, 80, 4)  # 20 of the random programs, narrow (seed % 3 == 0) and wide


def all_ops_variant(words) -> np.ndarray:
    """The program with every op as an output, in op order: out_idxs 0..n_ops-1, out shifts 0, not negated."""
    w = np.asarray(words, np.int32)
    n_in, n_out, n_ops = int(w[2]), int(w[3]), int(w[4])
    head, inp_shifts, rest = w[:6].copy(), w[6 : 6 + n_in], w[6 + n_in + 3 * n_out :]
    head[3] = n_ops
    return np.concatenate([head, inp_shifts, np.arange(n_ops), np.zeros(2 * n_ops, np.int32), rest]).astype(np.int32)


def cases():
    """(case name, program words, inputs) of every stored case."""
    from test_oracle_cross import load_stored

    stored = load_stored('dais_programs.json.gz')
    for key in sorted(k for k in stored if k.startswith('words/')):
        name, prog = key.split('/', 1)[1], stored[key].astype(np.int32)
        for tag, x in G.stored_inputs(name, prog):
            yield f'{name}/{tag}', prog, x
    for seed in PROFILE_SEEDS:
        prog, x = G.random_case(seed)
        yield f'random{seed}', prog, x


def fractionals(words) -> np.ndarray:
    w = np.asarray(words, np.int32)
    n_in, n_out, n_ops = int(w[2]), int(w[3]), int(w[4])
    o = 6 + n_in + 3 * n_out
    return w[o : o + 8 * n_ops].reshape(n_ops, 8)[:, 7].astype(np.int64)


def entry(prog, x) -> dict:
    try:
        y = np.ascontiguousarray(dais_ref.run(all_ops_variant(prog), x))
    except RuntimeError as e:
        return {'error': str(e)}
    codes = np.ldexp(y, fractionals(prog)[None, :])  # exact wherever |code| < 2^53
    exact = np.all(np.isfinite(codes) & (np.abs(codes) < 2.0**53), axis=0)
    ops = np.flatnonzero(exact)
    c = codes[:, ops].astype(np.int64)
    assert np.array_equal(np.ldexp(c.astype(np.float64), -fractionals(prog)[None, ops]), y[:, ops])
    return {
        'sha256': hashlib.sha256(y.tobytes()).hexdigest(),
        'ops': ops.tolist(),
        'min': c.min(axis=0, initial=(1 << 63) - 1).tolist(),
        'max': c.max(axis=0, initial=-(1 << 63)).tolist(),
        'or': np.bitwise_or.reduce(c, axis=0).tolist() if len(c) else [0] * len(ops),
    }


def main():
    assert dais_ref.available(), 'oracle/_ref is not built'
    out = {name: entry(prog, x) for name, prog, x in cases()}
    with gzip.GzipFile(HERE / OUT, 'wb', mtime=0) as f:
        f.write(json.dumps(out, separators=(',', ':'), sort_keys=True).encode())
    errors = sum('error' in v for v in out.values())
    print(OUT, len(out), 'cases,', errors, 'errors,', (HERE / OUT).stat().st_size // 1024, 'KiB')


if __name__ == '__main__':
    main()
