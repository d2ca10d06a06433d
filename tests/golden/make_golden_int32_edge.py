"""Store the reference's answers for the CMVM int32-edge family (tests/cmvm_int32_cases.py) in cmvm_int32_edge.json.gz,
in the format of reference_checks.json.gz (name -> [dtype, shape, values]; read with test_oracle_cross.load_stored):

  {case}_single_{method}_{key}       solve_single with each selector
  {case}_solve{dc}{a}_s{i}_{key}     solve with decompose_dc = dc; `a` marks search_all_decompose_dc on
  {case}_csd{center}_{j}             csd_decompose -> (digits, shift0, shift1)
  {case}_kd{dc}_{j}                  kernel_decompose -> (m0, m1)
  ints_{name}                        int_arr_to_csd

Needs oracle/_ref built from the reference sources (``make -C oracle REF=<reference checkout>``):

    python tests/golden/make_golden_int32_edge.py
"""

import gzip
import json
import sys
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
ROOT = HERE.parents[1]
sys.path[:0] = [str(ROOT), str(ROOT / 'tests'), str(HERE)]

import cmvm_int32_cases as F  # noqa: E402
from make_golden_refchecks import put_stage  # noqa: E402

from oracle import ref  # noqa: E402


def save(name, out):
    """As make_golden_refchecks.save, with a zero gzip timestamp so that a rerun writes the same bytes."""
    enc = {k: [np.asarray(v).dtype.str, list(np.shape(v)), np.asarray(v).ravel().tolist()] for k, v in out.items()}
    with open(HERE / name, 'wb') as raw, gzip.GzipFile(name, 'wb', fileobj=raw, mtime=0) as f:
        f.write(json.dumps(enc, separators=(',', ':'), sort_keys=True).encode())
    print(name, len(out), 'entries')


def solve_key(dc, search_all):
    return f'solve{dc}{"a" if search_all else ""}'


def int32_edge():
    out = {}
    for name, W in F.matrices().items():
        for m in F.METHODS:
            put_stage(out, f'{name}_single_{m}', ref.solve_single(W, m))
        for dc, search_all in F.SOLVES:
            stages = ref.solve(W, decompose_dc=dc, search_all_decompose_dc=search_all)
            assert len(stages) == 2
            for i, st in enumerate(stages):
                put_stage(out, f'{name}_{solve_key(dc, search_all)}_s{i}', st)
        for center in (True, False):
            for j, a in enumerate(ref.csd_decompose(W, center)):
                out[f'{name}_csd{int(center)}_{j}'] = a
        for dc in F.KD_DCS:
            m0, m1 = ref.kernel_decompose(W, dc)
            out[f'{name}_kd{dc}_0'], out[f'{name}_kd{dc}_1'] = m0, m1
    for name, x in F.ints().items():
        out[f'ints_{name}'] = ref.int_arr_to_csd(x)
    save('cmvm_int32_edge.json.gz', out)


if __name__ == '__main__':
    assert ref.available(), 'oracle/_ref is not built'
    int32_edge()
