"""Store the reference's own answers for the inputs of the tests that compare with it, so that those tests run without
the reference:

  reference_checks.json.gz   oracle/_ref (the reference's CMVM translation units) on the inputs of tests/test_oracle_cross.py
                             and of tests/test_oracle.py::test_port_matches_reference_random
  dais_reference.json.gz     oracle/_ref/libdais_ref.so (the reference's DAIS interpreter) on the programs and inputs of
                             tests/test_dais_replay.py, keyed by test_dais_replay.run_key

Each file maps a name to [dtype, shape, values] (exact: float32 / float64 values round-trip through JSON).

Needs oracle/_ref built from the reference sources (``make -C oracle REF=<reference checkout>``):

    python tests/golden/make_golden_refchecks.py
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

from conftest import STAGE_KEYS, int_matrix  # noqa: E402

from oracle import dais_ref, ref  # noqa: E402


def save(name, out):
    enc = {k: v if isinstance(v, str) else [np.asarray(v).dtype.str, list(np.shape(v)), np.asarray(v).ravel().tolist()] for k, v in out.items()}
    with gzip.open(HERE / name, 'wt') as f:
        json.dump(enc, f, separators=(',', ':'), sort_keys=True)
    print(name, len(out), 'entries')


def put_stage(out, prefix, st):
    for k in STAGE_KEYS:
        out[f'{prefix}_{k}'] = np.asarray(st[k])


def reference_checks():
    import test_oracle
    import test_oracle_cross as X

    out = {}
    for seed in range(60):
        W, _, kw = X.single_case(seed)
        put_stage(out, f'cross_single{seed}', ref.solve_single(W, **kw))
    for seed in range(40):
        W, _, kw = X.full_case(seed)
        stages = ref.solve(W, **kw)
        assert len(stages) == 2
        for i, st in enumerate(stages):
            put_stage(out, f'cross_full{seed}_s{i}', st)
    for seed in range(20):
        W, ints, Wi = X.helper_case(seed)
        p = f'cross_helpers{seed}'
        for center in (True, False):
            for j, a in enumerate(ref.csd_decompose(W, center)):
                out[f'{p}_csd{int(center)}_{j}'] = a
        out[f'{p}_ints_csd'] = ref.int_arr_to_csd(ints)
        for dc in X.HELPER_DCS:
            m0, m1 = ref.kernel_decompose(Wi, dc)
            out[f'{p}_kd{dc}_0'], out[f'{p}_kd{dc}_1'] = m0, m1
    for seed in range(6):
        W, kw = test_oracle.random_case(seed)
        stages = ref.solve(W, **kw)
        assert len(stages) == 2
        for i, st in enumerate(stages):
            put_stage(out, f'random{seed}_s{i}', st)
    save('reference_checks.json.gz', out)


def dais_reference():
    import da4ml_b200._binary as B
    import test_dais_replay as D
    from da4ml_b200.types import pipeline_from_arrays

    out = {}

    def run(prog, x, n_threads=1):
        y = dais_ref.run(prog, x)
        out[D.run_key(prog, x)] = y
        return y

    for _, sol, x in D.float_replay_inputs():
        run(sol.to_binary(), x)
    for _, sol, x in D.cuda_replay_inputs():
        run(sol.to_binary(), x)

    class _KeepRecorder:  # the probe test installs its stand-in through monkeypatch; keep the recorder installed instead
        def setattr(self, *a):
            pass

    B.dais_interp_run = run
    D.test_kernel_from_fixed_point_probes(_KeepRecorder(), None)
    # the CUDA solve equals the reference's solve bit for bit (tests/test_cmvm_gpu.py), so its program is the reference's
    stages = ref.solve(int_matrix(*D.SOLVED_W), search_all_decompose_dc=False, decompose_dc=-1)
    y = dais_ref.run(pipeline_from_arrays(stages).solutions[0].to_binary(), D.solved_matrix_inputs())
    out['solved_sha256'] = hashlib.sha256(np.ascontiguousarray(y).tobytes()).hexdigest()
    save('dais_reference.json.gz', out)


if __name__ == '__main__':
    assert ref.available() and dais_ref.available(), 'oracle/_ref is not built'
    reference_checks()
    dais_reference()
