"""Pipelined pricing on the GPU against the pure-Python ``emit`` path, on the same tasks: the bench's 256x256 int8 design
(seed 0, default solve), and the kept candidates of the BASELINE config 5 stand-in's ``solve_sweep_batch`` under the 42
option sets of dev_sweep_perf.py (five int6 layers, seeds 40-44), each at cutoffs 2, 3, 5 and 8, with and without retiming.

    python scripts/dev_pipeline_price_perf.py [--reps 3] [--out pipeline_price_perf.json]

GPU: ``price_pipelined`` (device time from the library's CUDA events, launches, wall time with a device synchronise on
both sides; the first call of each workload is a warm-up).  Python: ``emit._retrace`` + ``emit.to_pipeline`` (and
``emit.retime_pipeline``) per design and cutoff, wall time, once.  The answers of both are compared.  The card's name,
power limit and SM clock are read in the same run.
"""

import argparse
import json
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / 'scripts'))

import da4ml_b200._binary as B  # noqa: E402
from da4ml_b200 import emit  # noqa: E402
from da4ml_b200.types import minimal_kif_array  # noqa: E402
from dev_sweep_perf import HARD_DC, METHODS, card, int_matrix  # noqa: E402

CUTOFFS = [2.0, 3.0, 5.0, 8.0]
SHAPES = [(16, 64), (64, 64), (64, 32), (32, 32), (32, 5)]


def python_path(designs, retiming):
    """(status, stages, reg_bits) per (design, cutoff) through emit."""
    out = np.zeros((len(designs), len(CUTOFFS), 3), np.int64)
    for d, stages in enumerate(designs):
        for j, c in enumerate(CUTOFFS):
            try:
                comb = emit._retrace(stages, c, B.cost_add)
            except AssertionError:
                out[d, j] = (1, -1, -1)
                continue
            except NotImplementedError:
                out[d, j] = (2, -1, -1)
                continue
            split = emit.to_pipeline(comb, c, retiming=retiming)
            qi, _ = emit._qint_io(split[0])
            bits = int(minimal_kif_array(qi).sum()) + sum(int(minimal_kif_array(emit._qint_io(s)[1]).sum()) for s in split)
            out[d, j] = (0, len(split), bits)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    B.set_stream(torch.cuda.current_stream().cuda_stream)
    rows = [dict(card=card())]
    print(json.dumps(rows[0]), flush=True)
    big = [emit.as_stage(s) for s in B.solve_raw(int_matrix(256, 256, 8, 0)).stages]
    layers = [int_matrix(a_, b_, 6, 40 + i) for i, (a_, b_) in enumerate(SHAPES)]
    sets = [dict(method0=m, hard_dc=h) for m in METHODS for h in HARD_DC]
    sweeps = B.solve_sweep_batch(layers, sets)
    kept = [[emit.as_stage(s) for s in sw.raw(int(i)).stages] for sw in sweeps for i in np.flatnonzero(sw.candidates['kept'])]
    for name, designs in (('bench_256x256_int8', [big]), ('config5_sweep_kept', kept)):
        n_ops = sum(len(s['ops_i']) for d in designs for s in d)
        for rt in (False, True):
            B.price_pipelined(designs, CUTOFFS, retiming=rt)  # (warm-up)
            dev, wall, launches = [], [], 0
            for _ in range(a.reps):
                torch.cuda.synchronize()
                t = time.perf_counter()
                pr = B.price_pipelined(designs, CUTOFFS, retiming=rt)
                torch.cuda.synchronize()
                wall.append(time.perf_counter() - t)
                dev.append(pr.profile['device_ms'])
                launches = pr.profile['launches']
            t = time.perf_counter()
            ref = python_path(designs, rt)
            py = time.perf_counter() - t
            got = np.stack([pr.status, pr.stages, pr.reg_bits], axis=-1)
            row = dict(workload=name, designs=len(designs), ops=n_ops, cutoffs=CUTOFFS, retiming=rt, gpu_wall_s=[round(w, 5) for w in wall],
                       gpu_device_ms=[round(v, 4) for v in dev], launches=launches, python_wall_s=round(py, 3), equal=bool(np.array_equal(got, ref)),
                       ok_tasks=int((pr.status == 0).sum()), tasks=int(pr.status.size), stages=sorted(set(pr.stages[pr.status == 0].tolist())))  # fmt: skip
            rows.append(row)
            print(json.dumps(row), flush=True)
    rows.append(dict(card_after=card()))
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(rows, indent=1))


if __name__ == '__main__':
    main()
