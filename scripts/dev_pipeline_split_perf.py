"""Register stages of designs on the GPU (``price_pipelined(..., keep_split=True)``) against ``keep_split=False`` and the
pure-Python ``emit`` path, on the workloads of dev_pipeline_price_perf.py: the bench's 256x256 int8 design (seed 0,
default solve), and the kept candidates of the BASELINE config 5 stand-in's ``solve_sweep_batch`` under the 42 option
sets of dev_sweep_perf.py, each at cutoffs 2, 3, 5 and 8, with and without retiming.

    python scripts/dev_pipeline_split_perf.py [--reps 3] [--out pipeline_split_perf.json]

GPU (both settings of ``keep_split``): device time from the library's CUDA events, launches, wall time with a device
synchronise on both sides, and the bytes of op tables copied back; the first call of each workload is a warm-up.
Python: ``emit._retrace`` + ``emit.to_pipeline(..., retiming)`` per design and cutoff, wall time, once.  Every split is
compared with the Python path's, array for array and bit for bit.  The card's name, power limit and SM clock are read
in the same run.
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
from dev_pipeline_price_perf import CUTOFFS, SHAPES  # noqa: E402
from dev_sweep_perf import HARD_DC, METHODS, card, int_matrix  # noqa: E402


def python_path(designs, retiming):
    """emit's split per (design, cutoff) (None where the tracer refuses the cutoff)."""
    out = []
    for stages in designs:
        row = []
        for c in CUTOFFS:
            try:
                comb = emit._retrace(stages, c, B.cost_add)
            except (AssertionError, NotImplementedError):
                row.append(None)
                continue
            row.append(emit.to_pipeline(comb, c, retiming=retiming))
        out.append(row)
    return out


def same(a, b) -> bool:
    if len(a) != len(b):
        return False
    for x, y in zip(a, b):
        if tuple(x['shape']) != tuple(y['shape']) or not np.array_equal(x['ops_f'].view(np.uint64), np.asarray(y['ops_f'], np.float64).view(np.uint64)):
            return False
        if not all(np.array_equal(np.asarray(x[k], np.int64), np.asarray(y[k], np.int64)) for k in ('out_idxs', 'out_shifts', 'out_negs', 'ops_i')):
            return False
    return True


def timed(designs, rt, keep, reps):
    B.price_pipelined(designs, CUTOFFS, retiming=rt, keep_split=keep)  # (warm-up)
    dev, wall = [], []
    for _ in range(reps):
        torch.cuda.synchronize()
        t = time.perf_counter()
        pr = B.price_pipelined(designs, CUTOFFS, retiming=rt, keep_split=keep)
        torch.cuda.synchronize()
        wall.append(time.perf_counter() - t)
        dev.append(pr.profile['device_ms'])
    return pr, dict(wall_ms=[round(1e3 * w, 2) for w in wall], device_ms=[round(v, 3) for v in dev], launches=pr.profile['launches'],
                    bytes_back=pr.profile.get('split_bytes', 0))  # fmt: skip


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
        for rt in (False, True):
            _, price = timed(designs, rt, False, a.reps)
            pr, split = timed(designs, rt, True, a.reps)
            t = time.perf_counter()
            ref = python_path(designs, rt)
            py = time.perf_counter() - t
            n_eq = n_split = 0
            for d in range(len(designs)):
                for j in range(len(CUTOFFS)):
                    if int(pr.status[d, j]) != 0:
                        n_eq += ref[d][j] is None
                        continue
                    n_split += 1
                    n_eq += ref[d][j] is not None and same(pr.split(d, j), ref[d][j])
            rows_ = sum(len(s['ops_i']) for d in range(len(designs)) for j in range(len(CUTOFFS)) if int(pr.status[d, j]) == 0 for s in pr.split(d, j))
            row = dict(workload=name, designs=len(designs), cutoffs=CUTOFFS, retiming=rt, tasks=int(pr.status.size), splits=n_split, split_rows=rows_,
                       keep_split=split, price_only=price, python_wall_s=round(py, 3), equal=n_eq == pr.status.size)  # fmt: skip
            rows.append(row)
            print(json.dumps(row), flush=True)
    rows.append(dict(card_after=card()))
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(rows, indent=1))


if __name__ == '__main__':
    main()
