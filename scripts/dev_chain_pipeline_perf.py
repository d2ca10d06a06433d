"""A whole chain priced and split as one pipeline on the GPU (``price_pipelined(chain_design(...), ..., keep_split=True)``):
the five layers of the BASELINE config 5 stand-in (dev_pipeline_price_perf.py's shapes, int6, default solves) with a
relu quantizer between consecutive layers, at cutoffs 2, 3, 5 and 8, with and without retiming.

    python scripts/dev_chain_pipeline_perf.py [--reps 3] [--out chain_pipeline_perf.json]

GPU: device time from the library's CUDA events, launches and wall time with a device synchronise on both sides; the
first call is a warm-up.  This library has no Python path for chains (``emit`` re-traces adder graphs only), so the
comparison is the CPU build of the same kernels and host code under the SIMT shim (tests/simt, 128 threads per CTA),
timed once; every answer (status, stages, register bits, latencies, cutoffs and the split, bit for bit) must be equal.
The card's name, power limit and SM clock are read in the same run.
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
sys.path.insert(0, str(ROOT / 'tests'))

import da4ml_b200._binary as B  # noqa: E402
from dev_pipeline_price_perf import CUTOFFS, SHAPES  # noqa: E402
from dev_sweep_perf import card, int_matrix  # noqa: E402
from simt import pipeline_split as SIM  # noqa: E402


def same(a, b) -> bool:
    for key in ('status', 'stages', 'reg_bits'):
        if not np.array_equal(getattr(a, key), getattr(b, key)):
            return False
    for key in ('latency_max', 'cutoff'):
        if not np.array_equal(getattr(a, key), getattr(b, key), equal_nan=True):
            return False
    for j in range(len(a.cutoffs)):
        if int(a.status[0, j]) != 0:
            continue
        try:
            x, y = a.split(0, j), b.split(0, j)
        except ValueError:
            continue
        if len(x) != len(y):
            return False
        for s, t in zip(x, y):
            if not all(np.array_equal(np.asarray(s[k], np.int64), np.asarray(t[k], np.int64)) for k in ('out_idxs', 'out_shifts', 'out_negs', 'ops_i')):
                return False
            if not np.array_equal(s['ops_f'].view(np.uint64), t['ops_f'].view(np.uint64)):
                return False
    return True


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    layers = [B.solve_raw(int_matrix(n, m, 6, 40 + i)) for i, (n, m) in enumerate(SHAPES)]
    acts = [('relu', (0, 8, 0))] * (len(layers) - 1)
    design = B.chain_design(layers, acts)
    n_act = sum(int(np.isin(st['ops_i'][:, 2], (2, 3)).sum()) for st in design.stages)
    res = dict(card=card(), layers=SHAPES, cutoffs=CUTOFFS, activation_ops=n_act, runs=[])
    for rt in (False, True):
        B.price_pipelined([design], CUTOFFS, retiming=rt, keep_split=True)  # warm-up
        walls, dev, launches = [], [], 0
        for _ in range(a.reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            pr = B.price_pipelined([design], CUTOFFS, retiming=rt, keep_split=True)
            for j in range(len(CUTOFFS)):
                if int(pr.status[0, j]) == 0:
                    try:
                        pr.split(0, j)
                    except ValueError:
                        pass
            torch.cuda.synchronize()
            walls.append(1e3 * (time.perf_counter() - t0))
            dev.append(pr.profile['device_ms'])
            launches = pr.profile['launches'] + pr.profile.get('split_launches', 0)
        t0 = time.perf_counter()
        sim = SIM.split([design], CUTOFFS, retiming=rt, threads=128)
        sim_ms = 1e3 * (time.perf_counter() - t0)
        res['runs'].append(dict(retiming=rt, wall_ms=walls, device_ms=dev, launches=launches, cpu_sim_ms=sim_ms, equal=same(pr, sim),
                                status=pr.status[0].tolist(), stages=pr.stages[0].tolist(), reg_bits=pr.reg_bits[0].tolist(),
                                latency_max=pr.latency_max[0].tolist(), cutoff=pr.cutoff[0].tolist()))  # fmt: skip
        print(json.dumps(res['runs'][-1]), flush=True)
    res['card_after'] = card()
    print(json.dumps(dict(card=res['card'], card_after=res['card_after'], activation_ops=n_act)))
    if a.out:
        Path(a.out).write_text(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
