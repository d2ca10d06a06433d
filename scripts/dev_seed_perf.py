"""What seeded tie-breaks buy and cost on the GPU.

    python scripts/dev_seed_perf.py [--parent DIR] [--bench-reps 3] [--out seed_perf.json]

1. Bench unchanged: ``bench.py --gpus 1 --steps 3 --warmup 3`` of this tree alternated with the parent build in DIR (a
   built checkout of the parent commit), ``--bench-reps`` times each; the JSON line of every run is reported.
2. Seeds' gain: ``solve_best_of`` with N = 1, 4, 16, 64 seeds of the default options on a 64x64 int8 matrix, a 128x128
   int6 one (the config-4 shape) and the five config-5 stand-in layers of dev_sweep_batch_perf.py: adders of seed 0 and
   of the best seed, which seed, the float32 cost, wall time (with a device synchronise) and device time of the call.
3. Seeds on the chain front: ``chain_front`` of the five layers under the 42 sets of dev_sweep_perf.py, and under the
   same sets with seeds 0-3 each (168 sets); the front at budgets 36 / 45 / 54, wall and device time.

The card's name, power limit and SM clock are read in the same run.
"""

import argparse
import json
import os
import subprocess
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / 'scripts'))

import da4ml_b200._binary as B  # noqa: E402
from da4ml_b200.cmvm import chain_front  # noqa: E402
from dev_sweep_batch_perf import SHAPES, timed  # noqa: E402
from dev_sweep_perf import HARD_DC, METHODS, card, int_matrix  # noqa: E402

BUDGETS = [36, 45, 54]
N_SEEDS = [1, 4, 16, 64]


def bench(tree: Path):
    env = {k: v for k, v in os.environ.items() if k != 'PYTHONPATH'}
    r = subprocess.run([sys.executable, 'bench.py', '--gpus', '1', '--steps', '3', '--warmup', '3'], cwd=tree, capture_output=True, text=True, env=env, timeout=3000)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith('{')]
    return json.loads(lines[-1]) if lines else dict(error=r.stderr[-2000:], rc=r.returncode)


def best_of_rows(name, W):
    rows = []
    a0 = B.solve_raw(W).n_adders
    for n in N_SEEDS:
        (raw, s), wall = timed(lambda: B.solve_best_of_raw(W, n_seeds=n))
        c = np.float32(0)
        for st in raw.stages:
            for v in st['ops_f'][:, 4]:
                c = np.float32(c + v)
        rows.append(dict(matrix=name, n_seeds=n, adders_seed0=a0, adders_best=raw.n_adders, best_seed=s, cost=float(c), wall_s=wall,
                         device_ms=raw.profile['device_ms'], launches=raw.profile['launches'], jobs_run=raw.profile['jobs_run']))  # fmt: skip
        print(json.dumps(rows[-1]), flush=True)
    return rows


def front_rows(cf):
    out = dict(front=[dict(cost=float(c), latency=float(l)) for c, l in zip(cf.cost, cf.latency)], best={})
    for b in BUDGETS:
        try:
            p = cf.best(b)
            out['best'][b] = dict(cost=p.cost, latency=p.latency)
        except ValueError as e:
            out['best'][b] = str(e)
    return out


def main():
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument('--parent', default=None)
    ap.add_argument('--bench-reps', type=int, default=3)
    ap.add_argument('--bench-only', action='store_true', help='only part 1')
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    rows = [dict(card=card())]
    print(json.dumps(rows[0]), flush=True)
    if a.parent:
        for rep in range(a.bench_reps):
            for tag, tree in (('parent', Path(a.parent)), ('this', ROOT)):
                rows.append(dict(bench=tag, rep=rep, line=bench(tree)))
                print(json.dumps(rows[-1]), flush=True)
    if a.bench_only:
        rows.append(dict(card_after=card()))
        print(json.dumps(rows[-1]), flush=True)
        if a.out:
            Path(a.out).parent.mkdir(parents=True, exist_ok=True)
            Path(a.out).write_text(json.dumps(rows, indent=1))
        return
    B.set_stream(torch.cuda.current_stream().cuda_stream)
    B.solve_raw(int_matrix(16, 16, 8, 1))  # (warm: device set up, buffers grown)
    mats = [('64x64 int8', np.random.default_rng(0).integers(-128, 128, (64, 64)).astype(np.float32)), ('128x128 int6', int_matrix(128, 128, 6, 0))]
    mats += [(f'layer {i} {m}x{n} int6', int_matrix(m, n, 6, 40 + i)) for i, (m, n) in enumerate(SHAPES)]
    for name, W in mats:
        rows += best_of_rows(name, W)
    layers = [int_matrix(m, n, 6, 40 + i) for i, (m, n) in enumerate(SHAPES)]
    sets = [dict(method0=m, hard_dc=h) for m in METHODS for h in HARD_DC]
    for tag, ss in (('42 sets', sets), ('42 sets x seeds 0-3', [{**s, 'seed': k} for s in sets for k in range(4)])):
        cf, wall = timed(lambda: chain_front(layers, ss))
        row = dict(chain=tag, sets=len(ss), wall_s=wall, **{k: cf.profile[k] for k in ('launches', 'device_ms', 'jobs_run', 'jobs_total')}, **front_rows(cf))
        rows.append(row)
        print(json.dumps(row), flush=True)
    rows.append(dict(card_after=card()))
    print(json.dumps(rows[-1]), flush=True)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(rows, indent=1))


if __name__ == '__main__':
    main()
