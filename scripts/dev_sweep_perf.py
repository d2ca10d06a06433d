"""Sweep cost on the GPU: one matrix under method0 x hard_dc option sets in one solve_sweep call, against the same sets
solved one solve call at a time, and the resulting cost / latency front next to the default solve.

    python scripts/dev_sweep_perf.py [--out sweep_perf.json]

Workloads: the bench matrix (256x256 int8, seed 0), one 128x128 int6 matrix of config 4 (seed 0) and one 64x64 int8
matrix (seed 0).  Sets: method0 in {wmc, wmc-dc, wmc-pdc, mc, mc-dc, mc-pdc} x hard_dc in {-1, 0, 1, 2, 3, 4, 6}, with the
decompose_dc search on.  The card's name, power limit and SM clock are read in the same run.
"""

import argparse
import json
import subprocess
import sys
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))

import da4ml_b200._binary as B  # noqa: E402

METHODS = ['wmc', 'wmc-dc', 'wmc-pdc', 'mc', 'mc-dc', 'mc-pdc']
HARD_DC = [-1, 0, 1, 2, 3, 4, 6]


def int_matrix(n_in, n_out, bits, seed):
    rng = np.random.default_rng(seed)
    return rng.integers(-(2 ** (bits - 1)), 2 ** (bits - 1), size=(n_in, n_out)).astype(np.float32)


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:  # (reading only)
        return f'nvidia-smi unavailable: {e}'


def device_bytes():
    import torch

    free, total = torch.cuda.mem_get_info()
    return total - free


def run(name, W):
    sets = [dict(method0=m, hard_dc=h) for m in METHODS for h in HARD_DC]
    B.solve_raw(int_matrix(16, 16, 8, 1))  # (warm: device set up, buffers grown)
    before = device_bytes()
    t = time.perf_counter()
    res = B.solve_sweep(W, sets)
    wall = time.perf_counter() - t
    held = device_bytes()
    t = time.perf_counter()
    one_ms, one_launches = 0.0, 0
    for s in sets:
        r = B.solve_raw(W, **s)
        one_ms += r.device_ms
        one_launches += r.launches
    one_wall = time.perf_counter() - t
    default = B.solve_raw(W)
    c = res.candidates
    dflt_cost = float(np.float32(sum(np.float32(v) for st in default.stages for v in st['ops_f'][:, 4])))
    front = sorted(((float(c['cost'][i]), float(c['latency_max'][i]), int(c['n_adders'][i]), sets[c['set'][i]], int(c['hard_dc'][i]), int(c['decompose_dc_start'][i]))
                    for i in res.front), key=lambda x: x[1])
    out = dict(
        workload=name,
        sets=len(sets),
        candidates=len(res),
        candidates_solved=res.n_solved,
        sweep_wall_s=wall,
        sweep_device_ms=res.profile['device_ms'],
        sweep_launches=res.profile['launches'],
        jobs_total=res.profile['jobs_total'],
        jobs_run=res.profile['jobs_run'],
        device_bytes_before=before,
        device_bytes_after=held,
        one_at_a_time_wall_s=one_wall,
        one_at_a_time_device_ms=one_ms,
        one_at_a_time_launches=one_launches,
        default=dict(cost=dflt_cost, latency=list(default.to_pipeline().latency), n_adders=default.n_adders),
        front=[dict(cost=f[0], latency_max=f[1], n_adders=f[2], options=f[3], H=f[4], d=f[5]) for f in front],
    )
    print(json.dumps(out), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    rows = [dict(card=card())]
    print(json.dumps(rows[0]), flush=True)
    for name, W in (('256x256 int8 seed 0', int_matrix(256, 256, 8, 0)), ('128x128 int6 seed 0', int_matrix(128, 128, 6, 0)), ('64x64 int8 seed 0', int_matrix(64, 64, 8, 0))):
        rows.append(run(name, W))
    rows.append(dict(card_after=card()))
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(rows, indent=1))


if __name__ == '__main__':
    main()
