"""Model sweep cost on the GPU: the five layers of the BASELINE config 5 stand-in (shapes (16,64), (64,64), (64,32),
(32,32), (32,5), int6, seeds 40-44, as in tests/test_cmvm_gpu.py::test_dense_stack_batch_vs_checker) under the 42 option
sets of dev_sweep_perf.py, three ways, alternating in one run: one solve_sweep_batch call, five solve_sweep calls (one per
layer), and the 210 solve calls.  Then the network front of the batch and its best design at a few latency budgets.

    python scripts/dev_sweep_batch_perf.py [--reps 3] [--out sweep_batch_perf.json]
    python -m torch.distributed.run --nproc-per-node=2 scripts/dev_sweep_batch_perf.py   # ... and sweep_sharded over the GPUs

Wall times are taken with a device synchronise on both sides.  The card's name, power limit and SM clock are read in the
same run.
"""

import argparse
import json
import os
import sys
import time
from pathlib import Path

import numpy as np
import torch

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / 'scripts'))

import da4ml_b200._binary as B  # noqa: E402
from da4ml_b200.cmvm import network_front  # noqa: E402
from dev_sweep_perf import HARD_DC, METHODS, card, int_matrix  # noqa: E402

SHAPES = [(16, 64), (64, 64), (64, 32), (32, 32), (32, 5)]


def timed(f):
    torch.cuda.synchronize()
    t = time.perf_counter()
    r = f()
    torch.cuda.synchronize()
    return r, time.perf_counter() - t


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    world = int(os.environ.get('WORLD_SIZE', '1'))
    rank = int(os.environ.get('RANK', '0'))
    if world > 1:
        import torch.distributed as dist

        torch.cuda.set_device(int(os.environ['LOCAL_RANK']))
        dist.init_process_group('nccl')
    B.set_stream(torch.cuda.current_stream().cuda_stream)
    layers = [int_matrix(a_, b_, 6, 40 + i) for i, (a_, b_) in enumerate(SHAPES)]
    sets = [dict(method0=m, hard_dc=h) for m in METHODS for h in HARD_DC]
    B.solve_raw(int_matrix(16, 16, 8, 1))  # (warm: device set up, buffers grown)
    B.solve_sweep_batch(layers, sets)
    rows = [dict(card=card(), rank=rank, world=world)]
    say = (lambda r: print(json.dumps(r), flush=True)) if rank == 0 else (lambda r: None)
    say(rows[0])
    batch = None
    for rep in range(a.reps):
        batch, w_batch = timed(lambda: B.solve_sweep_batch(layers, sets))
        per, w_per = timed(lambda: [B.solve_sweep(W, sets) for W in layers])
        calls, w_calls = timed(lambda: [B.solve_raw(W, **s) for W in layers for s in sets])
        for x, y in zip(batch, per, strict=True):  # (the same candidates either way)
            assert np.array_equal(x.candidates['cost'], y.candidates['cost']) and np.array_equal(x.winners, y.winners)
        p0 = batch[0].profile
        row = dict(
            rep=rep,
            sets=len(sets),
            candidates=sum(len(r) for r in batch),
            candidates_solved=sum(r.n_solved for r in batch),
            batch=dict(wall_s=w_batch, device_ms=p0['device_ms'], launches=p0['launches'], jobs_total=p0['jobs_total'], jobs_run=p0['jobs_run']),
            per_layer_sweeps=dict(wall_s=w_per, device_ms=sum(r.profile['device_ms'] for r in per), launches=sum(r.profile['launches'] for r in per),
                                  jobs_total=sum(r.profile['jobs_total'] for r in per), jobs_run=sum(r.profile['jobs_run'] for r in per)),
            solve_calls=dict(n=len(calls), wall_s=w_calls, device_ms=sum(r.device_ms for r in calls), launches=sum(r.launches for r in calls),
                             jobs_total=sum(r.profile['jobs_total'] for r in calls), jobs_run=sum(r.profile['jobs_run'] for r in calls)),
        )
        rows.append(row)
        say(row)
    nf = network_front(batch)
    default = [r.winners[sets.index(dict(method0='wmc', hard_dc=-1))] for r in batch]  # solve()'s defaults, layer by layer
    d_cost, d_lat = np.float32(0), np.float32(0)
    for r, i in zip(batch, default):
        d_cost, d_lat = np.float32(d_cost + r.candidates['cost'][i]), np.float32(d_lat + r.candidates['latency_max'][i])
    budgets = sorted({float(nf.latency[0]), float(np.median(nf.latency)), float(d_lat), float(nf.latency[-1])})
    best = {}
    for b in budgets:
        p = nf.best(b)
        best[b] = dict(cost=p.cost, latency=p.latency, layers=[dict(options=sets[int(r.candidates['set'][i])], H=int(r.candidates['hard_dc'][i]),
                                                                    d=int(r.candidates['decompose_dc_start'][i]), n_adders=int(r.candidates['n_adders'][i]))
                                                               for r, i in zip(batch, p.choice)])
    front = dict(default_chain=dict(cost=float(d_cost), latency=float(d_lat)), points=[dict(cost=float(c), latency=float(l)) for c, l in zip(nf.cost, nf.latency)],
                 best=best)
    rows.append(front)
    say(front)
    if world > 1:
        from da4ml_b200.distributed import sweep_sharded

        for rep in range(a.reps):
            dist.barrier()
            got, w = timed(lambda: sweep_sharded(layers, sets))
            dist.barrier()
            for x, y in zip(got, batch, strict=True):
                assert np.array_equal(x.candidates['cost'], y.candidates['cost'])
            row = dict(rep=rep, sweep_sharded=dict(world=world, wall_s=w))
            rows.append(row)
            say(row)
    else:
        rows.append(dict(sweep_sharded='not measured: one process (run under torch.distributed.run on two or more GPUs)'))
        say(rows[-1])
    rows.append(dict(card_after=card()))
    say(rows[-1])
    if a.out and rank == 0:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(rows, indent=1))
    if world > 1:
        dist.destroy_process_group()


if __name__ == '__main__':
    main()
