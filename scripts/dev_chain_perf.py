"""Chain search cost on the GPU, and how far the exact chain latency falls below network_front's bound: the five layers of
the config-5 stand-in of dev_sweep_batch_perf.py (int6, seeds 40-44) under the 42 option sets of dev_sweep_perf.py.

    python scripts/dev_chain_perf.py [--reps 2] [--out chain_perf.json]

Each repetition runs one chain_front call and one solve_sweep_batch call + network_front, alternating, wall times with a
device synchronise.  Reported: per layer the input-latency states, candidates, points kept, launches and device time;
the exact chain front next to network_front's (summed latency_max); best(b) of both at budgets 36, 45 and 54, with the
latency and cost the network_front choice really has when each layer is solved under the previous one's output
latencies (as a traced model solves it); and the default solve of every layer, both ways.  The card's name, power limit
and SM clock are read in the same run.
"""

import argparse
import json
import sys
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / 'scripts'))

import da4ml_b200._binary as B  # noqa: E402
from da4ml_b200.cmvm import chain_front, network_front  # noqa: E402
from dev_sweep_batch_perf import SHAPES, timed  # noqa: E402
from dev_sweep_perf import HARD_DC, METHODS, card, int_matrix  # noqa: E402

BUDGETS = [36, 45, 54]


def cost_of(raw):
    c = np.float32(0)
    for st in raw.stages:
        for v in st['ops_f'][:, 4]:
            c = np.float32(c + v)
    return c


def traced(layers, calls):
    """Solve layer k with ``calls[k]`` under the output latencies of layer k - 1's result: (cost, latency) of the chain."""
    lat, cost = None, np.float32(0)
    for W, kw in zip(layers, calls):
        raw = B.solve_raw(W, **{**kw, 'latencies': None if lat is None else [float(v) for v in lat]})
        cost, lat = np.float32(cost + cost_of(raw)), np.asarray(raw.to_pipeline().out_latencies, np.float32)
    return float(cost), float(lat.max())


def main():
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=2)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    B.set_stream(torch.cuda.current_stream().cuda_stream)
    layers = [int_matrix(a_, b_, 6, 40 + i) for i, (a_, b_) in enumerate(SHAPES)]
    sets = [dict(method0=m, hard_dc=h) for m in METHODS for h in HARD_DC]
    rows = [dict(card=card(), sets=len(sets), shapes=SHAPES)]
    print(json.dumps(rows[0]), flush=True)
    B.solve_raw(int_matrix(16, 16, 8, 1))  # (warm: device set up, buffers grown)
    B.solve_sweep_batch(layers, sets)
    cf = nf = sweeps = None
    for rep in range(a.reps):
        cf, w_chain = timed(lambda: chain_front(layers, sets))
        sweeps, w_batch = timed(lambda: B.solve_sweep_batch(layers, sets))
        nf = network_front(sweeps)
        row = dict(rep=rep, chain_front=dict(wall_s=w_chain, **{k: cf.profile[k] for k in ('launches', 'device_ms', 'jobs_run', 'jobs_total')}, layers=cf.profile['layers']),
                   sweep_batch=dict(wall_s=w_batch, launches=sweeps[0].profile['launches'], device_ms=sweeps[0].profile['device_ms']))
        rows.append(row)
        print(json.dumps(row), flush=True)
    best = {}
    for b in BUDGETS:
        entry = {}
        try:
            p = cf.best(b)
            i = [float(v) for v in cf.latency].index(p.latency)
            entry['chain'] = dict(cost=p.cost, latency=p.latency, layers=[{k: v for k, v in c.items() if k in ('method0', 'method1', 'hard_dc', 'decompose_dc')} for c in cf.reference_calls(i)])
        except ValueError as e:
            entry['chain'] = str(e)
        try:
            p = nf.best(b)
            calls = [sw.reference_call(i) for sw, i in zip(sweeps, p.choice)]
            t_cost, t_lat = traced(layers, calls)
            entry['network_front'] = dict(cost=p.cost, summed_latency=p.latency, traced_cost=t_cost, traced_latency=t_lat,
                                          layers=[{k: v for k, v in c.items() if k in ('method0', 'method1', 'hard_dc', 'decompose_dc')} for c in calls])
        except ValueError as e:
            entry['network_front'] = str(e)
        best[b] = entry
    default_sum = [np.float32(0), np.float32(0)]
    for W in layers:
        raw = B.solve_raw(W)
        default_sum = [np.float32(default_sum[0] + cost_of(raw)), np.float32(default_sum[1] + raw.to_pipeline().latency[1])]  # (latency_max, as network_front)
    d_cost, d_lat = traced(layers, [{}] * len(layers))
    front = dict(chain=[dict(cost=float(c), latency=float(l)) for c, l in zip(cf.cost, cf.latency)],
                 network_front=[dict(cost=float(c), latency=float(l)) for c, l in zip(nf.cost, nf.latency)], best=best,
                 default=dict(summed=dict(cost=float(default_sum[0]), latency=float(default_sum[1])), traced=dict(cost=d_cost, latency=d_lat)))
    rows.append(front)
    print(json.dumps(front), flush=True)
    rows.append(dict(card_after=card()))
    print(json.dumps(rows[-1]), flush=True)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(rows, indent=1))


if __name__ == '__main__':
    main()
