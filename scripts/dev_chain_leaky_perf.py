"""chain_front with leaky ReLU activations against relu on the MLP of dev_chain_traced_perf.py (16 -> 64 -> 32 -> 32 ->
5, int6 / int8 weights, 10 option sets): leaky_relu(0.125) then quantize(1, 6, 2) between the layers, against relu(6, 2),
at cutoffs 0, 3 and 5; then ``price_pipelined(keep_split=True)`` of the cheapest leaky and the cheapest relu design at
cutoffs 2, 3, 5 and 8 (the cost of the mux's third operand in the split kernels).

    python scripts/dev_chain_leaky_perf.py [--out chain_leaky_perf.json]

Per layer: states, points, the sweep's device time, the host replay (``replay_ms``), the pricing call's device time and
the layer's wall time, each the median of ``--reps`` runs (default 5; configurations interleaved, after one warm-up
call); ``wall_ms_all`` keeps every run's total.  The card's name, power limit and SM clock are read in the same run.
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
from dev_chain_traced_perf import BITS, DIMS, Q0, SETS  # noqa: E402

RELU = [('relu', (0, 6, 2))] * (len(DIMS) - 2)
LEAKY = [[('leaky_relu', 0.125), ('quantize', (1, 6, 2))]] * (len(DIMS) - 2)
from dev_sweep_perf import card, int_matrix  # noqa: E402


def run(kernels, c, acts):
    marks = []

    def solver(*args, **kw):
        marks.append(time.perf_counter())
        return B.solve_sweep_batch(*args, **kw)

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    cf = B.chain_front(kernels, SETS, qintervals=[Q0] + [None] * (len(kernels) - 1), latency_cutoff=c, activations=acts, solver=solver)
    torch.cuda.synchronize()
    marks.append(time.perf_counter())
    rows = [dict(layer=k, states=layer['states'], points=layer['points'], sweep_device_ms=round(layer['device_ms'], 2), replay_ms=round(layer.get('replay_ms', 0.0), 2),
                 price_device_ms=round(layer.get('price_device_ms', 0.0), 2), wall_ms=round(1e3 * (marks[k + 1] - marks[k]), 2),
                 dropped_constant=layer.get('dropped_constant', 0)) for k, layer in enumerate(cf.profile['layers'])]  # fmt: skip
    return cf, dict(cutoff=c, leaky=acts is LEAKY, points=len(cf), total_wall_ms=round(1e3 * (marks[-1] - t0), 2), cheapest=float(cf.cost.min()), layers=rows)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--reps', type=int, default=5)
    a = ap.parse_args()
    kernels = [int_matrix(n, m, b, 90 + i) for i, (n, m, b) in enumerate(zip(DIMS[:-1], DIMS[1:], BITS))]
    res = dict(card=card(), dims=DIMS, bits=BITS, n_sets=len(SETS), runs=[], split=[])
    run(kernels, 0.0, LEAKY)  # warm-up
    best, runs = {}, {}
    for _ in range(a.reps):  # (interleaved: relu and leaky alternate within every round)
        for c in (0.0, 3.0, 5.0):
            for acts in (RELU, LEAKY):
                cf, r = run(kernels, c, acts)
                runs.setdefault((c, acts is LEAKY), []).append(r)
                if c == 5.0:
                    best['leaky' if acts is LEAKY else 'relu'] = cf.design(int(np.argmin(cf.cost)))
    med = lambda v: round(float(np.median(v)), 2)  # noqa: E731
    for (c, leaky), rs in runs.items():
        layers = [{key: (med([r['layers'][k][key] for r in rs]) if key.endswith('_ms') else rs[0]['layers'][k][key]) for key in rs[0]['layers'][k]}
                  for k in range(len(rs[0]['layers']))]  # fmt: skip
        r = dict(cutoff=c, leaky=leaky, points=rs[0]['points'], reps=len(rs), total_wall_ms=med([r['total_wall_ms'] for r in rs]),
                 wall_ms_all=[r['total_wall_ms'] for r in rs], cheapest=rs[0]['cheapest'], layers=layers)  # fmt: skip
        res['runs'].append(r)
        print(json.dumps(r), flush=True)
    cuts = [2.0, 3.0, 5.0, 8.0]
    for kind, d in best.items():
        B.price_pipelined([d], cuts, keep_split=True)  # warm-up
    for c in cuts:
        for kind, d in best.items():
            walls = []
            for _ in range(a.reps):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                pr = B.price_pipelined([d], c, keep_split=True)
                walls.append(1e3 * (time.perf_counter() - t0))
            r = dict(kind=kind, cutoff=c, status=int(pr.status[0, 0]), stages=int(pr.stages[0, 0]), reg_bits=int(pr.reg_bits[0, 0]), device_ms=round(pr.profile['device_ms'], 3),
                     launches=pr.profile['launches'], split_launches=pr.profile['split_launches'], wall_ms=med(walls))  # fmt: skip
            res['split'].append(r)
            print(json.dumps(r), flush=True)
    res['card_after'] = card()
    print(json.dumps(dict(card=res['card'], card_after=res['card_after'])))
    if a.out:
        Path(a.out).write_text(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
