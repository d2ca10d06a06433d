"""chain_front with and without activations on a realistic MLP: 16 -> 64 -> 32 -> 32 -> 5 with int6 / int8 weights,
relu(6, 2) and quantizers between the layers, 10 option sets, latency cutoffs 0, 3 and 5.

    python scripts/dev_chain_traced_perf.py [--out chain_traced_perf.json]

Per layer: the states (distinct problems), the points kept, the sweep's device time (the library's CUDA events), the
host interval replay (``replay_ms``), the pricing call's device time and the layer's wall time (from its sweep call to
the next layer's, with a device synchronise at both ends of the whole call).  Each configuration runs once after one
warm-up call.  The card's name, power limit and SM clock are read in the same run.
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
from dev_sweep_perf import card, int_matrix  # noqa: E402

DIMS = [16, 64, 32, 32, 5]
BITS = [8, 6, 6, 8]
SETS = [dict(method0=m, hard_dc=h) for m, h in (('wmc', -1), ('wmc', 0), ('wmc', 2), ('mc', -1), ('mc', 2), ('wmc-dc', 1), ('wmc-dc', 3), ('mc-dc', 2))] + \
    [dict(method0='wmc', seed=1), dict(method0='wmc', hard_dc=2, seed=2)]  # fmt: skip
ACTS = [('relu', (0, 6, 2)), ('quantize', (1, 7, 1)), ('relu', (0, 6, 2))]
Q0 = [(-8.0, 7.875, 0.125)] * DIMS[0]


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
    rows = []
    for k, layer in enumerate(cf.profile['layers']):
        rows.append(dict(layer=k, states=layer['states'], points=layer['points'], sweep_device_ms=round(layer['device_ms'], 2),
                         replay_ms=round(layer.get('replay_ms', 0.0), 2), price_device_ms=round(layer.get('price_device_ms', 0.0), 2),
                         wall_ms=round(1e3 * (marks[k + 1] - marks[k]), 2)))  # fmt: skip
    return dict(cutoff=c, activations=acts is not None, points=len(cf), total_wall_ms=round(1e3 * (marks[-1] - t0), 2), cheapest=float(cf.cost.min()),
                fastest=float(cf.latency.min()), layers=rows)  # fmt: skip


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    kernels = [int_matrix(n, m, b, 90 + i) for i, (n, m, b) in enumerate(zip(DIMS[:-1], DIMS[1:], BITS))]
    res = dict(card=card(), dims=DIMS, bits=BITS, n_sets=len(SETS), activations=ACTS, runs=[])
    run(kernels, 0.0, ACTS)  # warm-up
    for c in (0.0, 3.0, 5.0):
        for acts in (None, ACTS):
            r = run(kernels, c, acts)
            res['runs'].append(r)
            print(json.dumps(r), flush=True)
    res['card_after'] = card()
    print(json.dumps(dict(card=res['card'], card_after=res['card_after'])))
    if a.out:
        Path(a.out).write_text(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
