"""Store the reference's answers for sweeps (one matrix under many solver option sets) in sweep.json.gz.

For each matrix the file holds the matrix, its input intervals / latencies, the cost model, the option sets, and for
every candidate of every set (the decompose_dc tries of ``solve``, api.cc:176-201) the result of the reference call
``solve(W, method0, method1, hard_dc=H, decompose_dc=d, search_all_decompose_dc=False, ...)``: sha256 over the stage
arrays (the digest bench.py uses), the float32 cost summed over both stages in op order (api.cc:222-227), the latencies
of ``Pipeline.latency`` and the adder count.  Each set's winner index is checked against ``solve(W, **set)``.

The reference's latency-retry loop (api.cc:83-140) has no bound, so every reference call runs in its own process under
a time limit; a set with a call that fails or does not finish is left out of the family.

Needs oracle/_ref built from the reference sources (``make -C oracle REF=<reference checkout>``):

    python tests/golden/make_golden_sweep.py
"""

import gzip
import hashlib
import json
import multiprocessing as mp
import os
import sys
import time
from pathlib import Path

os.environ.setdefault('OMP_NUM_THREADS', '1')  # (one reference call per worker process)
import numpy as np  # noqa: E402

HERE = Path(__file__).resolve().parent
ROOT = HERE.parents[1]
sys.path[:0] = [str(ROOT)]

from oracle import ref  # noqa: E402

METHODS = ['mc', 'mc-dc', 'mc-pdc', 'wmc', 'wmc-dc', 'wmc-pdc', 'dummy']
HARD_DC = [-1, 0, 1, 2, 4, 7]
DECOMPOSE_DC = [-2, -1, 1]
TIME_LIMIT_S = 30.0
STAGE_KEYS = ['inp_shifts', 'out_idxs', 'out_shifts', 'out_negs', 'ops_i', 'ops_f']


def digest(stages) -> str:
    h = hashlib.sha256()
    for st in stages:
        for k in STAGE_KEYS:
            a = np.ascontiguousarray(st[k])
            h.update(k.encode())
            h.update(str(a.shape).encode())
            h.update(a.tobytes())
    return h.hexdigest()


def summary(stages) -> dict:
    cost = np.float32(0.0)
    for st in stages:  # api.cc:222-227: one float accumulator, op order
        for v in st['ops_f'][:, 4]:
            cost = np.float32(cost + v)
    last = stages[-1]
    lat = [float(last['ops_f'][i, 3]) for i in last['out_idxs']]  # Pipeline.latency (Python indexing of ops)
    return dict(sha256=digest(stages), cost=float(cost), latency=[min(lat), max(lat)], n_adders=int(sum(np.count_nonzero(st['ops_i'][:, 2] >= 0) for st in stages)))


def matrices():
    rng = np.random.default_rng(20261015)
    W16 = rng.integers(-128, 128, size=(16, 16)).astype(np.float32)
    q16 = np.stack([-(2.0 ** rng.integers(0, 8, 16)), 2.0 ** rng.integers(0, 8, 16) - 0.5, np.full(16, 0.5)], axis=1).astype(np.float32)
    q16[3] = (0.0, 0.0, 1.0)
    lat16 = rng.integers(0, 4, 16).astype(np.float32)
    W32 = rng.integers(-128, 128, size=(32, 32)).astype(np.float32)
    W64 = rng.integers(-128, 128, size=(64, 64)).astype(np.float32)
    return [
        dict(name='int8_16x16_hetero', kernel=W16, qintervals=q16, latencies=lat16, adder_size=-1, carry_size=-1, n_sets=42),
        dict(name='int8_32x32_add1_carry1', kernel=W32, qintervals=None, latencies=None, adder_size=1, carry_size=1, n_sets=42),
        dict(name='int8_64x64', kernel=W64, qintervals=None, latencies=None, adder_size=-1, carry_size=-1, n_sets=21),
    ]


def option_sets(n, offset):
    """Every selector for method0, method1 'auto' or explicit, and every hard_dc / decompose_dc / search_all value."""
    out = []
    for i in range(offset, offset + n):
        out.append(dict(method0=METHODS[i % 7], method1='auto' if i % 2 == 0 else METHODS[(i // 2) % 6], hard_dc=HARD_DC[(i // 7) % 6],
                        decompose_dc=DECOMPOSE_DC[i % 3], search_all_decompose_dc=(i // 3) % 2 == 0))
    return out


def candidates(n_in, s):
    """(H, d) of each decompose_dc try of set s (api.cc:176-201)."""
    if not s['search_all_decompose_dc']:
        return [(s['hard_dc'], s['decompose_dc'])]
    H = s['hard_dc'] if s['hard_dc'] >= 0 else 1000000000
    return [(H, d) for d in range(-1, min(H, int(np.ceil(np.log2(np.float32(n_in))))) + 1)]


def _worker(conn, m, kw):
    try:
        conn.send(('ok', summary(ref.solve(m['kernel'], qintervals=m['qintervals'], latencies=m['latencies'], adder_size=m['adder_size'], carry_size=m['carry_size'], **kw))))
    except Exception as e:  # noqa: BLE001
        conn.send(('error', str(e)))


def run_calls(m, calls):
    """Each call in its own forked process, one per CPU at a time; None for a call that fails or runs over the time
    limit."""
    ctx = mp.get_context('fork')
    res, todo, live = {}, list(calls), []
    while todo or live:
        while todo and len(live) < max(1, os.cpu_count() or 1):
            kw = todo.pop(0)
            a, b = ctx.Pipe(False)
            p = ctx.Process(target=_worker, args=(b, m, dict(kw)))
            p.start()
            live.append((kw, p, a, time.time()))
        time.sleep(0.01)
        for item in list(live):
            kw, p, a, t0 = item
            if a.poll():
                st, v = a.recv()
                res[kw] = v if st == 'ok' else None
                if st != 'ok':
                    print(m['name'], dict(kw), 'fails in the reference:', v)
            elif time.time() - t0 > TIME_LIMIT_S:
                p.kill()
                res[kw] = None
                print(m['name'], dict(kw), f'does not finish within {TIME_LIMIT_S:.0f} s in the reference')
            else:
                continue
            p.join()
            live.remove(item)
    return res


def main():
    t0 = time.time()
    out = []
    for mi, m in enumerate(matrices()):
        n_in = m['kernel'].shape[0]
        sets = option_sets(m['n_sets'], 11 * mi)
        calls = set()
        for s in sets:
            for H, d in candidates(n_in, s):
                calls.add(tuple(sorted(dict(method0=s['method0'], method1=s['method1'], hard_dc=H, decompose_dc=d, search_all_decompose_dc=False).items())))
            if s['search_all_decompose_dc']:
                calls.add(tuple(sorted(s.items())))
        res = run_calls(m, sorted(calls))
        kept = []
        for s in sets:
            cand_keys = [tuple(sorted(dict(method0=s['method0'], method1=s['method1'], hard_dc=H, decompose_dc=d, search_all_decompose_dc=False).items())) for H, d in candidates(n_in, s)]
            whole = tuple(sorted(s.items()))
            if any(res[k] is None for k in cand_keys) or (s['search_all_decompose_dc'] and res[whole] is None):
                print(m['name'], 'set left out:', s)
                continue
            cands = [dict(hard_dc=H, decompose_dc=d, **res[k]) for (H, d), k in zip(candidates(n_in, s), cand_keys, strict=True)]
            costs = [np.float32(c['cost']) for c in cands]
            win = int(np.argmin(costs))  # the first minimum (api.cc:243-249)
            if s['search_all_decompose_dc']:
                assert res[whole]['sha256'] == cands[win]['sha256'], (m['name'], s)
            kept.append(dict(options=s, candidates=cands, winner=win))
        out.append(dict(name=m['name'], kernel=m['kernel'].ravel().tolist(), shape=list(m['kernel'].shape),
                        qintervals=None if m['qintervals'] is None else m['qintervals'].tolist(), latencies=None if m['latencies'] is None else m['latencies'].tolist(),
                        adder_size=m['adder_size'], carry_size=m['carry_size'], sets=kept))
        print(m['name'], len(kept), 'sets,', sum(len(s['candidates']) for s in kept), 'candidates,', f'{time.time() - t0:.0f} s', flush=True)
    with open(HERE / 'sweep.json.gz', 'wb') as raw, gzip.GzipFile('sweep.json.gz', 'wb', fileobj=raw, mtime=0) as f:
        f.write(json.dumps(out, separators=(',', ':'), sort_keys=True).encode())
    print(f'sweep.json.gz written in {time.time() - t0:.0f} s')


if __name__ == '__main__':
    assert ref.available(), 'oracle/_ref is not built'
    main()
