"""Golden splits for ``price_pipelined(..., keep_split=True).split(d, j)`` from the reference's OWN tracer: the designs and
tasks of make_golden_pipeline_price.py (and one more latency set per design: every input at 6.5), plus the hand-made
designs of ``_extra_designs`` under their own latencies (stored in ``designs``, numbered after those of
pipeline_price.json.gz), each design replayed
on ``FixedVariable`` inputs at the task's latencies under ``HWConfig(adder_size, carry_size, cutoff)``, gathered with
``trace.comb_trace`` and split with ``trace/pipeline.py::to_pipeline(retiming=False)``; the retimed split is what
``retime_pipeline`` keeps.

Per task: the status (as in pipeline_price.json.gz), and per split (``split``: without retiming, ``retimed``) its stage
count, per-stage (n_in, n_out, n_ops), the sha256 of ``split_bytes`` and, for splits of at most ``FULL_ROWS`` rows, the
full stage arrays (``ops_f`` as float64 bits).  ``split`` is null where the reference's ``to_pipeline`` raises
KeyError.  ``interleaved``: the task's gather order by ``latency * N + i`` differs from the order by (latency, i).

Container only: imports /root/reference/src/da4ml through tests/ref_trace.py, as make_golden_pipeline_price.py does.
Writes tests/golden/pipeline_split.json.gz; running it again rewrites the same bytes.
"""
import gzip
import hashlib
import importlib
import json
import sys
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parents[1]))
sys.path.insert(0, str(HERE.parent))
sys.path.insert(0, str(HERE))

FULL_ROWS = 100
KEYS = ('inp_shifts', 'out_idxs', 'out_shifts', 'out_negs')


def split_bytes(stages) -> bytes:
    """Fixed byte layout of a split (little-endian): per stage int64 (n_in, n_out, n_ops, adder_size, carry_size),
    inp_shifts, out_idxs, out_shifts, out_negs (int64), ops_i (int64 [n,4]) and ops_f (float64 [n,5]), row-major."""
    out = []
    for st in stages:
        oi = np.asarray(st['ops_i'], '<i8').reshape(-1, 4)
        out.append(np.asarray([st['shape'][0], st['shape'][1], len(oi), st['adder_size'], st['carry_size']], '<i8').tobytes())
        out += [np.asarray(st[k], np.int64).astype('<i8').tobytes() for k in KEYS]
        out += [oi.tobytes(), np.asarray(st['ops_f'], '<f8').reshape(-1, 5).tobytes()]
    return b''.join(out)


def record(stages) -> dict:
    rows = sum(len(st['ops_i']) for st in stages)
    rec = {'stages': len(stages), 'meta': [[int(st['shape'][0]), int(st['shape'][1]), len(st['ops_i'])] for st in stages],
           'sha256': hashlib.sha256(split_bytes(stages)).hexdigest()}  # fmt: skip
    if rows <= FULL_ROWS:
        rec['full'] = [{k: np.asarray(st[k], np.int64).tolist() for k in KEYS} | {'ops_i': np.asarray(st['ops_i'], np.int64).tolist(),
                                                                                  'ops_f_bits': np.asarray(st['ops_f'], np.float64).view(np.uint64).tolist()}
                       for st in stages]  # fmt: skip
    return rec


def _stage(n_in, ops, out_idxs, out_negs=None):
    """One stage dict from [(id0, id1, opcode, data, (lo, hi, step))] (latency and cost 0: the tracer recomputes them)."""
    return dict(inp_shifts=[0] * n_in, out_idxs=list(out_idxs), out_shifts=[0] * len(out_idxs), out_negs=out_negs or [0] * len(out_idxs),
                ops_i=np.asarray([o[:4] for o in ops], np.int64).reshape(-1, 4), ops_f=np.asarray([[*o[4], 0.0, 0.0] for o in ops], np.float32).reshape(-1, 5),
                adder_size=-1, carry_size=-1)  # fmt: skip


def _extra_designs():
    """Designs whose outputs read inputs directly next to inputs nothing reads: under late input latencies
    dead_statement_elimination keeps an unread input (a kept input op marks the op at the position of its input number),
    which can land in a stage after the last output's, where to_pipeline raises KeyError.  (name, stages, latency sets,
    cutoffs)."""
    q0, q1, q2 = (-8.0, 7.5, 0.5), (0.0, 15.0, 1.0), (-4.0, 3.75, 0.25)
    return [
        ('inputs_out_3', [_stage(3, [(0, -1, -1, 0, q0), (1, -1, -1, 0, q1), (2, -1, -1, 0, q2)], [2])], [None, [10.0, 10.0, 0.0], [0.0, 10.0, 0.0], [1.0, 0.0, 3.0]],
         [1.0, 2.0, 4.0, 40.0]),
        ('inputs_out_4', [_stage(4, [(k, -1, -1, 0, (q0, q1, q2, q0)[k]) for k in range(4)], [2, 3])], [None, [3.0, 3.0, 0.0, 0.0], [0.0, 3.0, 0.0, 0.5]],
         [1.0, 2.0, 5.0]),
        ('adder_and_input_out', [_stage(4, [(0, -1, -1, 0, q0), (1, -1, -1, 0, q1), (2, -1, -1, 0, q2), (3, -1, -1, 0, q1), (0, 1, 0, 1, (-16.0, 37.0, 0.5))], [4, 3], [0, 1])],
         [None, [0.0, 0.0, 9.0, 0.0], [0.0, 0.0, 0.0, 9.0], [5.0, 0.0, 9.0, 0.0]], [2.0, 3.0, 5.0, 20.0]),
        ('point_input_unread', [_stage(3, [(1, -1, -1, 0, q0), (2, -1, -1, 0, q1)], [0, 1])], [None, [4.0, 0.0, 0.0], [0.0, 0.0, 4.0]], [1.0, 2.0, 8.0]),
    ]  # fmt: skip


def main():
    import ref_trace
    from make_golden_pipeline_price import CUTOFFS, _designs, _lat_sets

    from da4ml_b200 import emit
    from da4ml_b200._binary import cost_add as abi_cost_add
    from da4ml_b200.types import pipeline_from_arrays

    from oracle import port

    T, trace = ref_trace.load(None, port.get_lsb_loc, port.iceil_log2, port.cost_add)
    P = importlib.import_module('da4ml.trace.pipeline')
    FV = importlib.import_module('da4ml.trace.fixed_variable')
    TR = importlib.import_module('da4ml.trace.tracer')
    rng = np.random.default_rng(5)  # (the same latency sets as make_golden_pipeline_price.py)
    tasks = []
    base = _designs()
    extra = _extra_designs()
    work = [(name, stages, None, CUTOFFS) for name, stages in base] + extra
    for d, (name, stages, lat_sets, cutoffs) in enumerate(work):
        for st in stages:
            st['shape'] = (len(st['inp_shifts']), len(st['out_idxs']))
        pipe = pipeline_from_arrays(stages, types_module=T)
        n_in = stages[0]['shape'][0]
        a_sz, c_sz = int(stages[0]['adder_size']), int(stages[0]['carry_size'])
        if lat_sets is None:
            lat_sets = _lat_sets(n_in, rng) + [[6.5] * n_in]  # (and every input late: the reference's KeyError below 6.5)
        for lats in lat_sets:
            for cut in cutoffs:
                rec = {'design': d, 'latencies': lats, 'cutoff': cut}
                try:
                    emit._retrace([emit.as_stage(s) for s in stages], cut, abi_cost_add)
                except NotImplementedError:
                    rec['status'] = 2
                    tasks.append(rec)
                    continue
                except AssertionError:
                    pass
                hw = FV.HWConfig(a_sz, c_sz, cut)
                inp = [FV.FixedVariable(*q, hwconf=hw, latency=(0.0 if lats is None else lats[i]), cost=0.0) for i, q in enumerate(pipe.inp_qint)]
                try:
                    out = list(pipe(inp))
                except AssertionError:
                    rec['status'] = 1
                    tasks.append(rec)
                    continue
                rec['status'] = 0
                gathered = {v.id: v for v in inp}
                for o in out:
                    TR._recursive_gather(o, gathered)
                vs = list(gathered.values())
                N = len(vs)
                rec['interleaved'] = sorted(range(N), key=lambda i: vs[i].latency * N + i) != sorted(range(N), key=lambda i: (vs[i].latency, i))
                comb = trace.comb_trace(inp, out)
                try:
                    split = P.to_pipeline(comb, cut, retiming=False)
                except KeyError:
                    rec['split'] = None
                    tasks.append(rec)
                    continue
                rec['split'] = record([emit.as_stage(s) for s in split.solutions])
                rt = P.retime_pipeline(split, verbose=False)
                rec['retimed'] = record([emit.as_stage(s) for s in rt.solutions])
                tasks.append(rec)
    designs = [{'name': name, 'stages': [{k: np.asarray(st[k]).tolist() for k in ('inp_shifts', 'out_idxs', 'out_shifts', 'out_negs', 'ops_i')}
                                         | {'ops_f_bits': np.asarray(st['ops_f'], np.float32).view(np.uint32).tolist(), 'adder_size': int(st['adder_size']),
                                            'carry_size': int(st['carry_size'])} for st in stages]} for name, stages, _, _ in extra]  # fmt: skip
    raw = json.dumps({'designs': designs, 'tasks': tasks}, separators=(',', ':')).encode()
    with gzip.GzipFile(HERE / 'pipeline_split.json.gz', 'wb', mtime=0) as f:
        f.write(raw)
    ok = [t for t in tasks if t['status'] == 0]
    print(len(tasks), 'tasks,', len(ok), 'ok,', sum(t['split'] is None for t in ok), 'KeyError,', sum(t['interleaved'] for t in ok), 'interleaved,',
          (HERE / 'pipeline_split.json.gz').stat().st_size // 1024, 'KiB')  # fmt: skip


if __name__ == '__main__':
    main()
