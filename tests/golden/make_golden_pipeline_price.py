"""Golden answers for pipelined pricing (``da4ml_b200._binary.price_pipelined``) from the reference's OWN tracer: every design is
replayed on ``FixedVariable`` inputs under ``HWConfig(adder_size, carry_size, cutoff)`` (``Pipeline.__call__``), gathered
with ``trace.comb_trace``, split with ``trace/pipeline.py::to_pipeline(retiming=False)`` and balanced with
``retime_pipeline``; ``Pipeline.reg_bits`` and ``CombLogic.out_latency`` give the numbers.

Container only: imports /root/reference/src/da4ml as a package with its native module replaced by a stand-in
(tests/ref_trace.py) whose ``cost_add`` is the oracle's.  Designs are golden solves, solves of the reference's object code
(oracle/_ref) and the oracle, plus two hand-edited ones (a design with an all-zero column, and one with a stage-0 op that
nothing reads).  Writes tests/golden/pipeline_price.json.gz.
"""
import contextlib
import gzip
import importlib
import io
import json
import sys
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parents[1]))
sys.path.insert(0, str(HERE.parent))

GOLDEN = ['c1_8x8_int4_default', 'int_16x16_int8_default', 'single_16x12_hetero_wmc', 'int_17x5_int8_mcpdc', 'pytest_8_b4_harddc2_add1', 'int_12x20_int6_harddc1']
CUTOFFS = [0.5, 1.0, 2.0, 2.5, 3.0, 4.0, 5.0, 7.5, 12.0, 40.0]


def _designs():
    from conftest import golden_cases, load_golden

    from oracle import oracle_solve

    out = []
    for name in GOLDEN:
        meta = golden_cases()[name]
        _, stages = load_golden(name)
        kw = meta['kwargs']
        out.append((name, [dict(st, adder_size=kw.get('adder_size', -1), carry_size=kw.get('carry_size', -1)) for st in stages]))
    rng = np.random.default_rng(2024)
    for k in range(6):
        n_in, n_out = int(rng.integers(4, 14)), int(rng.integers(3, 14))
        W = rng.integers(-40, 40, size=(n_in, n_out)).astype(np.float32)
        kw = dict(adder_size=int(rng.integers(1, 9)), carry_size=int(rng.integers(1, 5))) if k % 3 else {}
        if k == 1:
            W[:, 1] = 0  # an all-zero column: a dead output, the constant 0 the tracer carries to the last stage
        if k == 4:
            kw['qintervals'] = [(-8.0, 7.5, 0.5) if i % 2 else (0.0, 15.0, 1.0) for i in range(n_in)]
        stages = [dict(st) for st in oracle_solve(W, **kw)[0]]
        out.append((f'random_{k}_{n_in}x{n_out}', [dict(st, adder_size=kw.get('adder_size', -1), carry_size=kw.get('carry_size', -1)) for st in stages]))
    # one-stage designs: the first stage of a two-stage one on its own
    out.append(('stage0_of_' + out[1][0], [out[1][1][0]]))
    out.append(('stage0_of_' + out[-2][0], [out[-2][1][0]]))
    # a stage-0 op nothing reads: the tracer still traces it (it can fail the cutoff), comb_trace drops it
    name, stages = out[7]
    st0 = dict(stages[0])
    oi, of = np.asarray(st0['ops_i'], np.int64), np.asarray(st0['ops_f'], np.float32)
    n = len(oi)
    a, b = n - 1, n - 2
    extra_f = np.array([[of[a, 0] + of[b, 0], of[a, 1] + of[b, 1], min(of[a, 2], of[b, 2]), max(of[a, 3], of[b, 3]) + 1, 1]], np.float32)
    st0['ops_i'] = np.concatenate([oi, [[a, b, 0, 0]]])
    st0['ops_f'] = np.concatenate([of, extra_f])
    out.append(('dead_op_' + name, [st0] + list(stages[1:])))
    return out


def _lat_sets(n_in, rng):
    het = rng.choice([0.0, 0.5, 1.0, 2.0, 3.0, 6.5], size=n_in)
    return [None, [float(v) for v in het], [float(v) for v in rng.choice([0.0, 1.0, 2.5], size=n_in)]]


def main():
    import ref_trace

    from da4ml_b200 import emit
    from da4ml_b200._binary import cost_add as abi_cost_add
    from da4ml_b200.types import pipeline_from_arrays

    from oracle import port

    T, trace = ref_trace.load(None, port.get_lsb_loc, port.iceil_log2, port.cost_add)
    P = importlib.import_module('da4ml.trace.pipeline')
    FV = importlib.import_module('da4ml.trace.fixed_variable')
    rng = np.random.default_rng(5)
    designs, tasks = [], []
    for d, (name, stages) in enumerate(_designs()):
        for st in stages:
            st['shape'] = (len(st['inp_shifts']), len(st['out_idxs']))
        pipe = pipeline_from_arrays(stages, types_module=T)
        designs.append({'name': name, 'stages': [{k: np.asarray(st[k]).tolist() for k in ('inp_shifts', 'out_idxs', 'out_shifts', 'out_negs', 'ops_i')}
                                                 | {'ops_f_bits': np.asarray(st['ops_f'], np.float32).view(np.uint32).tolist(), 'adder_size': int(st['adder_size']),
                                                    'carry_size': int(st['carry_size'])} for st in stages]})  # fmt: skip
        n_in = stages[0]['shape'][0]
        a_sz, c_sz = int(stages[0]['adder_size']), int(stages[0]['carry_size'])
        for lats in _lat_sets(n_in, rng):
            for cut in CUTOFFS:
                rec = {'design': d, 'latencies': lats, 'cutoff': cut}
                try:  # the case this library reports as "not supported": a constant intermediate value
                    emit._retrace([emit.as_stage(s) for s in stages], cut, abi_cost_add)
                except NotImplementedError:
                    rec['status'] = 2
                    tasks.append(rec)
                    continue
                except AssertionError:
                    pass
                hw = FV.HWConfig(a_sz, c_sz, cut)
                inp = [FV.FixedVariable(*q, hwconf=hw, latency=(0.0 if lats is None else lats[i]), cost=0.0) for i, q in enumerate(pipe.inp_qint)]  # (an input at its latency, as FixedVariableInput makes one)
                try:
                    out = list(pipe(inp))
                except AssertionError:
                    rec['status'] = 1
                    tasks.append(rec)
                    continue
                comb = trace.comb_trace(inp, out)
                rec['status'] = 0
                rec['out_latency'] = [float(v) for v in comb.out_latency]
                try:
                    split = P.to_pipeline(comb, cut, retiming=False)
                except KeyError:  # a stage with no op: every input arrives after the first stage
                    rec['split'] = None
                    tasks.append(rec)
                    continue
                rec['split'] = {'stages': len(split.solutions), 'reg_bits': int(split.reg_bits)}
                buf = io.StringIO()
                with contextlib.redirect_stdout(buf):
                    rt = P.retime_pipeline(split, verbose=True)
                rec['retimed'] = {'stages': len(rt.solutions), 'reg_bits': int(rt.reg_bits), 'cutoff': float(buf.getvalue().strip().split()[-1])}
                tasks.append(rec)
    raw = json.dumps({'designs': designs, 'tasks': tasks}, separators=(',', ':')).encode()
    with gzip.GzipFile(HERE / 'pipeline_price.json.gz', 'wb', mtime=0) as f:
        f.write(raw)
    st = np.bincount([t['status'] for t in tasks], minlength=3)
    print(len(designs), 'designs,', len(tasks), 'tasks (ok / slow adder / not supported:', st.tolist(), '),', (HERE / 'pipeline_price.json.gz').stat().st_size // 1024, 'KiB')


if __name__ == '__main__':
    main()
