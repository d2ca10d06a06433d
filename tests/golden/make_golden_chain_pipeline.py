"""Golden answers for chain designs (``da4ml_b200._binary.chain_design``) priced and split as one pipeline, from the
reference's OWN tracer: every layer of a chain is replayed with ``CombLogic.__call__`` on ``FixedVariable`` inputs under
``HWConfig(adder_size, carry_size, cutoff)``, the outputs of every layer but the last go through ``relu(i, f)`` or
``quantize(k, i, f)`` (TRN / WRAP), and the model is gathered with ``trace.comb_trace``, split with
``trace/pipeline.py::to_pipeline(retiming=False)`` and balanced with ``retime_pipeline``.

Chains are oracle solves of small random matrices (with a dead column feeding a quantizer, unsigned inputs whose relu
changes nothing, signed and unsigned quantizers, per-output and shared kif, formats that drop integer bits and ones that
drop fractional bits) and the 16x16 and 8x8 golden designs of the pricing fixture chained with themselves or with oracle
solves.  ``chains[c]``: the layers (stage arrays, ``ops_f`` as float32 bits), the activations (kind, [n, 3] kif) and,
per activation and value, what the tracer records for that value alone (``comb_trace`` of a fresh input at the value's
interval and latency through the activation): ``"self"``, ``["const", value]`` or the op (opcode, data, qint, latency,
cost).  Per task: status (0 ok, 1 an adder slower than the cutoff), and for ok tasks the first trace's output latencies
and, per split (``split``: without retiming, ``retimed``; null where to_pipeline raises KeyError) the stage count,
``reg_bits``, the record of make_golden_pipeline_split.py (``retimed`` also its ``cutoff``) and ``text``: the sha256 of
the reference emitters' text for that split (``text_digests``: Verilog with latencies, VHDL, Vitis HLS with latencies),
null where a network input lands past the first stage (an input op whose input number the stage does not have, which
the reference's emitters cannot index).

Container only: imports /root/reference/src/da4ml through tests/ref_trace.py, as make_golden_pipeline_price.py does.
Writes tests/golden/chain_pipeline.json.gz; running it again rewrites the same bytes.
"""
import contextlib
import gzip
import hashlib
import importlib
import io
import json
import sys
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parents[1]))
sys.path.insert(0, str(HERE.parent))
sys.path.insert(0, str(HERE))

CUTOFFS = [0.5, 1.0, 2.0, 3.0, 5.0, 8.0, 40.0]


def _solve(W, **kw):
    from oracle import oracle_solve

    stages = [dict(st) for st in oracle_solve(np.asarray(W, np.float32), **kw)[0]]
    return [dict(st, adder_size=kw.get('adder_size', -1), carry_size=kw.get('carry_size', -1)) for st in stages]


def _golden(name):
    from conftest import golden_cases, load_golden

    kw = golden_cases()[name]['kwargs']
    return [dict(st, adder_size=kw.get('adder_size', -1), carry_size=kw.get('carry_size', -1)) for st in load_golden(name)[1]]


def _chains():
    """(name, layers, activations): activations[k] = (kind, kif triple or [n, 3])."""
    rng = np.random.default_rng(77)
    W = lambda n, m, lo=-24, hi=24: rng.integers(lo, hi, size=(n, m)).astype(np.float32)  # noqa: E731
    out = []
    out.append(('relu_quantize_6x5x4x3', [_solve(W(6, 5)), _solve(W(5, 4)), _solve(W(4, 3))],
                [('relu', (0, 6, 0)), ('quantize', [(1, 5, 0), (0, 4, 0), (1, 9, 0), (0, 12, 0)])]))
    w0, w1 = W(8, 6), W(6, 4)
    w0[:, 2] = 0  # a dead column feeding the quantizer (its value is the constant 0), which the next layer does not read
    w1[2, :] = 0
    q = [(-4.0, 3.75, 0.25) if i % 2 else (0.0, 7.5, 0.5) for i in range(8)]
    out.append(('dead_column_frac_8x6x4', [_solve(w0, qintervals=q, adder_size=4, carry_size=2), _solve(w1, adder_size=4, carry_size=2)],
                [('quantize', (1, 6, 1))]))  # (drops fractional bits: TRN)
    out.append(('relu_frac_per_output_8x6x4', [_solve(w0, qintervals=q, adder_size=4, carry_size=2), _solve(w1, adder_size=4, carry_size=2)],
                [('relu', [(0, 3, 0), (0, 8, 2), (0, 2, 1), (0, 10, 0), (0, 5, -1), (0, 7, 3)])]))
    out.append(('golden16_wrap_16x16x6', [_golden('int_16x16_int8_default'), _solve(W(16, 6, -6, 6))], [('quantize', (1, 7, 0))]))  # (drops integer bits: WRAP)
    out.append(('golden8_relu_8x8x8', [_golden('c1_8x8_int4_default'), _golden('c1_8x8_int4_default')], [('relu', (0, 4, 1))]))
    u = [(0.0, 15.0, 1.0)] * 4
    out.append(('unsigned_noop_4x4x4x3', [_solve(W(4, 4, 0, 8), qintervals=u), _solve(W(4, 4, -8, 8)), _solve(W(4, 3))],
                [('relu', (0, 14, 0)), ('quantize', (1, 16, 2))]))  # (the relu changes nothing, the quantizer is wider)
    l4 = [_solve(W(5, 5), adder_size=2, carry_size=1) for _ in range(3)] + [_solve(W(5, 4), adder_size=2, carry_size=1)]
    out.append(('four_layers_5x5x5x5x4', l4, [('relu', (0, 5, 0)), ('quantize', [(0, 6, 0), (1, 4, 0), (0, 3, 0), (1, 8, 0), (0, 7, 0)]), ('relu', (0, 4, 0))]))
    return out


def _lat_sets(n_in, rng):
    return [None, [float(v) for v in rng.choice([0.0, 0.5, 1.0, 2.0, 3.0, 6.5], size=n_in)], [float(v) for v in rng.choice([0.0, 1.0, 2.5], size=n_in)]]


def text_digests(verilog, vhdl, hls) -> dict:
    """sha256 of the emitted text of one split: the Verilog and VHDL file dicts (sorted by name) and the HLS (function,
    bridge) pairs of its stages, in order."""
    h = lambda x: hashlib.sha256(json.dumps(x, sort_keys=True).encode()).hexdigest()  # noqa: E731
    return {'verilog': h(verilog), 'vhdl': h(vhdl), 'hls': h([list(t) for t in hls])}


def _kif_rows(kif, n):
    a = np.asarray(kif, np.int64)
    return np.tile(a, (n, 1)) if a.shape == (3,) else a.reshape(n, 3)


def main():
    import ref_trace
    from make_golden_pipeline_split import record

    from da4ml_b200 import emit
    from da4ml_b200.types import pipeline_from_arrays

    from oracle import port

    T, trace = ref_trace.load(None, port.get_lsb_loc, port.iceil_log2, port.cost_add)
    P = importlib.import_module('da4ml.trace.pipeline')
    FV = importlib.import_module('da4ml.trace.fixed_variable')
    V = importlib.import_module('da4ml.codegen.rtl.verilog')
    VH = importlib.import_module('da4ml.codegen.rtl.vhdl')
    H = importlib.import_module('da4ml.codegen.hls.hls_codegen')

    def text(sp):
        if any(op.opcode == -1 and op.id0 >= sol.shape[0] for sol in sp.solutions for op in sol.ops):
            return None  # (a network input that lands past the first stage keeps its input number: the emitters cannot index it)
        return text_digests(V.pipeline_logic_gen(sp, 'chain', print_latency=True), VH.pipeline_logic_gen(sp, 'chain'),
                            [H.hls_logic_and_bridge_gen(c, f'chain{k}', 'vitis', print_latency=True) for k, c in enumerate(sp.solutions)])

    rng = np.random.default_rng(6)
    chains, tasks = [], []
    for c, (name, layers, acts) in enumerate(_chains()):
        for stages in layers:
            for st in stages:
                st['shape'] = (len(st['inp_shifts']), len(st['out_idxs']))
        pipes = [pipeline_from_arrays(stages, types_module=T) for stages in layers]
        kifs = [_kif_rows(kif, layers[k][-1]['shape'][1]) for k, (_, kif) in enumerate(acts)]
        a_sz, c_sz = int(layers[0][0]['adder_size']), int(layers[0][0]['carry_size'])

        def activate(k, vals):
            kind = acts[k][0]
            return [v.relu(int(r[1]), int(r[2])) if kind == 'relu' else v.quantize(int(r[0]), int(r[1]), int(r[2])) for v, r in zip(vals, kifs[k])]

        # what the tracer records for each value alone: a fresh input at the value's interval and latency
        traced_ops = []
        hw0 = FV.HWConfig(a_sz, c_sz, -1)
        inp = [FV.FixedVariable(*q, hwconf=hw0, latency=0.0, cost=0.0) for q in pipes[0].inp_qint]
        vals = list(pipes[0](inp))
        for k in range(len(acts)):
            recs = []
            for v, r in zip(vals, kifs[k]):
                if v.low == v.high:
                    recs.append(['const', float(v.low)])
                    continue
                x = FV.FixedVariable(*v.qint, hwconf=hw0, latency=float(v.latency), cost=0.0)
                y = x.relu(int(r[1]), int(r[2])) if acts[k][0] == 'relu' else x.quantize(int(r[0]), int(r[1]), int(r[2]))
                if y is x:
                    recs.append('self')
                elif y.low == y.high:
                    recs.append(['const', float(y.low)])
                else:
                    op = trace.comb_trace([x], [y]).ops[-1]
                    recs.append([int(op.opcode), int(op.data), [float(t) for t in op.qint], float(op.latency), float(op.cost)])
            traced_ops.append(recs)
            vals = list(pipes[k + 1](activate(k, vals)))
        chains.append({'name': name, 'layers': [[{key: np.asarray(st[key]).tolist() for key in ('inp_shifts', 'out_idxs', 'out_shifts', 'out_negs', 'ops_i')}
                                                  | {'ops_f_bits': np.asarray(st['ops_f'], np.float32).view(np.uint32).tolist(), 'adder_size': int(st['adder_size']),
                                                     'carry_size': int(st['carry_size'])} for st in stages] for stages in layers],
                       'activations': [[kind, kifs[k].tolist()] for k, (kind, _) in enumerate(acts)], 'traced_ops': traced_ops})  # fmt: skip
        n_in = layers[0][0]['shape'][0]
        for lats in _lat_sets(n_in, rng):
            for cut in CUTOFFS:
                rec = {'chain': c, 'latencies': lats, 'cutoff': cut}
                hw = FV.HWConfig(a_sz, c_sz, cut)
                inp = [FV.FixedVariable(*q, hwconf=hw, latency=(0.0 if lats is None else lats[i]), cost=0.0) for i, q in enumerate(pipes[0].inp_qint)]
                try:
                    vals = list(pipes[0](inp))
                    for k in range(len(acts)):
                        vals = list(pipes[k + 1](activate(k, vals)))
                except AssertionError:
                    rec['status'] = 1
                    tasks.append(rec)
                    continue
                comb = trace.comb_trace(inp, vals)
                rec['status'] = 0
                rec['out_latency'] = [float(v) for v in comb.out_latency]
                try:
                    split = P.to_pipeline(comb, cut, retiming=False)
                except KeyError:
                    rec['split'] = None
                    tasks.append(rec)
                    continue
                rec['split'] = record([emit.as_stage(s) for s in split.solutions]) | {'reg_bits': int(split.reg_bits), 'text': text(split)}
                buf = io.StringIO()
                with contextlib.redirect_stdout(buf):
                    rt = P.retime_pipeline(split, verbose=True)
                rec['retimed'] = record([emit.as_stage(s) for s in rt.solutions]) | {'reg_bits': int(rt.reg_bits), 'cutoff': float(buf.getvalue().strip().split()[-1]),
                                                                                     'text': text(rt)}
                tasks.append(rec)
    raw = json.dumps({'chains': chains, 'tasks': tasks}, separators=(',', ':')).encode()
    with gzip.GzipFile(HERE / 'chain_pipeline.json.gz', 'wb', mtime=0) as f:
        f.write(raw)
    ok = [t for t in tasks if t['status'] == 0]
    print(len(chains), 'chains,', len(tasks), 'tasks,', len(ok), 'ok,', sum(t['split'] is None for t in ok), 'KeyError,',
          (HERE / 'chain_pipeline.json.gz').stat().st_size // 1024, 'KiB')  # fmt: skip


if __name__ == '__main__':
    main()
