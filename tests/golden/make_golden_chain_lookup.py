"""Golden answers for chains of layers with lookup-table activations (``('apply', fn, kif[, round_mode[,
overflow_mode]])`` in ``chain_front`` / ``chain_design``), from the reference's OWN tracer: a model is traced as a user
traces ``act_seq(x @ W_k + b_k)`` -- ``FixedVariableArray.from_lhs(..., hwconf=HWConfig(adder_size, carry_size, c))``,
``@ W_k`` under the option set chosen for the layer, ``+ b_k``, then each activation of the layer's sequence in order:
``.relu(i, f)``, ``.quantize(k, i, f)`` or ``.apply(fn).quantize(k, i, f, overflow_mode, round_mode)`` -- with
``oracle.oracle_solve`` standing in for the native ``solve`` and ``chain_lookup_fns.get_fixed_quantizer_np`` for the
``quantizers`` package.

Every model is traced under every tuple of per-layer option sets and every cutoff.  ``models[m]``: the kernels, the cost
model, layer 0's input intervals, the activations ([kind, kif] or [kind, fn name, kif, round, overflow] per element of
each layer's sequence), the biases, and ``traces``: per (choice, cutoff) every ``solve`` call, whether the trace raised
(``raised``: the exception's class name, or ``null``), and when it did not: the traced output latencies, ``lookups``
(per layer, every lookup the tracer created in the order it created them: [lo, hi, step, cost, latency, table sha256]),
and the model gathered with ``comb_trace`` and split with ``to_pipeline`` without retiming (``split``: the record of
make_golden_pipeline_split.py, ``reg_bits``, ``tables``, per stage the [sha256 of the int32 values, out_qint] of
its lookup tables, ``text``, the sha256 of the reference emitters' text as make_golden_chain_pipeline.py's
``text_digests`` gives them, and ``mem``, the sha256 of every ``.mem`` file ``table_mem_gen`` makes for the split's
stages, by name) and with retiming (``retimed``: the same, or the class name of what ``retime_pipeline`` raised).
``rows`` / ``outputs``: input rows on layer 0's grid and what the traced model (option set 0 at every layer, cutoff 5)
gives for them.

Container only: imports /root/reference/src/da4ml through tests/ref_trace.py and needs the oracle built by build().
Writes tests/golden/chain_lookup.json.gz; running it again rewrites the same bytes.
"""
import gzip
import hashlib
import importlib
import itertools
import json
import sys
import types
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parents[1]))
sys.path.insert(0, str(HERE.parent))
sys.path.insert(0, str(HERE))

from make_golden_chain_traced import SETS as ALL_SETS, digest, latency_max, seq_cost  # noqa: E402

import chain_lookup_fns as F  # noqa: E402

SETS = ALL_SETS[:2]
CUTOFFS = [2.0, 3.0, 5.0]
FNS = {'tanh': np.tanh, 'sigmoid': F.sigmoid, 'odd_cube': F.odd_cube}


def models():
    """(name, kernels, adder_size, carry_size, layer-0 intervals, activations (fn by name), biases)."""
    rng = np.random.default_rng(9431)
    W = lambda n, m, lo=-8, hi=8: rng.integers(lo, hi, size=(n, m)).astype(np.float32)  # noqa: E731
    out = []
    # quantize -> tanh between the layers (b_in = 6 after the quantizer); a dead column (tanh(0) = 0: dead)
    w0 = W(6, 5)
    w0[:, 2] = 0
    out.append(('quantize_tanh_6x5x3', [w0, W(5, 3)], -1, -1, [(-8.0, 7.0, 1.0)] * 6,
                [[('quantize', (1, 2, 3)), ('apply', 'tanh', (1, 0, 6))]], [None, None]))
    # relu -> sigmoid with RND / SAT, and a bias first; b_in >= 8 (latency > 1)
    out.append(('bias_relu_sigmoid_5x4x3', [W(5, 4), W(4, 3)], 1, -1, [(-4.0, 3.5, 0.5)] * 5,
                [[('relu', (0, 4, 4)), ('apply', 'sigmoid', (0, 0, 8), 'RND', 'SAT')]], [[0.5, -1.0, 0.25, 0.0], None]))
    # an odd function straight on a narrow layer output (b_in < 5: scaled cost), on a negated (-1) and a shifted (2)
    # pass-through column (negative factor: a reversed table); two outputs sharing a table
    w1 = np.zeros((3, 4), np.float32)
    w1[0, 0], w1[1, 1], w1[2, 2], w1[0, 3] = 1, -1, 2, 1
    out.append(('odd_narrow_3x4x2', [w1, W(4, 2)], -1, -1, [(-2.0, 1.5, 0.5), (-2.0, 1.0, 1.0), (0.0, 3.0, 1.0)],
                [[('apply', 'odd_cube', (1, 2, 2), 'TRN', 'SAT_SYM')]], [None, None]))
    # a dead column into sigmoid: the non-zero constant 0.5 (refused / dropped)
    w2 = W(4, 3)
    w2[:, 1] = 0
    # a wide lookup input: a fractional pre-quantizer (1, 4, 4) gives b_in = 9 (latency increment 3, cost 2**4 * ...),
    # whose latency crosses a register boundary at the small cutoffs
    out.append(('wide_tanh_5x4x2', [W(5, 4, -4, 4), W(4, 2)], -1, -1, [(-2.0, 1.875, 0.125)] * 5,
                [[('quantize', (1, 4, 4)), ('apply', 'tanh', (1, 1, 7))]], [None, None]))
    out.append(('dead_sigmoid_4x3x2', [w2, W(3, 2)], -1, -1, [(-4.0, 3.0, 1.0)] * 4,
                [[('quantize', (1, 3, 0)), ('apply', 'sigmoid', (0, 0, 4))]], [None, None]))
    return out


def main():
    sys.modules['quantizers'] = q0 = types.ModuleType('quantizers')
    q0.fixed_point = q1 = types.ModuleType('quantizers.fixed_point')
    q1.fixed_point_ops_np = q2 = types.ModuleType('quantizers.fixed_point.fixed_point_ops_np')
    q2.get_fixed_quantizer_np = F.get_fixed_quantizer_np
    sys.modules.update({'quantizers.fixed_point': q1, 'quantizers.fixed_point.fixed_point_ops_np': q2})
    import ref_trace
    from make_golden_chain_pipeline import text_digests
    from make_golden_pipeline_split import record

    from da4ml_b200 import emit
    from da4ml_b200.types import pipeline_from_arrays

    from oracle import oracle_solve
    from oracle import port

    calls = []

    def solve(kernel, **kw):
        stages, _ = oracle_solve(np.asarray(kernel, np.float32), **kw)
        stages = [dict(st) for st in stages]
        opts = {k: v for k, v in kw.items() if k not in ('qintervals', 'latencies')}
        calls.append(dict(options=opts, qintervals=[[float(v) for v in q] for q in kw['qintervals']], latencies=[float(v) for v in kw['latencies']],
                          cost=seq_cost(stages), latency_max=latency_max(stages), digest=digest(stages)))  # fmt: skip
        for st in stages:
            st['shape'] = (len(st['inp_shifts']), len(st['out_idxs']))
        return pipeline_from_arrays(stages, types_module=T)

    T, trace = ref_trace.load(solve, port.get_lsb_loc, port.iceil_log2, port.cost_add)
    FV = importlib.import_module('da4ml.trace.fixed_variable')
    FVA = importlib.import_module('da4ml.trace.fixed_variable_array').FixedVariableArray
    P = importlib.import_module('da4ml.trace.pipeline')
    V = importlib.import_module('da4ml.codegen.rtl.verilog')
    VC = importlib.import_module('da4ml.codegen.rtl.verilog.comb')
    VH = importlib.import_module('da4ml.codegen.rtl.vhdl')
    H = importlib.import_module('da4ml.codegen.hls.hls_codegen')

    def text(sp):
        return text_digests(V.pipeline_logic_gen(sp, 'chain', print_latency=True), VH.pipeline_logic_gen(sp, 'chain'),
                            [H.hls_logic_and_bridge_gen(c, f'chain{k}', 'vitis', print_latency=True) for k, c in enumerate(sp.solutions)])  # fmt: skip

    def mem(sp):
        files = {}
        for c in sp.solutions:
            files.update(VC.table_mem_gen(c))
        return {k: hashlib.sha256(v.encode()).hexdigest() for k, v in sorted(files.items())}

    def tables_of(sp):
        return [[[hashlib.sha256(np.asarray(t.table, np.int32).tobytes()).hexdigest(), [float(v) for v in t.spec.out_qint]] for t in (s.lookup_tables or ())]
                for s in sp.solutions]  # fmt: skip

    def sha(t):
        return hashlib.sha256(np.asarray(t.table, np.int32).tobytes()).hexdigest()

    rng = np.random.default_rng(10)
    out = []
    for name, kernels, a_sz, c_sz, q0_, acts, biases in models():
        traces = []
        q = np.asarray(q0_, np.float64)
        rows = [[float(rng.integers(round(lo / st), round(hi / st) + 1) * st) for lo, hi, st in q0_] for _ in range(32)]
        outputs = None
        for choice in itertools.product(range(len(SETS)), repeat=len(kernels)):
            for cut in CUTOFFS:
                calls.clear()
                x = FVA.from_lhs(q[:, 0], q[:, 1], q[:, 2], hwconf=FV.HWConfig(a_sz, c_sz, cut))
                inp = list(x._vars.ravel())
                rec = dict(choice=list(choice), cutoff=cut, raised=None)
                lookups = []
                try:
                    for k, W in enumerate(kernels):
                        x.solver_options = dict(SETS[choice[k]])
                        x = x @ W
                        if biases[k] is not None:
                            x = x + np.asarray(biases[k], np.float64)
                        made = []
                        for act in acts[k] if k < len(acts) else ():
                            kif = np.tile(np.asarray(act[-1] if act[0] != 'apply' else act[2], np.int64), (x.size, 1))
                            if act[0] == 'relu':
                                x = x.relu(kif[:, 1], kif[:, 2])
                            elif act[0] == 'quantize':
                                x = x.quantize(kif[:, 0], kif[:, 1], kif[:, 2])
                            else:
                                rnd, ovf = (list(act[3:]) + ['TRN', 'WRAP'][len(act) - 3 :])[:2]
                                x = x.apply(FNS[act[1]]).quantize(kif[:, 0], kif[:, 1], kif[:, 2], overflow_mode=ovf, round_mode=rnd)
                                for v in x._vars.ravel():
                                    if v.opr == 'lookup':
                                        t = FV.table_context.get_table_from_index(int(v._data))
                                        made.append([float(v.low), float(v.high), float(v.step), float(v.cost), float(v.latency), sha(t)])
                        lookups.append(made)
                except (AssertionError, ValueError) as e:
                    rec['raised'] = type(e).__name__
                else:
                    outs = list(x._vars.ravel())
                    rec['out_latency'] = [float(v.latency) for v in outs]
                    rec['lookups'] = lookups
                    comb = trace.comb_trace(inp, outs)
                    if choice == (0,) * len(kernels) and cut == 5.0:
                        outputs = [[float(v) for v in comb(np.asarray(r))] for r in rows]
                    try:
                        split = P.to_pipeline(comb, cut, retiming=False)
                    except KeyError:
                        rec['split'] = None
                    else:
                        rec['split'] = record([emit.as_stage(s) for s in split.solutions]) | {'reg_bits': int(split.reg_bits), 'tables': tables_of(split), 'text': text(split),
                                                                                         'mem': mem(split)}
                        try:
                            rt = P.retime_pipeline(split, verbose=False)
                        except Exception as e:  # noqa: BLE001  (recorded: the reference's retiming of lookups)
                            rec['retimed'] = type(e).__name__
                        else:
                            rec['retimed'] = record([emit.as_stage(s) for s in rt.solutions]) | {'reg_bits': int(rt.reg_bits), 'tables': tables_of(rt), 'text': text(rt),
                                                                                               'mem': mem(rt)}
                rec['calls'] = [dict(c) for c in calls]
                traces.append(rec)
        out.append(dict(name=name, kernels=[W.tolist() for W in kernels], adder_size=a_sz, carry_size=c_sz, qintervals=[list(r) for r in q0_],
                        activations=[[list(a[:2]) + [list(a[2])] + list(a[3:]) if a[0] == 'apply' else [a[0], list(a[1])] for a in seq] for seq in acts],
                        biases=biases, traces=traces, rows=rows, outputs=outputs))  # fmt: skip
    raw = json.dumps({'sets': SETS, 'cutoffs': CUTOFFS, 'models': out}, separators=(',', ':')).encode()
    with gzip.GzipFile(HERE / 'chain_lookup.json.gz', 'wb', mtime=0) as f:
        f.write(raw)
    n = sum(len(m['traces']) for m in out)
    print(len(out), 'models,', n, 'traces,', sum(bool(t['raised']) for m in out for t in m['traces']), 'raised,',
          (HERE / 'chain_lookup.json.gz').stat().st_size // 1024, 'KiB')


if __name__ == '__main__':
    main()
