"""Golden answers for chains of layers with leaky ReLU activations (``('leaky_relu', alpha)`` in ``chain_front`` /
``chain_design``), from the reference's OWN tracer: a model is traced as a user traces ``act_seq(x @ W_k + b_k)`` --
``FixedVariableArray.from_lhs(..., hwconf=HWConfig(adder_size, carry_size, c))``, ``@ W_k`` under the option set chosen
for the layer, ``+ b_k``, then each activation of the layer's sequence in order: ``np.maximum(x, alpha * x)``,
``.relu(i, f)``, ``.quantize(k, i, f)`` or ``.apply(fn).quantize(k, i, f, overflow_mode, round_mode)`` -- with
``oracle.oracle_solve`` standing in for the native ``solve`` and ``chain_lookup_fns.get_fixed_quantizer_np`` for the
``quantizers`` package.

Every model is traced under every tuple of per-layer option sets and every cutoff.  ``models[m]``: the kernels, the cost
model, layer 0's input intervals, the activations ([kind, kif] or [kind, fn name, kif, round, overflow] per element of
each layer's sequence), the biases, and ``traces``: per (choice, cutoff) every ``solve`` call, whether the trace raised
(``raised``: the exception's class name, or ``null``), and when it did not: the traced output latencies, ``muxes``
(per layer, for every value a leaky ReLU turned into an MSB mux, in value order: [[lo, hi, step, cost, latency] of the
condition adder, the same of the mux as the tracer hands it on (a negated view for a negative factor), the mux's opcode
sign]), ``leaky_cases`` (per layer, per value of each leaky ReLU: 'x' for x itself, 'view' for alpha * x, 'zero',
'mux'), ``lookups`` (per layer, every lookup the tracer created in the order it created them: [lo, hi, step, cost,
latency, table sha256]),
and the model gathered with ``comb_trace`` and split with ``to_pipeline`` without retiming (``split``: the record of
make_golden_pipeline_split.py, ``reg_bits``, ``tables``, per stage the [sha256 of the int32 values, out_qint] of
its lookup tables, ``text``, the sha256 of the reference emitters' text as make_golden_chain_pipeline.py's
``text_digests`` gives them, and ``mem``, the sha256 of every ``.mem`` file ``table_mem_gen`` makes for the split's
stages, by name) and with retiming (``retimed``: the same, or the class name of what ``retime_pipeline`` raised).
``rows`` / ``outputs``: input rows on layer 0's grid and what the traced model (option set 0 at every layer, cutoff 5)
gives for them.

``hand_muxes``: a hand-made design (``hand_muxes()``) whose MSB muxes read a condition independent of their data
operands, with opcodes 6 and -6: its stages, and per (input latencies, cutoff) the traced output latencies, the mux
opcodes of the traced model, and its split without and with retiming (the record, ``reg_bits`` and ``text``).

Container only: imports /root/reference/src/da4ml through tests/ref_trace.py and needs the oracle built by build().
Writes tests/golden/chain_leaky.json.gz; running it again rewrites the same bytes.
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
FNS = {'tanh': np.tanh}


def models():
    """(name, kernels, adder_size, carry_size, layer-0 intervals, activations (fn by name), biases)."""
    rng = np.random.default_rng(7321)
    W = lambda n, m, lo=-8, hi=8: rng.integers(lo, hi, size=(n, m)).astype(np.float32)  # noqa: E731
    out = []
    # leaky(0.125) then a quantizer: mixed-sign columns, an all-non-negative column (x.low = 0 < alpha * x.high: still a
    # mux), a dead column, and a column -3 * x0 that the solver builds from adders (its traced interval crosses zero: a mux)
    w0 = W(5, 6)
    w0[:, 1] = np.abs(w0[:, 1])
    w0[:, 2] = 0
    w0[:, 3] = 0
    w0[0, 3] = -3
    out.append(('leaky_quantize_5x6x3', [w0, W(6, 3)], -1, -1, [(1.0, 7.0, 1.0)] + [(-8.0, 7.0, 1.0)] * 4,
                [[('leaky_relu', 0.125), ('quantize', (1, 6, 2))]], [None, None]))
    # negated and shifted pass-through columns: negative factors (the mirrored mux path, opcode -6)
    w1 = np.zeros((3, 4), np.float32)
    w1[0, 0], w1[1, 1], w1[2, 2], w1[0, 3] = -1, -2, 4, 1
    out.append(('leaky_negated_3x4x2', [w1, W(4, 2)], -1, -1, [(-4.0, 3.5, 0.5), (-2.0, 3.0, 1.0), (-1.0, 1.0, 0.25)],
                [[('leaky_relu', 0.25)]], [None, None]))
    # a bias, then leaky(0.25) and a quantizer, under a non-default adder / carry size
    out.append(('bias_leaky_4x4x2', [W(4, 4), W(4, 2)], 16, -1, [(-4.0, 3.5, 0.5)] * 4,
                [[('leaky_relu', 0.25), ('quantize', (1, 5, 2))]], [[0.5, -1.0, 0.0, 0.25], None]))
    # leaky into a tanh table: opcodes 6 and 8 in one stage sequence
    out.append(('leaky_tanh_4x3x2', [W(4, 3, -4, 4), W(3, 2)], -1, -1, [(-2.0, 1.5, 0.5)] * 4,
                [[('leaky_relu', 0.5), ('quantize', (1, 2, 3)), ('apply', 'tanh', (1, 0, 6))]], [None, None]))
    # a wide condition: 16-bit layer outputs, whose condition adder crosses a register boundary at cutoff 2
    out.append(('wide_leaky_4x3x2', [W(4, 3, -128, 128), W(3, 2)], -1, -1, [(-128.0, 127.0, 1.0)] * 4,
                [[('leaky_relu', 0.0625), ('quantize', (1, 12, 0))]], [None, None]))
    # the two no-op cases on a strictly positive input x0 in [1, 7]: the identity column x0 (x.low >= alpha * x.high: x
    # itself) and the negated pass-through -x0 (x.high <= alpha * x.low: the view alpha * x, whose scaled interval the
    # quantizer / relu and the next layer see), next to a mixed-sign column and a shifted one
    w3 = np.zeros((2, 4), np.float32)
    w3[0, 0], w3[0, 1], w3[0, 2], w3[1, 2], w3[1, 3] = 1, -1, 1, 1, -2
    out.append(('leaky_noop_2x4x2', [w3, W(4, 2)], -1, -1, [(1.0, 7.0, 1.0), (-2.0, 3.0, 1.0)],
                [[('leaky_relu', 0.125), ('quantize', (1, 6, 2))]], [None, None]))
    out.append(('leaky_noop_relu_2x4x2', [w3, W(4, 2)], -1, -1, [(1.0, 7.0, 1.0), (-2.0, 3.0, 1.0)],
                [[('leaky_relu', 0.125), ('relu', (0, 6, 3))]], [None, None]))
    return out


def _stage(n_in, ops, out_idxs):
    """One stage dict from [(id0, id1, opcode, data, (lo, hi, step))] (latency and cost 0: the tracer recomputes them)."""
    return dict(inp_shifts=[0] * n_in, out_idxs=list(out_idxs), out_shifts=[0] * len(out_idxs), out_negs=[0] * len(out_idxs),
                ops_i=np.asarray([o[:4] for o in ops], np.int64).reshape(-1, 4), ops_f=np.asarray([[*o[4], 0.0, 0.0] for o in ops], np.float32).reshape(-1, 5),
                adder_size=-1, carry_size=-1)  # fmt: skip


def hand_muxes():
    """A hand-made design with MSB muxes whose condition is a node of its own, independent of the data operands (as
    clip / abs / min will have them): a = x0 + x1, b = x2 - x3, the condition x1 - x3, then mux(a, b) (opcode 6) and
    mux(a, -b * 2) (opcode -6, shift 1).  Under late inputs and small cutoffs a, b and the condition are carried into
    the muxes' stage, so the order of their copies there pins the condition's event slot and its place in the gather.
    (stages, latency sets, cutoffs)."""
    q0, q1, q2, q3 = (-8.0, 7.5, 0.5), (0.0, 15.0, 1.0), (-4.0, 3.75, 0.25), (-2.0, 3.0, 1.0)
    ops = [(0, -1, -1, 0, q0), (1, -1, -1, 0, q1), (2, -1, -1, 0, q2), (3, -1, -1, 0, q3), (0, 1, 0, 0, (-8.0, 22.5, 0.5)), (2, 3, 1, 0, (-7.0, 5.75, 0.25)),
           (1, 3, 1, 0, (-3.0, 17.0, 1.0)), (4, 5, 6, 6, (-8.0, 22.5, 0.25)), (4, 5, -6, (1 << 32) | 6, (-11.5, 22.5, 0.25))]  # fmt: skip
    return [_stage(4, ops, [7, 8])], [None, [0.0, 2.5, 0.0, 1.0], [3.0, 0.0, 1.0, 0.0], [0.0, 0.0, 4.0, 0.0]], [1.0, 2.0, 3.0]


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
                lookups, muxes, cases = [], [], []
                try:
                    for k, W in enumerate(kernels):
                        x.solver_options = dict(SETS[choice[k]])
                        x = x @ W
                        if biases[k] is not None:
                            x = x + np.asarray(biases[k], np.float64)
                        made, mux_made, case_made = [], [], []
                        for act in acts[k] if k < len(acts) else ():
                            if act[0] == 'leaky_relu':
                                y = np.maximum(x, np.multiply(x, act[1]))
                                for u, v in zip(x._vars.ravel(), y._vars.ravel()):
                                    case_made.append('zero' if u.low == u.high == 0 else 'x' if v is u else 'mux' if v.opr == 'msb_mux' else 'view' if v.id == u.id else '?')
                                for v in y._vars.ravel():
                                    if v.opr == 'msb_mux':
                                        c, inner = v._from[0], -v if v._factor < 0 else v
                                        mux_made.append([[float(c.low), float(c.high), float(c.step), float(c.cost), float(c.latency)],
                                                         [float(v.low), float(v.high), float(v.step), float(v.cost), float(v.latency)],
                                                         6 if inner._from[2]._factor > 0 else -6])
                                x = y
                                continue
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
                        muxes.append(mux_made)
                        cases.append(case_made)
                except (AssertionError, ValueError) as e:
                    rec['raised'] = type(e).__name__
                else:
                    outs = list(x._vars.ravel())
                    rec['out_latency'] = [float(v.latency) for v in outs]
                    rec['lookups'] = lookups
                    rec['muxes'] = muxes
                    rec['leaky_cases'] = cases
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
                        activations=[[list(a[:2]) + [list(a[2])] + list(a[3:]) if a[0] == 'apply' else list(a) if a[0] == 'leaky_relu' else [a[0], list(a[1])] for a in seq]
                                     for seq in acts],
                        biases=biases, traces=traces, rows=rows, outputs=outputs))  # fmt: skip
    stages, lat_sets, cuts = hand_muxes()
    for st in stages:
        st['shape'] = (len(st['inp_shifts']), len(st['out_idxs']))
    pipe = pipeline_from_arrays(stages, types_module=T)
    hand = dict(stages=[{k: np.asarray(st[k]).tolist() for k in ('inp_shifts', 'out_idxs', 'out_shifts', 'out_negs', 'ops_i')}
                        | {'ops_f_bits': np.asarray(st['ops_f'], np.float32).view(np.uint32).tolist(), 'adder_size': -1, 'carry_size': -1} for st in stages], tasks=[])  # fmt: skip
    for lats in lat_sets:
        for cut in cuts:
            hw = FV.HWConfig(-1, -1, cut)
            inp = [FV.FixedVariable(*q, hwconf=hw, latency=(0.0 if lats is None else lats[i]), cost=0.0) for i, q in enumerate(pipe.inp_qint)]
            outs = list(pipe(inp))
            comb = trace.comb_trace(inp, outs)
            rec = dict(latencies=lats, cutoff=cut, out_latency=[float(v.latency) for v in outs],
                       opcodes=sorted({int(op.opcode) for op in comb.ops if abs(op.opcode) == 6}))
            try:
                split = P.to_pipeline(comb, cut, retiming=False)
            except KeyError:
                rec['split'] = None
            else:
                rec['split'] = record([emit.as_stage(s) for s in split.solutions]) | {'reg_bits': int(split.reg_bits), 'text': text(split)}
                rt = P.retime_pipeline(split, verbose=False)
                rec['retimed'] = record([emit.as_stage(s) for s in rt.solutions]) | {'reg_bits': int(rt.reg_bits), 'text': text(rt)}
            hand['tasks'].append(rec)
    raw = json.dumps({'sets': SETS, 'cutoffs': CUTOFFS, 'models': out, 'hand_muxes': hand}, separators=(',', ':')).encode()
    with gzip.GzipFile(HERE / 'chain_leaky.json.gz', 'wb', mtime=0) as f:
        f.write(raw)
    n = sum(len(m['traces']) for m in out)
    print(len(out), 'models,', n, 'traces,', sum(bool(t['raised']) for m in out for t in m['traces']), 'raised,',
          (HERE / 'chain_leaky.json.gz').stat().st_size // 1024, 'KiB')


if __name__ == '__main__':
    main()
