"""Golden answers for chains of layers with biases (``chain_front(..., activations=..., biases=...)`` and
``chain_design(designs, activations, biases)``), from the reference's OWN tracer: a model is traced as a user traces
``act(x @ W_k + b_k)`` -- ``FixedVariableArray.from_lhs(..., hwconf=HWConfig(adder_size, carry_size, c))``, then ``@ W_k``
with the array's ``solver_options`` set to the option set chosen for that layer, then ``+ b_k`` (``FixedVariable._const_add``)
and ``.relu(i, f)`` or ``.quantize(k, i, f)`` (TRN / WRAP), and the last layer's bias -- with ``oracle.oracle_solve``
standing in for the native ``solve``.

Every model is traced under every tuple of per-layer option sets and every cutoff.  ``models[m]``: the kernels, the cost
model, layer 0's input intervals, the activations (kind, [n, 3] kif), the biases (one list per layer) and ``traces``: per
(choice, cutoff) every ``solve`` call (as make_golden_chain_traced.py records them), whether the trace raised, and when
it did not: the traced output latencies, ``bias_ops`` (per layer and output, what the tracer records for ``v + b`` on the
layer's traced output ``v``: ``null`` for a zero bias, ``["const", value]``, ``"folded"`` or [4, data in steps of the
result, (lo, hi, step) of the value, cost]), and the model gathered with ``comb_trace`` and split with ``to_pipeline``
(``split``: without retiming; ``retimed``: ``retime_pipeline``'s, with its ``cutoff``), each with its stage count,
``reg_bits``, the record of make_golden_pipeline_split.py and the sha256 of the reference emitters' text
(make_golden_chain_pipeline.py's ``text_digests``).  ``rows`` / ``outputs``: input rows on layer 0's grid and what the
traced model (``CombLogic.__call__`` of the gathered trace of option set 0 at every layer, cutoff 5) gives for them.

The models cover a bias then relu and a bias then a signed WRAP quantizer that drops integer bits; positive, negative,
zero and fractional biases, one finer than the value's step; a bias on a negated and on a shifted output; a bias after
the last layer; a dead column with zero bias and one with a non-zero bias (a non-zero constant, which ``chain_design``
refuses); and a pass-through column whose bias the tracer folds into the bias of the layer before.

Container only: imports /root/reference/src/da4ml through tests/ref_trace.py and needs the oracle built by build(), as
make_golden_chain_traced.py does.  Writes tests/golden/chain_bias.json.gz; running it again rewrites the same bytes.
"""
import contextlib
import gzip
import importlib
import io
import itertools
import json
import sys
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parents[1]))
sys.path.insert(0, str(HERE.parent))
sys.path.insert(0, str(HERE))

from make_golden_chain_traced import SETS as ALL_SETS, digest, latency_max, seq_cost  # noqa: E402

SETS = ALL_SETS[:2]
CUTOFFS = [3.0, 5.0]


def models():
    """(name, kernels, adder_size, carry_size, layer-0 intervals, activations, biases)."""
    rng = np.random.default_rng(4711)
    W = lambda n, m, lo=-8, hi=8: rng.integers(lo, hi, size=(n, m)).astype(np.float32)  # noqa: E731
    out = []
    # bias then relu, bias then a signed WRAP quantizer that drops integer bits, and a bias after the last layer; a
    # negated (-1) and a shifted (2) pass-through column of layer 0; biases positive, negative, zero and fractional,
    # 0.375 finer than the integer step of its value
    w0 = W(6, 5)
    w0[:, 3] = 0
    w0[1, 3] = -1
    w0[:, 4] = 0
    w0[2, 4] = 2
    out.append(('bias_relu_wrap_6x5x4x3', [w0, W(5, 4), W(4, 3)], -1, -1, [(-8.0, 7.0, 1.0)] * 6,
                [('relu', [(0, 6, 1)] * 5), ('quantize', [(1, 3, 0)] * 4)],
                [[1.5, -2.0, 0.0, 0.375, 3.0], [-0.5, 0.25, 0.0, 7.0], [0.5, -1.0, 0.125]]))
    # fractional inputs, a dead column with zero bias, and a relu after it
    w1 = W(8, 6, -12, 12)
    w1[:, 2] = 0
    out.append(('frac_dead_zero_bias_8x6x3', [w1, W(6, 3)], 1, -1, [(-4.0, 3.75, 0.25) if i % 2 else (0.0, 7.5, 0.5) for i in range(8)],
                [('relu', [(0, 8, 2)] * 6)], [[0.25, -0.75, 0.0, 1.0, -3.5, 0.0625], None]))
    # a dead column with a non-zero bias: a non-zero constant
    w2 = W(5, 4)
    w2[:, 1] = 0
    out.append(('dead_nonzero_bias_5x4x3', [w2, W(4, 3)], -1, -1, [(-8.0, 7.0, 1.0)] * 5, [('quantize', [(1, 9, 0)] * 4)], [[1.0, 2.0, -1.0, 0.5], None]))
    # folding: layer 1 passes its input 0 through, which is layer 0's biased value that the wide quantizer left
    # unchanged, and adds a bias of its own to it
    w3 = W(4, 4)
    w4 = W(4, 3)
    w4[:, 0] = 0
    w4[0, 0] = 1
    out.append(('folded_bias_4x4x3', [w3, w4], -1, -1, [(-8.0, 7.0, 1.0)] * 4, [('quantize', [(1, 20, 4)] * 4)], [[2.0, -1.0, 0.5, 0.0], [1.0, 0.0, -0.25]]))
    return out


def main():
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
    VH = importlib.import_module('da4ml.codegen.rtl.vhdl')
    H = importlib.import_module('da4ml.codegen.hls.hls_codegen')

    def text(sp):
        if any(op.opcode == -1 and op.id0 >= sol.shape[0] for sol in sp.solutions for op in sol.ops):
            return None
        return text_digests(V.pipeline_logic_gen(sp, 'chain', print_latency=True), VH.pipeline_logic_gen(sp, 'chain'),
                            [H.hls_logic_and_bridge_gen(c, f'chain{k}', 'vitis', print_latency=True) for k, c in enumerate(sp.solutions)])  # fmt: skip

    def bias_op(v, b):
        if b == 0:
            return None
        if v.low == v.high:
            return ['const', float(v.low + FV.Decimal(b))]
        if v.opr == 'cadd':
            return 'folded'
        y = v + b
        step = float(y.step)
        return [4, int(float(b) / step), [float(y.low), float(y.high), step], float(y.cost)]

    rng = np.random.default_rng(8)
    out = []
    for name, kernels, a_sz, c_sz, q0, acts, biases in models():
        traces = []
        q = np.asarray(q0, np.float64)
        rows = [[float(rng.integers(round(lo / st), round(hi / st) + 1) * st) for lo, hi, st in q0] for _ in range(32)]
        outputs = None
        for choice in itertools.product(range(len(SETS)), repeat=len(kernels)):
            for cut in CUTOFFS:
                calls.clear()
                x = FVA.from_lhs(q[:, 0], q[:, 1], q[:, 2], hwconf=FV.HWConfig(a_sz, c_sz, cut))
                inp = list(x._vars.ravel())
                rec = dict(choice=list(choice), cutoff=cut)
                ops = []
                try:
                    for k, W in enumerate(kernels):
                        x.solver_options = dict(SETS[choice[k]])
                        x = x @ W
                        if biases[k] is not None:
                            ops.append([bias_op(v, b) for v, b in zip(x._vars.ravel(), biases[k])])
                            x = x + np.asarray(biases[k], np.float64)
                        else:
                            ops.append(None)
                        if k < len(acts):
                            kind, kif = acts[k]
                            kif = np.asarray(kif, np.int64)
                            x = x.relu(kif[:, 1], kif[:, 2]) if kind == 'relu' else x.quantize(kif[:, 0], kif[:, 1], kif[:, 2])
                except AssertionError:
                    rec['raised'] = True
                else:
                    rec['raised'] = False
                    outs = list(x._vars.ravel())
                    rec['out_latency'] = [float(v.latency) for v in outs]
                    rec['bias_ops'] = ops
                    comb = trace.comb_trace(inp, outs)
                    if choice == (0,) * len(kernels) and cut == 5.0:
                        outputs = [[float(v) for v in comb(np.asarray(r))] for r in rows]
                    try:
                        split = P.to_pipeline(comb, cut, retiming=False)
                    except KeyError:
                        rec['split'] = None
                    else:
                        rec['split'] = record([emit.as_stage(s) for s in split.solutions]) | {'reg_bits': int(split.reg_bits), 'text': text(split)}
                        buf = io.StringIO()
                        with contextlib.redirect_stdout(buf):
                            rt = P.retime_pipeline(split, verbose=True)
                        rec['retimed'] = record([emit.as_stage(s) for s in rt.solutions]) | {'reg_bits': int(rt.reg_bits), 'cutoff': float(buf.getvalue().strip().split()[-1]),
                                                                                             'text': text(rt)}  # fmt: skip
                rec['calls'] = [dict(c) for c in calls]
                traces.append(rec)
        out.append(dict(name=name, kernels=[W.tolist() for W in kernels], adder_size=a_sz, carry_size=c_sz, qintervals=[list(r) for r in q0],
                        activations=[[kind, np.asarray(kif, np.int64).tolist()] for kind, kif in acts], biases=biases, traces=traces, rows=rows,
                        outputs=outputs))  # fmt: skip
    raw = json.dumps({'sets': SETS, 'cutoffs': CUTOFFS, 'models': out}, separators=(',', ':')).encode()
    with gzip.GzipFile(HERE / 'chain_bias.json.gz', 'wb', mtime=0) as f:
        f.write(raw)
    n = sum(len(m['traces']) for m in out)
    print(len(out), 'models,', n, 'traces,', sum(t['raised'] for m in out for t in m['traces']), 'raised,', (HERE / 'chain_bias.json.gz').stat().st_size // 1024, 'KiB')


if __name__ == '__main__':
    main()
