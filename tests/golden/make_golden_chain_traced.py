"""Golden answers for chains of layers solved under the intervals their relu / quantizers hand each layer
(``chain_front(..., activations=...)``), from the reference's OWN tracer: a model is traced layer by layer as a user
would trace it -- ``FixedVariableArray.from_lhs(..., hwconf=HWConfig(adder_size, carry_size, c))``, then ``@ W_k`` with
the array's ``solver_options`` set to the option set chosen for that layer, then ``.relu(i, f)`` or ``.quantize(k, i,
f)`` (TRN / WRAP) -- with ``oracle.oracle_solve`` standing in for the native ``solve``.

Every model is traced under every tuple of per-layer option sets and every cutoff.  ``models[m]``: the kernels, the cost
model, layer 0's input intervals, the activations (kind, [n, 3] kif) and ``traces``: per (choice, cutoff) every ``solve``
call the tracer made -- its options, ``qintervals`` and ``latencies`` as the tracer passed them, and the result's cost
(the float32 sum over its ops in op order), ``latency_max`` and sha256 of its stage arrays -- whether the trace raised
(an adder slower than the cutoff; the calls up to and including that layer's are kept) and, when it did not, the traced
output latencies of the model.

The models cover a relu that saturates every value (intervals that do not depend on the design), a relu and a wide
quantizer that pass design-dependent intervals on, a signed WRAP quantizer that drops integer bits, and per-output kif
with one value left with no bits (a dead input of the next layer).

Container only: imports /root/reference/src/da4ml through tests/ref_trace.py and needs the oracle built by build(), as
make_golden_chain_pipeline.py does.  Writes tests/golden/chain_traced.json.gz; running it again rewrites the same bytes.
"""
import gzip
import hashlib
import importlib
import itertools
import json
import sys
from pathlib import Path

import numpy as np

HERE = Path(__file__).resolve().parent
sys.path.insert(0, str(HERE.parents[1]))
sys.path.insert(0, str(HERE.parent))

STAGE_KEYS = ['inp_shifts', 'out_idxs', 'out_shifts', 'out_negs', 'ops_i', 'ops_f']
SETS = [dict(method0='wmc', method1='auto', hard_dc=-1, decompose_dc=-2, search_all_decompose_dc=False),
        dict(method0='mc', method1='auto', hard_dc=2, decompose_dc=-2, search_all_decompose_dc=False),
        dict(method0='wmc-dc', method1='auto', hard_dc=1, decompose_dc=-2, search_all_decompose_dc=False)]  # fmt: skip
CUTOFFS = [3.0, 5.0]


def digest(stages) -> str:
    """sha256 of a design's stage arrays (int64 index arrays, float32 ``ops_f``), stage by stage."""
    h = hashlib.sha256()
    for st in stages:
        for k in STAGE_KEYS:
            a = np.ascontiguousarray(np.asarray(st[k], np.float32 if k == 'ops_f' else np.int64))
            h.update(k.encode())
            h.update(str(a.shape).encode())
            h.update(a.tobytes())
    return h.hexdigest()


def seq_cost(stages) -> float:
    c = np.float32(0.0)  # one float accumulator over every stage, op order (the sweep's cost)
    for st in stages:
        for v in np.asarray(st['ops_f'], np.float32).reshape(-1, 5)[:, 4]:
            c = np.float32(c + v)
    return float(c)


def latency_max(stages) -> float:
    last = stages[-1]
    ops_f = np.asarray(last['ops_f'], np.float32).reshape(-1, 5)
    return float(max(ops_f[i, 3] for i in np.asarray(last['out_idxs'], np.int64).tolist()))  # (Pipeline.latency: -1 is the last op)


def models():
    """(name, kernels, adder_size, carry_size, layer-0 intervals, activations)."""
    rng = np.random.default_rng(2024)
    W = lambda n, m, lo=-8, hi=8: rng.integers(lo, hi, size=(n, m)).astype(np.float32)  # noqa: E731
    out = []
    # a relu that saturates every value (the next layer's intervals do not depend on the design), then a wide quantizer
    # that passes design-dependent intervals on
    out.append(('saturating_relu_wide_quantize_6x8x6x4', [W(6, 8), W(8, 6), W(6, 4)], -1, -1, [(-8.0, 7.0, 1.0)] * 6,
                [('relu', [(0, 2, 0)] * 8), ('quantize', [(1, 14, 0)] * 6)]))
    # a relu that passes design-dependent intervals on, then a signed WRAP quantizer that drops integer bits
    out.append(('relu_wrap_8x6x5x3', [W(8, 6, -12, 12), W(6, 5), W(5, 3)], -1, -1, [(-4.0, 3.75, 0.25) if i % 2 else (0.0, 7.5, 0.5) for i in range(8)],
                [('relu', [(0, 12, 1)] * 6), ('quantize', [(1, 4, 0)] * 5)]))
    # per-output kif with one value left with no bits (k + i + f <= 0): a dead input of the next layer
    out.append(('per_output_dead_value_6x5x4', [W(6, 5), W(5, 4)], 1, -1, [(-16.0, 15.0, 1.0)] * 6,
                [('quantize', [(1, 9, 0), (0, 0, 0), (1, 3, 1), (1, 12, -1), (0, 6, 0)])]))
    return out


def main():
    import ref_trace
    from oracle import oracle_solve
    from oracle import port

    from da4ml_b200.types import pipeline_from_arrays

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

    out = []
    for name, kernels, a_sz, c_sz, q0, acts in models():
        traces = []
        for choice in itertools.product(range(len(SETS)), repeat=len(kernels)):
            for cut in CUTOFFS:
                calls.clear()
                q = np.asarray(q0, np.float64)
                x = FVA.from_lhs(q[:, 0], q[:, 1], q[:, 2], hwconf=FV.HWConfig(a_sz, c_sz, cut))
                rec = dict(choice=list(choice), cutoff=cut)
                try:
                    for k, W in enumerate(kernels):
                        x.solver_options = dict(SETS[choice[k]])
                        x = x @ W
                        if k < len(acts):
                            kind, kif = acts[k]
                            kif = np.asarray(kif, np.int64)
                            x = x.relu(kif[:, 1], kif[:, 2]) if kind == 'relu' else x.quantize(kif[:, 0], kif[:, 1], kif[:, 2])
                except AssertionError:
                    rec['raised'] = True
                else:
                    rec['raised'] = False
                    rec['out_latency'] = [float(v.latency) for v in x._vars.ravel()]
                rec['calls'] = [dict(c) for c in calls]
                traces.append(rec)
        out.append(dict(name=name, kernels=[W.tolist() for W in kernels], adder_size=a_sz, carry_size=c_sz, qintervals=[list(r) for r in q0],
                        activations=[[kind, np.asarray(kif, np.int64).tolist()] for kind, kif in acts], traces=traces))  # fmt: skip
    raw = json.dumps({'sets': SETS, 'cutoffs': CUTOFFS, 'models': out}, separators=(',', ':')).encode()
    with gzip.GzipFile(HERE / 'chain_traced.json.gz', 'wb', mtime=0) as f:
        f.write(raw)
    n = sum(len(m['traces']) for m in out)
    print(len(out), 'models,', n, 'traces,', sum(t['raised'] for m in out for t in m['traces']), 'raised,', (HERE / 'chain_traced.json.gz').stat().st_size // 1024, 'KiB')


if __name__ == '__main__':
    main()
