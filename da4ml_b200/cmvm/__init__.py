"""``da4ml_b200.cmvm`` -- the public face of the solver, name-compatible with the reference's ``da4ml.cmvm``
(reference ``src/da4ml/cmvm/__init__.py``: ``solve``, ``kernel_decompose``, ``QInterval``, ``Op``, ``CombLogic`` and the
``solver_options_t`` keyword bundle that tracing code splats into ``solve``).  ``solve_batch`` / ``solve_calls`` are the
GPU-side additions for many independent matrices, ``solve_sweep`` for one matrix under many option sets,
``solve_sweep_batch`` for many matrices under many option sets, ``network_front`` for the cheapest per-layer choice of a
chain of layers under a latency budget, and ``chain_front`` for the same with each layer solved under the output latencies
of the design before it (the designs and latencies a traced model gets; with ``activations=`` also under the intervals
the relu / quantizers between the layers hand each layer).  ``solve``'s ``seed`` keyword picks the
tie-break order of the greedy pair selection (0 = the reference's), and ``solve_best_of`` keeps the cheapest of many seeds.
``price_pipelined`` prices designs as they will be pipelined under a latency cutoff: clock stages, register bits and the
tracer's latencies; ``chain_design`` joins a chain's designs, with the relu / quantizers between its layers, into one
design that it prices and splits as one pipeline."""

from typing import TypedDict

from .._binary import (ChainFront, NetworkFront, PipelinePrice, SweepResult, chain_design, chain_front, kernel_decompose, network_front, price_pipelined, solve, solve_batch,
                       solve_best_of, solve_sweep, solve_sweep_batch)  # fmt: skip
from ..batching import CmvmCall, SolveBatcher, solve_calls
from ..types import CombLogic, Op, Pipeline, QInterval

# keyword bundle accepted by solve(); every key is optional.  `offload_fn(constant_matrix, variables) -> bool mask`
# is consumed by the tracing front-end before the solver is called (weights it selects go to multipliers).
solver_options_t = TypedDict(
    'solver_options_t',
    {
        'method0': str,
        'method1': str,
        'hard_dc': int,
        'decompose_dc': int,
        'adder_size': int,
        'carry_size': int,
        'search_all_decompose_dc': bool,
        'seed': int,
        'offload_fn': object,
    },
    total=False,
)

__all__ = ['solve', 'solve_batch', 'solve_best_of', 'solve_sweep', 'solve_sweep_batch', 'SweepResult', 'network_front', 'NetworkFront', 'chain_front', 'ChainFront', 'chain_design', 'price_pipelined', 'PipelinePrice', 'solve_calls', 'CmvmCall', 'SolveBatcher', 'kernel_decompose', 'QInterval', 'Op', 'CombLogic', 'Pipeline', 'solver_options_t']
