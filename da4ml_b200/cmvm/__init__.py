"""``da4ml_b200.cmvm`` -- the public face of the solver, name-compatible with the reference's ``da4ml.cmvm``
(reference ``src/da4ml/cmvm/__init__.py``: ``solve``, ``kernel_decompose``, ``QInterval``, ``Op``, ``CombLogic`` and the
``solver_options_t`` keyword bundle that tracing code splats into ``solve``).  ``solve_batch`` / ``solve_calls`` are the
GPU-side additions for many independent matrices."""

from typing import TypedDict

from .._binary import kernel_decompose, solve, solve_batch
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
        'offload_fn': object,
    },
    total=False,
)

__all__ = ['solve', 'solve_batch', 'solve_calls', 'CmvmCall', 'SolveBatcher', 'kernel_decompose', 'QInterval', 'Op', 'CombLogic', 'Pipeline', 'solver_options_t']
