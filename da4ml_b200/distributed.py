"""Multi-GPU sharding of independent CMVM problems (one process per GPU, ``torch.distributed``).

The path shards at the grain the reference itself parallelises: independent constant matrices (every
``cmvm()`` call of a traced model, reference trace/fixed_variable_array.py:368-371) -- there is no exchange step
between them, so no data-path collective is issued during the solve.  Each rank solves its share on its own
GPU; the variable-length adder graphs are gathered afterwards with one ``all_gather_object`` (NCCL or gloo).
``sweep_sharded`` does the same for option sweeps of many matrices.
"""

from __future__ import annotations

from collections.abc import Callable, Sequence

import numpy as np


_PER_PROBLEM = ('qintervals', 'latencies')  # options that are lists with one entry per problem


def problem_weight(kernel: np.ndarray) -> float:
    """Work estimate used for balancing: the greedy loop scales roughly with (non-zero digits)^2."""
    k = np.asarray(kernel)
    nnz = float(np.count_nonzero(k)) * max(1.0, np.log2(1.0 + float(np.abs(k).max(initial=0.0))))
    return nnz * nnz


def shard_assignment(weights: Sequence[float], world_size: int) -> list[list[int]]:
    """Longest-processing-time-first assignment of problem indices to ranks (deterministic)."""
    order = sorted(range(len(weights)), key=lambda i: (-weights[i], i))
    loads = [0.0] * world_size
    shards: list[list[int]] = [[] for _ in range(world_size)]
    for i in order:
        r = min(range(world_size), key=lambda j: (loads[j], j))
        shards[r].append(i)
        loads[r] += weights[i]
    return [sorted(s) for s in shards]


def solve_sharded(kernels: Sequence[np.ndarray], solver: Callable | None = None, group=None, gather: bool = True, **opts):
    """Solve ``kernels`` across the ranks of ``group`` (default: WORLD).

    ``solver(list_of_kernels, **opts) -> list_of_results`` defaults to the CUDA batch solver.  Returns the full,
    input-ordered result list on every rank (``gather=True``) or only this rank's ``{index: result}``.
    """
    import torch.distributed as dist

    if solver is None:
        from ._binary import solve_batch_raw as solver  # noqa: PLC0415
    if dist.is_available() and dist.is_initialized():
        rank, world = dist.get_rank(group), dist.get_world_size(group)
    else:
        rank, world = 0, 1
    shards = shard_assignment([problem_weight(k) for k in kernels], world)
    mine = shards[rank]
    # per-problem option lists travel with their problems (the batch solver indexes them by local position)
    local_opts = {k: ([v[i] for i in mine] if k in _PER_PROBLEM and v is not None else v) for k, v in opts.items()}
    for k in _PER_PROBLEM:
        if opts.get(k) is not None and len(opts[k]) != len(kernels):
            raise ValueError(f'expected {len(kernels)} entries in {k}, got {len(opts[k])}')
    local = solver([kernels[i] for i in mine], **local_opts) if mine else []
    local_map = dict(zip(mine, local))
    if not gather or world == 1:
        return [local_map[i] for i in range(len(kernels))] if world == 1 else local_map
    gathered: list = [None] * world
    dist.all_gather_object(gathered, local_map, group=group)
    merged = {}
    for part in gathered:
        merged.update(part)
    return [merged[i] for i in range(len(kernels))]


def sweep_sharded(kernels: Sequence[np.ndarray], option_sets: Sequence[dict], group=None, gather: bool = True, solver: Callable | None = None, **kw):
    """Sweep ``kernels`` under ``option_sets`` across the ranks of ``group``: ``solve_sharded``'s assignment and gather
    around ``solver(list_of_kernels, option_sets, **kw) -> list_of_results`` (default ``solve_sweep_batch``, one GPU pass
    per rank).  Per-matrix ``qintervals`` / ``latencies`` travel with their matrices; gathered ``SweepResult``s are
    detached copies (see ``SweepResult``)."""
    if solver is None:
        from ._binary import solve_sweep_batch as solver  # noqa: PLC0415
    return solve_sharded(kernels, solver=lambda ks, **o: solver(ks, option_sets, **o), group=group, gather=gather, **kw)
