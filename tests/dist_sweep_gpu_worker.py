"""Worker of tests/test_sweep_batch_gpu.py::test_sweep_sharded_two_ranks_nccl (one process per GPU under
torch.distributed.run, NCCL): option sweeps of the BASELINE config 5 stand-in stack through sweep_sharded, gathered on every
rank, against solve_sweep_batch of the whole stack on one GPU."""
import os
import sys
from pathlib import Path

import numpy as np
import torch
import torch.distributed as dist

ROOT = Path(__file__).resolve().parents[1]
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / 'tests'))

from conftest import int_matrix  # noqa: E402
from test_sweep_batch_gpu import assert_same_sweep  # noqa: E402

import da4ml_b200._binary as B  # noqa: E402
from da4ml_b200.cmvm import network_front  # noqa: E402
from da4ml_b200.distributed import sweep_sharded  # noqa: E402


def main():
    rank, world, local = int(os.environ['RANK']), int(os.environ['WORLD_SIZE']), int(os.environ['LOCAL_RANK'])
    torch.cuda.set_device(local)
    dist.init_process_group('nccl', rank=rank, world_size=world)
    B.set_stream(torch.cuda.current_stream().cuda_stream)
    shapes = [(16, 64), (64, 64), (64, 32), (32, 32), (32, 5)]
    layers = [int_matrix(a, b, 6, 40 + i) for i, (a, b) in enumerate(shapes)]
    rng = np.random.default_rng(7)
    qs = [[(-float(2 ** rng.integers(1, 7)), float(2 ** rng.integers(1, 7)) - 1.0, 1.0) for _ in range(a)] for a, _ in shapes]
    ls = [[float(v) for v in rng.integers(0, 2, a)] for a, _ in shapes]
    sets = [dict(method0=m, hard_dc=h) for m in ('wmc', 'mc') for h in (-1, 0, 2)]
    got = sweep_sharded(layers, sets, qintervals=qs, latencies=ls)  # gathered on every rank
    assert len(got) == len(layers)
    want = B.solve_sweep_batch(layers, sets, qintervals=qs, latencies=ls)
    for p, (a, b) in enumerate(zip(got, want, strict=True)):
        assert_same_sweep(a, b, f'layer {p}')
    nf, nf1 = network_front(got), network_front(want)
    assert np.array_equal(nf.cost, nf1.cost) and np.array_equal(nf.latency, nf1.latency) and np.array_equal(nf.choice, nf1.choice)
    if rank == 0:
        print(f'SWEEP_DIST_OK world={world} front={len(nf)}', flush=True)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == '__main__':
    main()
