"""Throughput of the DAIS interpreter (da4ml_b200.dais) on the GPU, with the hardware it ran on.

  python scripts/dev_dais_perf.py [--samples N] [--ref-samples N] [--dump-samples N] [--parent-lib PATH] [--out FILE]

Programs: the largest traced fixture (tests/golden/dais_programs.json.gz, ``traced_mlp``) and the stage-0 adder graph
of a 256x256 int8 solve.  For each: samples/s of the device path (inputs and outputs resident, CUDA events around one
call), and bytes moved per the buffer model (8 B per operand read plus 8 B per result write, per op and sample) over
that time, against the H100 SXM data-sheet HBM bandwidth (3.35 TB/s).  In the same loop, alternated with the run:
``DaisProgram.profile`` on the same inputs (its time and the ratio to the run), and for the traced MLP the all-ops
``DaisProgram.dump`` of the first --dump-samples samples, in GB/s written.  The reference interpreter
(oracle/_ref/libdais_ref.so) runs on all host cores in the same process, one thread per core over sample chunks as the
reference's OpenMP loop does.  With --parent-lib (a libda4ml_b200_cmvm.so built from an earlier revision), the adder
graph is also replayed by that library's da4ml_dais_run and this one's, alternated, timing the kernels with
torch.profiler.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import threading
import time
from pathlib import Path

import numpy as np

ROOT = Path(__file__).resolve().parents[1]
sys.path[:0] = [str(ROOT), str(ROOT / 'tests')]

HBM_TBS = 3.35  # H100 SXM5 80 GB data sheet


def gpu_info():
    import torch

    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True, timeout=30)
        smi = q.stdout.strip().splitlines()[0]
    except Exception as e:  # (reading only)
        smi = f'nvidia-smi unavailable: {e}'
    return dict(torch_name=name, nvidia_smi=smi)


def buffer_bytes(prog) -> float:
    """8 B per operand read + 8 B per result write, per op and sample."""
    n_in, n_out, n_ops = int(prog[2]), int(prog[3]), int(prog[4])
    ops = np.asarray(prog[6 + n_in + 3 * n_out : 6 + n_in + 3 * n_out + 8 * n_ops]).reshape(-1, 8)
    reads = {-1: 1, 5: 0, 0: 2, 1: 2, 6: 3, -6: 3, 7: 2, 10: 2}
    return float(sum(8 * (reads.get(int(o), 1) + 1) for o in ops[:, 0]))


def time_device(prog, x_np, reps=5, dump_samples=0):
    """Device seconds {call: [reps]} of a run, a profile and (dump_samples > 0) an all-ops dump of that many samples,
    alternated; and the run's outputs."""
    import torch

    from da4ml_b200.dais import DaisProgram

    p = DaisProgram(prog)
    x = torch.from_numpy(x_np).cuda()
    calls = dict(run=lambda: p(x), profile=lambda: p.profile(x))
    if dump_samples:
        calls['dump'] = lambda: p.dump(x[:dump_samples])
    for fn in calls.values():  # (uploads the program, grows the scratch)
        fn()
    torch.cuda.synchronize()
    ts = {k: [] for k in calls}
    for _ in range(reps):
        for k, fn in calls.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            out = fn()
            b.record()
            torch.cuda.synchronize()
            ts[k].append(a.elapsed_time(b) / 1e3)
            if k == 'run':
                y = out
            del out
    p.close()
    return ts, y


def time_reference(prog, x, threads):
    from oracle import dais_ref

    dais_ref.run(prog, x[:64])
    parts = np.array_split(x, threads)
    outs = [None] * threads

    def work(i):
        outs[i] = dais_ref.run(prog, parts[i])

    t0 = time.perf_counter()
    th = [threading.Thread(target=work, args=(i,)) for i in range(threads)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    return time.perf_counter() - t0, np.concatenate(outs)


def kernel_seconds(fn):
    """Sum of the device time of the dais_* kernels launched by fn()."""
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
    return sum(e.device_time_total for e in prof.key_averages() if 'dais_' in e.key) / 1e6


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--samples', type=int, default=1_000_000)
    ap.add_argument('--ref-samples', type=int, default=200_000, help='0 skips the reference interpreter')
    ap.add_argument('--dump-samples', type=int, default=100_000)
    ap.add_argument('--parent-lib', default='')
    ap.add_argument('--out', default='')
    a = ap.parse_args()

    import dais_programs as G
    from test_oracle_cross import load_stored

    import da4ml_b200._binary as B

    res = dict(gpu=gpu_info(), host_cores=len(os.sched_getaffinity(0)), samples=a.samples, hbm_tbs_datasheet=HBM_TBS, programs={})
    z = load_stored('dais_programs.json.gz')
    mlp = z['words/traced_mlp'].astype(np.int32)
    W = np.random.default_rng(0).integers(-128, 128, size=(256, 256)).astype(np.float32)
    adder = B.solve(W, search_all_decompose_dc=False, decompose_dc=-1).solutions[0].to_binary()
    for name, prog, x in (
        ('traced_mlp', mlp, G.random_inputs(11, a.samples, int(mlp[2]))),
        ('adder_256x256_stage0', adder, np.random.default_rng(1).integers(-128, 128, size=(a.samples, 256)).astype(np.float64)),
    ):
        ts, y = time_device(prog, x, dump_samples=min(a.dump_samples, a.samples) if name == 'traced_mlp' else 0)
        med, best = float(np.median(ts['run'])), float(min(ts['run']))
        nb = buffer_bytes(prog) * a.samples
        r = dict(n_ops=int(prog[4]), n_in=int(prog[2]), n_out=int(prog[3]), device_s_median=med, device_s_best=best, samples_per_s=a.samples / med,
                 buffer_bytes=nb, buffer_tbs=nb / med / 1e12, hbm_fraction=nb / med / 1e12 / HBM_TBS, run_s=ts['run'], profile_s=ts['profile'],
                 profile_s_median=float(np.median(ts['profile'])), profile_over_run=float(np.median(ts['profile'])) / med)  # fmt: skip
        if 'dump' in ts:
            n_dump = min(a.dump_samples, a.samples)
            t = float(np.median(ts['dump']))
            r.update(dump_samples=n_dump, dump_s=ts['dump'], dump_s_median=t, dump_gbs_written=n_dump * int(prog[4]) * 8 / t / 1e9)
        n_ref = min(a.ref_samples, a.samples)
        if n_ref:
            t_ref, y_ref = time_reference(prog, x[:n_ref], res['host_cores'])
            same = bool(np.array_equal(y[:n_ref].cpu().numpy().view(np.uint64), y_ref.view(np.uint64)))
            r.update(ref_samples=n_ref, ref_s=t_ref, ref_samples_per_s=n_ref / t_ref, ref_equal=same)
        res['programs'][name] = r
        print(name, json.dumps(r), flush=True)
    if a.parent_lib:
        import torch

        old = C.CDLL(a.parent_lib)
        dp = C.POINTER(C.c_double)
        for L in (old, B._L):
            L.da4ml_dais_run.argtypes = [C.POINTER(C.c_int32), C.c_int64, dp, C.c_int64, dp]
        prog = np.ascontiguousarray(adder)
        x = np.random.default_rng(1).integers(-128, 128, size=(a.samples, 256)).astype(np.float64)
        outs = {}

        def run(L, tag):
            y = np.zeros((a.samples, int(prog[3])), np.float64)
            rc = L.da4ml_dais_run(prog.ctypes.data_as(C.POINTER(C.c_int32)), prog.size, x.ctypes.data_as(dp), a.samples, y.ctypes.data_as(dp))
            assert rc == 0, tag
            outs[tag] = y

        run(old, 'parent')
        run(B._L, 'this')
        torch.cuda.synchronize()
        rounds = []
        for _ in range(3):
            rounds.append(dict(parent=kernel_seconds(lambda: run(old, 'parent')), this=kernel_seconds(lambda: run(B._L, 'this'))))
        res['adder_parent_vs_this'] = dict(rounds=rounds, equal=bool(np.array_equal(outs['parent'].view(np.uint64), outs['this'].view(np.uint64))))
        print('parent vs this (kernel s):', json.dumps(res['adder_parent_vs_this']), flush=True)
    if a.out:
        Path(a.out).parent.mkdir(parents=True, exist_ok=True)
        Path(a.out).write_text(json.dumps(res, indent=1))


if __name__ == '__main__':
    main()
