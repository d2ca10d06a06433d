"""Developer profile of BASELINE config 4 (64 x 128x128 int6 default solves in one batch) under gpurun: wall time, launch profile and the
in-kernel phase timers of the stage-0 jobs, for the planner's group size and for pinned ones (GS=1,2,4)."""
import os, sys, time
import numpy as np
sys.path.insert(0, '.')
import da4ml_b200._binary as B

def mat(n, bits, seed):
    rng = np.random.default_rng(seed)
    return rng.integers(-2 ** (bits - 1), 2 ** (bits - 1), size=(n, n)).astype(np.float32)

nb = int(os.environ.get('NB', '64'))
ks = [mat(128, 6, s) for s in range(nb)]
B.solve_batch_raw(ks[:2])
for G in [int(g) for g in os.environ.get('GS', '0,1,2,4').split(',')]:
    B.set_group_size(G)
    t0 = time.time(); res = B.solve_batch_raw(ks); dt = time.time() - t0
    r = res[0]
    c = r.counters[0]
    T = max(c['T'], 1)
    ph = [round(v / 1.9e3 / T, 2) for v in c['phase_cycles']]
    print(f'G={G or "auto"}: {nb} x 128x128 int6 wall {dt*1e3:.0f} ms = {nb/dt:.1f} matrices/s | profile {r.profile} | job 0 stage 0: G={c["group_ctas"]} T={T} lcap={c["smem_list_cap"]} '
          f'phases us/step {ph} sum {sum(ph[:2]) + sum(ph[3:6]) + ph[7]:.1f} | stage 1: T={r.counters[1]["T"]} G={r.counters[1]["group_ctas"]}', flush=True)
    ms = c['milestones']
    prev = [0] * 10
    for k, v in sorted(ms.items()):
        d = [a - b for a, b in zip(v, prev)]
        steps = k - (k // 2 if k > 250 else 0)
        print(f'    steps ..{k}: {d[9]/1.9e3/steps:.1f} us/step, phases {[round(x/1.9e3/steps,1) for x in d[:8]]}, team R counting {d[8]/1.9e3/steps:.1f}')
        prev = v
B.set_group_size(0)
