"""Developer A/B run (under gpurun): time one build of the library on the bench workload and print a digest of the result."""
import hashlib, os, sys, time
import numpy as np
sys.path.insert(0, '.')
import da4ml_b200._binary as B

def mat(n, bits, seed):
    rng = np.random.default_rng(seed)
    return rng.integers(-2 ** (bits - 1), 2 ** (bits - 1), size=(n, n)).astype(np.float32)

def digest(raw):
    h = hashlib.sha1()
    for st in raw.stages:
        for k in ('inp_shifts', 'out_idxs', 'out_shifts', 'out_negs', 'ops_i', 'ops_f'):
            h.update(np.ascontiguousarray(st[k]).tobytes())
    return h.hexdigest()[:12]

tag = sys.argv[1]
B.solve_single_raw(mat(8, 4, 0))
W = mat(int(os.environ.get('SIZE', '256')), int(os.environ.get('BITS', '8')), 0)  # SIZE / BITS: the stage matrix (default: the bench workload)
G = int(sys.argv[2]) if len(sys.argv) > 2 else 22  # the planner's group size for the bench stage
B.set_group_size(G)
raw, _ = B.solve_single_raw(W, 'wmc')
c = raw.counters[0]
T = max(c['T'], 1)
c2 = None
# SM cycles per us, from this run: CTA 0's cycles in the greedy loop (its serial phase timers 0, 3, 1, 4, 5, 7; team R's
# phase 2 runs beside team C and the poll 6 is part of 7) over the stage's device time.  The stage also spends a little
# time outside the loop, so this slightly underestimates the clock.
mhz = sum(c['phase_cycles'][k] for k in (0, 1, 3, 4, 5, 7)) / (1e3 * raw.device_ms)
cyc = mhz  # cycles per us
print(f'{tag}: clock {mhz:.0f} MHz (CTA-0 loop cycles / stage device time), T={T}', flush=True)
line = f'{tag}: stage G={G} {raw.device_ms:.1f} ms us/step={1e3*raw.device_ms/T:.1f} phases={[round(v/cyc/T,2) for v in c["phase_cycles"]]} max-over-CTAs={[round(v/cyc/T,2) for v in c["phase_cycles_max"]]} dig={digest(raw)}'
prev = [0] * 10
for k, v in sorted(c['milestones'].items()):
    d = [a - b for a, b in zip(v, prev)]
    steps = k - (k // 2 if k > 250 else 0)
    # team R: its warps' share of the recount's first pass, counted once their refresh is done (CTA 0's last warp)
    print(f'  steps ..{k}: {d[9]/cyc/1e3:.1f} ms, {d[9]/cyc/steps:.1f} us/step, phase us/step={[round(x/cyc/steps,2) for x in d[:8]]} team R counting us/step={d[8]/cyc/steps:.2f}', flush=True)
    prev = v
B.set_group_size(0)
if os.environ.get('QUICK'):  # the stage only
    print(line, flush=True)
    sys.exit(0)
ms = []
for _ in range(2):
    raw = B.solve_raw(W)
    ms.append(raw.device_ms)
line += f' | solve {min(ms):.1f} ms adders={raw.n_adders} dig={digest(raw)}'
W6 = [mat(128, 6, s) for s in range(16)]
t0 = time.time(); rs = B.solve_batch_raw(W6); t1 = time.time()
line += f' | batch16x128x6 wall {1e3*(t1-t0):.0f} ms adders={[r.n_adders for r in rs][:3]}'
print(line, flush=True)
