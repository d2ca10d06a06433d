// sim_seeded.cc -- TEST INFRASTRUCTURE ONLY: the SIMT harness of tests/simt/sim_cmvm.cc (included unmodified) with a
// tie-break seed per job.  sim_seed_set(seeds, n) fixes the seeds of the jobs of the next sim_solve_single /
// sim_solve_many call (job i gets seeds[i], jobs beyond n seed 0); the harness's own launch of cmvm_solve_kernel is
// routed through seeded_solve_kernel, which writes tb_mask(seed) into each job's ProblemDesc before the kernel reads it.
#include "../simt/simt.h"

#include "../../da4ml_b200/csrc/cmvm_decompose.cuh"
#include "../../da4ml_b200/csrc/cmvm_kernel_own.cuh"
#include "../../da4ml_b200/csrc/host_plan.cuh"

#include <vector>

static std::vector<unsigned long long> g_seed_masks;

// Every simulated thread enters the solve kernel through here.  The threads are fibers of one OS thread that switch
// only at barriers and polls, so the first one to arrive writes every job's mask before any thread reads a descriptor;
// the later ones write the same values again.
static void seeded_solve_kernel(da::ProblemDesc *probs, int n_probs, const da::GroupWs *wss, const da::OwnWs *ows, da::LaunchCfg cfg, int n_out_max, int e_cap_max,
                                int lcap, int hlog, int narrow) {
    for (int i = 0; i < n_probs; ++i)
        probs[i].tb_mask = i < (int)g_seed_masks.size() ? g_seed_masks[i] : 0ull;
    da::cmvm_solve_kernel(probs, n_probs, wss, ows, cfg, n_out_max, e_cap_max, lcap, hlog, narrow);
}

#define cmvm_solve_kernel seeded_solve_kernel
#include "../simt/sim_cmvm.cc"
#undef cmvm_solve_kernel

extern "C" void sim_seed_set(const uint64_t *seeds, int n) {
    g_seed_masks.assign(n, 0ull);
    for (int i = 0; i < n; ++i)
        g_seed_masks[i] = da::tb_mask(seeds[i]);
}
