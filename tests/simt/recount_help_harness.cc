// recount_help_harness.cc -- TEST INFRASTRUCTURE ONLY: the simulator harness of sim_cmvm.cc with the solve kernel wrapped,
// so that the counters of team R's part in the recount (META_HELPED, META_HELPED_OVF), which that harness does not copy
// out, can be read after a launch (tests/test_kernel_sim_recount_help.py).
#include "simt.h"

#include "../../da4ml_b200/csrc/cmvm_kernel_own.cuh"

namespace {
long long g_helped[2] = {0, 0};
const da::ProblemDesc *g_launch = nullptr; // the launch being counted (its problem table)
long long g_left = 0;                      // simulated threads of that launch that have left the kernel
} // namespace

// Every simulated thread runs this in place of the kernel; the last one to leave sums the counters over the jobs.
void cmvm_solve_kernel_counted(const da::ProblemDesc *probs, int n_probs, const da::GroupWs *wss, const da::OwnWs *ows, da::LaunchCfg cfg, int n_out_max, int e_cap_max, int lcap, int hlog, int narrow) {
    da::cmvm_solve_kernel(probs, n_probs, wss, ows, cfg, n_out_max, e_cap_max, lcap, hlog, narrow);
    if (probs != g_launch) {
        g_launch = probs;
        g_left = 0;
    }
    if (++g_left == (long long)gridDim.x * blockDim.x) {
        g_helped[0] = g_helped[1] = 0;
        for (int i = 0; i < n_probs; ++i) {
            g_helped[0] += probs[i].result_meta[da::META_HELPED];
            g_helped[1] += probs[i].result_meta[da::META_HELPED_OVF];
        }
        g_launch = nullptr;
    }
}
#define cmvm_solve_kernel cmvm_solve_kernel_counted
#include "sim_cmvm.cc"

// Of the last launch, summed over its jobs: chunks of 32 recount items team R claimed, and first recount passes abandoned
// for want of hash slots after team R had claimed chunks of them.
extern "C" void sim_helped(long long out[2]) {
    out[0] = g_helped[0];
    out[1] = g_helped[1];
}
