// pipeline_price_harness.cc -- TEST INFRASTRUCTURE ONLY.  The product's pipelined-pricing kernel and host code
// (da4ml_b200/csrc/pipeline_price.cuh: pp_prepare, pipeline_price_kernel, pp_price with its retiming bisection) compiled
// with g++ under the SIMT shim, behind the argument layout of da4ml_pipeline_price, so that the CPU tests can compare the
// kernel's answers with stored reference answers without a GPU.  `threads` is the CTA size of every launch.
#include "simt.h"

#include "../../da4ml_b200/csrc/pipeline_price.cuh"

using namespace da;

static std::string g_err;

extern "C" {
const char *pph_last_error() { return g_err.c_str(); }

int pph_price(int64_t n_designs, const int64_t *n_stages, const int64_t *stage_meta, const int64_t *inp_shifts, const int64_t *out_idxs, const int64_t *out_shifts,
              const int64_t *out_negs, const int64_t *ops_i, const float *ops_f, const double *latencies, const double *cutoffs, int64_t n_cutoffs, int retiming,
              int threads, int32_t *status, int64_t *stages, int64_t *reg_bits, double *latency_max, double *cutoff_out, double *out_latency, int64_t *launches) {
    try {
        std::vector<PpPrepared> prep(n_designs);
        std::vector<int64_t> lat_off(n_designs);
        int64_t s0 = 0, o_in = 0, o_out = 0, o_ops = 0, lat_n = 0;
        for (int64_t d = 0; d < n_designs; ++d) {
            std::vector<PpStageIn> st(n_stages[d]);
            for (int64_t k = 0; k < n_stages[d]; ++k, ++s0) {
                const int64_t *m = stage_meta + 5 * s0;
                PpStageIn &S = st[k];
                S.n_in = m[0], S.n_out = m[1], S.n_ops = m[2], S.carry_size = m[3], S.adder_size = m[4];
                S.inp_shifts = inp_shifts + o_in, S.out_idxs = out_idxs + o_out, S.out_shifts = out_shifts + o_out, S.out_negs = out_negs + o_out;
                S.ops_i = ops_i + 4 * o_ops, S.ops_f = ops_f + 5 * o_ops;
                o_in += S.n_in, o_out += S.n_out, o_ops += S.n_ops;
            }
            prep[d] = pp_prepare(st.data(), n_stages[d]);
            lat_off[d] = lat_n;
            lat_n += prep[d].n_in;
        }
        std::vector<PpDesign> desc(n_designs);
        for (int64_t d = 0; d < n_designs; ++d) {
            const PpPrepared &P = prep[d];
            desc[d] = PpDesign{P.adds.data(), P.lvl_begin.data(), P.node_bits.data(), P.out_node.data(), P.n_in, P.n_nodes, (int)P.adds.size(),
                               (int)P.lvl_begin.size() - 1, P.n_out, P.adder_size, P.carry_size, 0, P.out_bits};
        }
        const int64_t n_tasks = n_designs * n_cutoffs;
        // the workspaces start as garbage, as device memory does
        std::vector<std::vector<double>> ws(n_tasks), olat(n_tasks);
        for (int64_t t = 0; t < n_tasks; ++t) {
            const PpPrepared &P = prep[t / n_cutoffs];
            ws[t].assign(P.n_nodes + (P.n_nodes + 1) / 2, -12345.678);
            olat[t].assign(P.n_out, -1.0);
        }
        *launches = 0;
        bool first = true;
        auto run = [&](const std::vector<PpRequest> &req, std::vector<PpResult> &res) {
            std::vector<PpTask> tasks(req.size());
            for (size_t k = 0; k < req.size(); ++k) {
                const PpRequest &q = req[k];
                PpTask &T = tasks[k];
                T.design = q.design;
                T.cutoff = q.cutoff;
                T.in_lat = latencies && !q.zero_latency ? latencies + lat_off[q.design] : nullptr;
                T.lat = ws[q.slot].data();
                T.last_use = (int *)(T.lat + prep[q.design].n_nodes);
                T.out_lat = !q.zero_latency ? olat[q.slot].data() : nullptr;
            }
            res.assign(req.size(), PpResult{});
            simt::launch(dim3((unsigned)req.size()), dim3((unsigned)threads), 0, [&] { pipeline_price_kernel(desc.data(), tasks.data(), res.data()); }, 64 * 1024);
            ++*launches;
            if (first)
                for (int64_t t = 0, o = 0; t < n_tasks; ++t)
                    for (int k = 0; k < prep[t / n_cutoffs].n_out; ++k, ++o)
                        out_latency[o] = res[t].status == PP_OK ? olat[t][k] : nan("");
            first = false;
        };
        const std::vector<PpAnswer> ans = pp_price((int)n_designs, cutoffs, (int)n_cutoffs, retiming != 0, run);
        for (int64_t t = 0; t < n_tasks; ++t) {
            status[t] = ans[t].status;
            stages[t] = ans[t].stages;
            reg_bits[t] = ans[t].reg_bits;
            latency_max[t] = ans[t].latency_max;
            cutoff_out[t] = ans[t].status == PP_OK ? ans[t].cutoff : nan("");
        }
        return 0;
    }
    catch (const std::exception &e) {
        g_err = e.what();
        return 1;
    }
}
}
