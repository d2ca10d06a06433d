// pipeline_split_harness.cc -- TEST INFRASTRUCTURE ONLY.  The product's split kernels and host code
// (da4ml_b200/csrc/pipeline_split.cuh: ps_prepare, pipeline_split_kernel, pipeline_split_write_kernel, ps_split, on top of
// pipeline_price.cuh's pp_prepare, pipeline_price_kernel and pp_price) compiled with g++ under the SIMT shim, behind the
// argument layout of da4ml_pipeline_split, so that the CPU tests can compare splits with stored reference splits
// without a GPU.  `threads` is the CTA size of every launch.
#include "simt.h"

#include "../../da4ml_b200/csrc/pipeline_split.cuh"

using namespace da;

static std::string g_err;
static PsResult g_split;

namespace {
struct SimDev { // ps_split's device: host memory, launches under the shim; buffers start as garbage, as device memory does
    int threads = 64;
    std::vector<std::vector<char>> buf = std::vector<std::vector<char>>(3);
    char *buffer(int which, size_t bytes) {
        buf[which].assign(bytes + 16, (char)0x5a);
        return buf[which].data();
    }
    void up(void *dst, const void *src, size_t bytes) { std::memcpy(dst, src, bytes); }
    void down(void *dst, const void *src, size_t bytes) { std::memcpy(dst, src, bytes); }
    void count(const PsDesign *d, const PsTask *t, int n) { simt::launch(dim3((unsigned)n), dim3((unsigned)threads), 0, [&] { pipeline_split_kernel(d, t); }, 64 * 1024); }
    void write(const PsDesign *d, const PsTask *t, int n) { simt::launch(dim3((unsigned)n), dim3((unsigned)threads), 0, [&] { pipeline_split_write_kernel(d, t); }, 64 * 1024); }
};
} // namespace

extern "C" {
const char *psh_last_error() { return g_err.c_str(); }

// pricing (as da4ml_pipeline_price) and the split of every ok task; the splits stay in g_split for psh_info / psh_copy
int psh_split(int64_t n_designs, const int64_t *n_stages, const int64_t *stage_meta, const int64_t *inp_shifts, const int64_t *out_idxs, const int64_t *out_shifts,
              const int64_t *out_negs, const int64_t *ops_i, const float *ops_f, const double *latencies, const double *cutoffs, int64_t n_cutoffs, int retiming,
              int threads, int32_t *status, int64_t *stages, int64_t *reg_bits, double *latency_max, double *cutoff_out, int64_t *launches) {
    try {
        std::vector<PpPrepared> prep(n_designs);
        std::vector<PsPrep> sp(n_designs);
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
            PpSplitInfo info;
            prep[d] = pp_prepare(st.data(), n_stages[d], &info);
            sp[d] = ps_prepare(prep[d], info);
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
        std::vector<std::vector<double>> ws(n_tasks);
        for (int64_t t = 0; t < n_tasks; ++t)
            ws[t].assign(prep[t / n_cutoffs].n_nodes + (prep[t / n_cutoffs].n_nodes + 1) / 2, -12345.678);
        *launches = 0;
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
                T.out_lat = nullptr;
            }
            res.assign(req.size(), PpResult{});
            simt::launch(dim3((unsigned)req.size()), dim3((unsigned)threads), 0, [&] { pipeline_price_kernel(desc.data(), tasks.data(), res.data()); }, 64 * 1024);
            ++*launches;
        };
        const std::vector<PpAnswer> ans = pp_price((int)n_designs, cutoffs, (int)n_cutoffs, retiming != 0, run);
        for (int64_t t = 0; t < n_tasks; ++t) {
            status[t] = ans[t].status;
            stages[t] = ans[t].stages;
            reg_bits[t] = ans[t].reg_bits;
            latency_max[t] = ans[t].latency_max;
            cutoff_out[t] = ans[t].status == PP_OK ? ans[t].cutoff : nan("");
        }
        SimDev dev;
        dev.threads = threads;
        g_split = ps_split(prep, sp, desc, ans, cutoffs, n_cutoffs, retiming != 0, latencies, latencies, lat_off, dev);
        *launches += g_split.launches;
        return 0;
    }
    catch (const std::exception &e) {
        g_err = e.what();
        return 1;
    }
}

void psh_info(int64_t t, int64_t out[4]) { ps_info(g_split, t, out); }

void psh_copy(int64_t t, int64_t *meta, int64_t *out_idxs, int64_t *out_shifts, int64_t *out_negs, int64_t *ops_i, double *ops_f) {
    ps_copy(g_split, t, meta, out_idxs, out_shifts, out_negs, ops_i, ops_f);
}
}
