// cmvm_lib.cu -- host driver and C ABI (include/da4ml_b200_cmvm.h) of the GPU-native CMVM solver.
//
// Host-side control mirrors the reference's api.cc: `solve` (candidate search over decompose_dc,
// api.cc:147-250) and `_solve` (two-stage driver with the latency-retry loop, api.cc:28-145).  The
// reference parallelises the candidates with OpenMP; here all pending solve_single jobs of all
// candidates (and of all problems of a batch) are solved concurrently by one persistent kernel
// launch per round.  All arithmetic of the path runs in the kernels of cmvm_kernels.cuh /
// cmvm_decompose.cuh; nothing here falls back to the CPU.
#include "dais_program.cuh"
#include "host_solve.cuh"
#include "pipeline_split.cuh"

namespace da {

// small export kernels for the helper entry points ------------------------------------------------
__global__ void csd_export_kernel(const uint2 *masks, int n, int nbits, int8_t *csd) {
    int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n)
        return;
    uint2 m = masks[idx];
    for (int k = 0; k < nbits; ++k)
        csd[(size_t)idx * nbits + k] = (int8_t)(((m.x >> k) & 1) - ((m.y >> k) & 1));
}
// plain digits without centring: the matrix is interpreted as already integer (bit_decompose.cc:22-42)
__global__ void int_csd_kernel(const int *x, int n, int nbits, int8_t *csd) {
    int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n)
        return;
    int32_t v = x[idx];
    for (int k = nbits - 1; k >= 0; --k)
        csd[(size_t)idx * nbits + k] = (int8_t)csd_digit_i32(v, k);
}
__global__ void int_absmax_kernel(const int *x, int n, int *out) {
    int idx = blockIdx.x * blockDim.x + threadIdx.x;
    int v = idx < n ? csd_abs(x[idx]) : 0;
    for (int off = 16; off > 0; off >>= 1)
        v = max(v, __shfl_xor_sync(0xffffffffu, v, off));
    if ((threadIdx.x & 31) == 0 && v)
        atomicMax(out, v);
}
__global__ void float_to_int_kernel(const float *x, int n, int *out) {
    int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx < n)
        out[idx] = trunc_i32(x[idx]);
}

} // namespace da

// ================================================================================================
using namespace da;

struct da4ml_pipeline {
    std::unique_ptr<PipelineImpl> impl;
};

struct da4ml_split {
    PsResult r;
};
struct da4ml_sweep {
    std::unique_ptr<SweepImpl> impl;
};

// ---- DAIS interpreter engine ------------------------------------------------------------------------------------------
// A loaded program: the validated host form plus its device copy (ops, level order, header arrays, table offsets and
// tables), uploaded on first use on a device and kept until the handle is freed.
struct da4ml_dais_program {
    DaisProgramHost h;
    int device = -1;
    char *d_mem = nullptr;
    size_t o_ops = 0, o_ord = 0, o_hdr = 0, o_toff = 0, o_tab = 0;
    da4ml_dais_program() = default;
    da4ml_dais_program(const da4ml_dais_program &) = delete;
    ~da4ml_dais_program() {
        if (d_mem)
            cudaFree(d_mem);
    }
};

namespace da {

static void dais_upload(da4ml_dais_program &P, cudaStream_t st) {
    int dev = 0;
    CK(cudaGetDevice(&dev));
    if (P.d_mem && P.device == dev)
        return;
    if (P.d_mem)
        cudaFree(P.d_mem);
    P.d_mem = nullptr;
    const DaisProgramHost &h = P.h;
    Carver c;
    P.o_ops = c.take(sizeof(DaisOp) * h.ops.size());
    P.o_ord = c.take(sizeof(int) * h.order.size());
    P.o_hdr = c.take(sizeof(int32_t) * h.header.size());
    P.o_toff = c.take(sizeof(long long) * h.table_off.size());
    P.o_tab = c.take(sizeof(int32_t) * h.tables.size());
    CK(cudaMalloc(&P.d_mem, std::max<size_t>(c.off, 256)));
    P.device = dev;
    auto up = [&](size_t off, const void *src, size_t bytes) {
        if (bytes)
            CK(cudaMemcpyAsync(P.d_mem + off, src, bytes, cudaMemcpyHostToDevice, st));
    };
    up(P.o_ops, h.ops.data(), sizeof(DaisOp) * h.ops.size());
    up(P.o_ord, h.order.data(), sizeof(int) * h.order.size());
    up(P.o_hdr, h.header.data(), sizeof(int32_t) * h.header.size());
    up(P.o_toff, h.table_off.data(), sizeof(long long) * h.table_off.size());
    up(P.o_tab, h.tables.data(), sizeof(int32_t) * h.tables.size());
}

// What a pass over the samples produces from each chunk's buffer after its last level: the program's outputs (run), the
// codes of selected ops (dump), or per-op statistics of every op's codes (profile).
enum class DaisPass { run, dump, profile };
struct DaisRequest {
    DaisPass pass = DaisPass::run;
    const int32_t *sel = nullptr; // dump: op ids [n_sel], host memory
    int64_t n_sel = 0;
    long long *stats = nullptr;   // profile: [n_ops][3] int64 host = {min, max, bitwise OR}
};

// Run a program on n_samples rows on stream st.  Samples are processed in chunks that keep the [n_ops][S] int64 buffer
// around 1 GB; with device_ptrs the inputs / outputs are read and written in place, otherwise they are staged through
// device buffers.  `outputs` holds 8-byte rows of n_out doubles (run) or n_sel int64 codes (dump); a profile has none and
// copies its statistics to the host once, after the last chunk.  A lookup out of range stops the run after its chunk
// with the reference's message for the first failing (sample, op).
//
// Every run shares one scratch buffer, and a run on device pointers without lookups returns before its kernels finish.
// Runs are therefore put in one order on the device whatever streams they come on: each run's stream first waits for the
// event the previous run recorded after its last use of the scratch, and records it again after its own.  (A newly
// uploaded program copy is written on the run's stream ahead of its kernels, so it is covered too, as are the selected op
// ids and the statistics accumulators, which live in the scratch.)
static void dais_execute(da4ml_dais_program &P, const double *inputs, int64_t n_samples, void *outputs, bool device_ptrs, cudaStream_t st,
                         const DaisRequest &req = DaisRequest()) {
    const DaisPass pass = req.pass;
    if (n_samples == 0) {
        for (int i = 0; pass == DaisPass::profile && i < P.h.n_ops; ++i) {
            req.stats[3LL * i] = LLONG_MAX;
            req.stats[3LL * i + 1] = LLONG_MIN;
            req.stats[3LL * i + 2] = 0;
        }
        return;
    }
    init_device();
    static cudaEvent_t scratch_free = nullptr; // recorded after the last run's final use of `work`
    static int scratch_dev = -1;
    if (scratch_dev != g_device) { // (a device change dropped every cached buffer, synchronising with the old device)
        if (scratch_free)
            cudaEventDestroy(scratch_free);
        scratch_free = nullptr;
        CK(cudaEventCreateWithFlags(&scratch_free, cudaEventDisableTiming));
        CK(cudaEventRecord(scratch_free, st));
        scratch_dev = g_device;
    }
    CK(cudaStreamWaitEvent(st, scratch_free, 0));
    dais_upload(P, st);
    const DaisProgramHost &h = P.h;
    const int n_in = h.n_in, n_out = h.n_out, n_ops = h.n_ops;
    // columns of an output row (8 bytes each); a dump with more columns than ops takes smaller chunks, so its staged
    // output stays the size of the buffer
    const long long n_cols = pass == DaisPass::run ? n_out : pass == DaisPass::dump ? req.n_sel : 0;
    const long long S_max = std::max<long long>(256, (1LL << 27) / std::max<long long>({1, n_ops, pass == DaisPass::dump ? n_cols : 0}));
    const long long S = std::min<long long>(n_samples, S_max);
    static DevBuf work;
    Carver c;
    const size_t o_in = c.take(device_ptrs ? 0 : sizeof(double) * S * n_in), o_out = c.take(device_ptrs ? 0 : sizeof(double) * S * n_cols),
                 o_buf = c.take(sizeof(long long) * S * n_ops), o_err = c.take(sizeof(unsigned long long)),
                 o_sel = c.take(pass == DaisPass::dump ? sizeof(int32_t) * req.n_sel : 0), o_stats = c.take(pass == DaisPass::profile ? sizeof(long long) * 3 * n_ops : 0);
    if (c.off > work.cap)
        CK(cudaEventSynchronize(scratch_free)); // the old buffer is freed: no earlier run may still be using it
    work.ensure(c.off, false);
    char *b = (char *)work.p;
    const DaisOp *d_ops = (const DaisOp *)(P.d_mem + P.o_ops);
    const int *d_ord = (const int *)(P.d_mem + P.o_ord), *d_hdr = (const int *)(P.d_mem + P.o_hdr);
    const int *d_inp_shifts = d_hdr, *d_out_idxs = d_hdr + n_in, *d_out_shifts = d_out_idxs + n_out, *d_out_negs = d_out_shifts + n_out;
    long long *d_buf = (long long *)(b + o_buf);
    unsigned long long *d_err = (unsigned long long *)(b + o_err);
    const int *d_sel = (const int *)(b + o_sel);
    long long *d_stats = (long long *)(b + o_stats);
    std::vector<long long> stats(pass == DaisPass::profile ? 3 * (size_t)n_ops : 0);
    if (pass == DaisPass::dump && req.n_sel)
        CK(cudaMemcpyAsync(b + o_sel, req.sel, sizeof(int32_t) * req.n_sel, cudaMemcpyHostToDevice, st));
    if (pass == DaisPass::profile && n_ops)
        dais_stats_init_kernel<<<(n_ops + 255) / 256, 256, 0, st>>>(d_stats, n_ops);
    for (int64_t s0 = 0; s0 < n_samples; s0 += S) {
        const long long Sc = std::min<long long>(S, n_samples - s0);
        const double *d_in = device_ptrs ? inputs + s0 * n_in : (const double *)(b + o_in);
        char *d_out = device_ptrs ? (char *)outputs + 8 * s0 * n_cols : b + o_out;
        if (!device_ptrs && n_in)
            CK(cudaMemcpyAsync(b + o_in, inputs + s0 * n_in, sizeof(double) * Sc * n_in, cudaMemcpyHostToDevice, st));
        if (h.has_lookup)
            CK(cudaMemsetAsync(d_err, 0xff, sizeof(unsigned long long), st));
        for (int l = 0; l < h.n_levels; ++l) {
            const int n_l = h.lvl_begin[l + 1] - h.lvl_begin[l];
            const long long threads = (long long)n_l * Sc;
            auto *kernel = h.lvl_adder[l] ? dais_level_kernel<true> : dais_level_kernel<false>;
            kernel<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(
                d_ops, d_ord + h.lvl_begin[l], n_l, d_inp_shifts, d_in, n_in, Sc, d_buf, (const int32_t *)(P.d_mem + P.o_tab), (const long long *)(P.d_mem + P.o_toff), d_err
            );
        }
        if (pass == DaisPass::run && n_out) {
            const long long threads = (long long)n_out * Sc;
            dais_output_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(d_ops, d_out_idxs, d_out_shifts, d_out_negs, n_out, Sc, d_buf, (double *)d_out);
        }
        if (pass == DaisPass::dump && n_cols) {
            const long long tiles = (n_cols + 31) / 32;
            dais_dump_kernel<<<dim3((unsigned)((Sc + 31) / 32), (unsigned)std::min<long long>(tiles, 65535)), dim3(32, 8), 0, st>>>(d_buf, Sc, d_sel, n_cols, (long long *)d_out);
        }
        if (pass == DaisPass::profile && n_ops) {
            const long long per_block = (long long)kDaisStatsThreads * kDaisStatsPerThread;
            dais_stats_kernel<<<dim3((unsigned)n_ops, (unsigned)std::min<long long>((Sc + per_block - 1) / per_block, 65535)), kDaisStatsThreads, 0, st>>>(d_buf, Sc, d_stats);
            if (s0 + Sc == n_samples) // the accumulators leave the scratch before the event below frees it
                CK(cudaMemcpyAsync(stats.data(), d_stats, sizeof(long long) * 3 * n_ops, cudaMemcpyDeviceToHost, st));
        }
        CK(cudaGetLastError());
        if (!device_ptrs && n_cols)
            CK(cudaMemcpyAsync((char *)outputs + 8 * s0 * n_cols, d_out, 8 * Sc * n_cols, cudaMemcpyDeviceToHost, st));
        if (h.has_lookup) {
            unsigned long long key = 0;
            CK(cudaMemcpyAsync(&key, d_err, sizeof(key), cudaMemcpyDeviceToHost, st));
            CK(cudaEventRecord(scratch_free, st));
            CK(cudaStreamSynchronize(st));
            if (key != ~0ull) {
                const long long s = (long long)(key >> 32);
                const int i = (int)(key & 0xffffffffu);
                long long v0 = 0;
                CK(cudaMemcpyAsync(&v0, d_buf + (long long)h.ops[i].id0 * Sc + s, sizeof(v0), cudaMemcpyDeviceToHost, st));
                CK(cudaStreamSynchronize(st));
                throw ApiError(DA4ML_E_RUNTIME, dais_lookup_error(h, i, v0));
            }
        }
        else {
            CK(cudaEventRecord(scratch_free, st));
            if (!device_ptrs || (pass == DaisPass::profile && s0 + Sc == n_samples))
                CK(cudaStreamSynchronize(st));
        }
    }
    if (pass == DaisPass::profile) // (only once every chunk passed its lookup check)
        std::copy(stats.begin(), stats.end(), req.stats);
}

} // namespace da

template <class F> static int guarded(F &&f) {
    try {
        std::lock_guard<std::mutex> lock(g_mutex);
        f();
        return DA4ML_OK;
    }
    catch (const ApiError &e) {
        g_err = e.what();
        return e.code;
    }
    catch (const std::exception &e) {
        g_err = e.what();
        return DA4ML_E_RUNTIME;
    }
}

extern "C" {

const char *da4ml_cmvm_last_error(void) { return g_err.c_str(); }

int da4ml_cmvm_device_info(int32_t out[5]) {
    out[0] = 1;
    out[1] = out[2] = out[3] = out[4] = 0;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess) {
        cudaGetLastError();
        return DA4ML_OK;
    }
    out[1] = ndev;
    if (ndev > 0) {
        int dev = 0;
        cudaDeviceProp prop;
        if (cudaGetDevice(&dev) == cudaSuccess && cudaGetDeviceProperties(&prop, dev) == cudaSuccess) {
            out[2] = prop.multiProcessorCount;
            out[3] = prop.major;
            out[4] = prop.minor;
        }
    }
    return DA4ML_OK;
}

int da4ml_cmvm_plan(const int64_t *jobs, int64_t n_jobs, int coop, int group_override, int64_t out[12]) {
    return guarded([&]() -> int {
        if (!jobs || !out || n_jobs <= 0 || coop <= 0)
            throw ApiError(DA4ML_E_INVALID, "da4ml_cmvm_plan: bad arguments");
        std::vector<PlanJob> pj((size_t)n_jobs);
        for (int64_t i = 0; i < n_jobs; ++i) {
            const int64_t *r = jobs + 8 * i;
            if (r[0] <= 0 || r[1] <= 0 || r[2] <= 0 || r[6] <= 0 || r[7] <= 0)
                throw ApiError(DA4ML_E_INVALID, "da4ml_cmvm_plan: bad job row");
            pj[i].n_in = (int)r[0];
            pj[i].n_out = (int)r[1];
            pj[i].nbits = (int)r[2];
            pj[i].d0 = r[3];
            pj[i].dcol_max = (int)r[4];
            pj[i].col_cap = (int)r[5];
            pj[i].f_mul = (int)r[6];
            pj[i].list_mul = (int)r[7];
            pj[i].e_cap = (int)(r[0] + std::min<long long>(r[3], r[3] / 2 + 1024) + 1); // as run_stage_jobs sizes it
        }
        PlanEnv env;
        env.coop = coop;
        env.group_override = group_override;
        const LaunchPlan P = plan_launch(pj, env);
        out[0] = P.cfg.G;
        out[1] = P.n_groups;
        out[2] = P.cfg.cpc;
        out[3] = P.lcap;
        out[4] = P.cfg.chunk_log;
        out[5] = P.cfg.nchunk_cap;
        out[6] = P.max_fcap;
        out[7] = P.hlog;
        out[8] = (int64_t)P.smem_bytes;
        out[9] = env.own_budget;
        out[10] = P.narrow;
        out[11] = P.ovf_cap;
        return DA4ML_OK;
    });
}

int da4ml_cmvm_set_stream(void *s) {
    g_stream = (cudaStream_t)s;
    return DA4ML_OK;
}
int da4ml_cmvm_set_group_size(int g) {
    g_group_override = g;
    return DA4ML_OK;
}
// Free every device / pinned buffer the library keeps between calls (they are re-grown on demand).
int da4ml_cmvm_release(void) {
    return guarded([&] {
        release_device_buffers();
        for (PinBuf *b : {&g_pin_up, &g_pin_down}) {
            if (b->p)
                cudaFreeHost(b->p);
            b->p = nullptr;
            b->cap = 0;
        }
    });
}
int da4ml_cmvm_set_job_sharing(int on) {
    g_share_jobs = on != 0;
    return DA4ML_OK;
}
int da4ml_cmvm_set_accounting(int on) {
    g_accounting = on;
    return DA4ML_OK;
}

int da4ml_cmvm_solve_batch(
    int64_t n_problems, const float *const *kernels, const int64_t *n_in, const int64_t *n_out, const char *method0,
    const char *method1, int hard_dc, int decompose_dc, const float *const *qintervals, const float *const *latencies,
    int adder_size, int carry_size, int search_all, da4ml_pipeline_t **out
) {
    return guarded([&] {
        if (n_problems <= 0 || !kernels || !n_in || !n_out || !out || !method0 || !method1)
            throw ApiError(DA4ML_E_INVALID, "invalid argument");
        std::vector<std::unique_ptr<PipelineImpl>> res;
        solve_many(n_problems, kernels, n_in, n_out, {SolveOptions{method0, method1, hard_dc, decompose_dc, search_all != 0}}, qintervals, latencies, adder_size, carry_size, res);
        for (int64_t i = 0; i < n_problems; ++i) {
            out[i] = new da4ml_pipeline();
            out[i]->impl = std::move(res[i]);
        }
    });
}

int da4ml_cmvm_solve_batch_device(
    int64_t n_problems, const float *const *kernels_dev, const int64_t *n_in, const int64_t *n_out, const char *method0,
    const char *method1, int hard_dc, int decompose_dc, const float *const *qintervals, const float *const *latencies,
    int adder_size, int carry_size, int search_all, da4ml_pipeline_t **out
) {
    return guarded([&] {
        if (n_problems <= 0 || !kernels_dev || !n_in || !n_out || !out || !method0 || !method1)
            throw ApiError(DA4ML_E_INVALID, "invalid argument");
        std::vector<std::unique_ptr<PipelineImpl>> res;
        solve_many(n_problems, kernels_dev, n_in, n_out, {SolveOptions{method0, method1, hard_dc, decompose_dc, search_all != 0}}, qintervals, latencies, adder_size, carry_size, res, true);
        for (int64_t i = 0; i < n_problems; ++i) {
            out[i] = new da4ml_pipeline();
            out[i]->impl = std::move(res[i]);
        }
    });
}

int da4ml_cmvm_solve_seeded(
    const float *kernel, int64_t n_in, int64_t n_out, const char *method0, const char *method1, int hard_dc, int decompose_dc,
    const float *qintervals, const float *latencies, int adder_size, int carry_size, int search_all, uint64_t seed, da4ml_pipeline_t **out
) {
    return guarded([&] {
        if (!kernel || !out || !method0 || !method1)
            throw ApiError(DA4ML_E_INVALID, "invalid argument");
        const float *ks[1] = {kernel};
        const float *qs[1] = {qintervals};
        const float *ls[1] = {latencies};
        SolveOptions o{method0, method1, hard_dc, decompose_dc, search_all != 0};
        o.seed = seed;
        std::vector<std::unique_ptr<PipelineImpl>> res;
        solve_many(1, ks, &n_in, &n_out, {o}, qs, ls, adder_size, carry_size, res);
        *out = new da4ml_pipeline();
        (*out)->impl = std::move(res[0]);
    });
}

int da4ml_cmvm_solve(
    const float *kernel, int64_t n_in, int64_t n_out, const char *method0, const char *method1, int hard_dc, int decompose_dc,
    const float *qintervals, const float *latencies, int adder_size, int carry_size, int search_all, da4ml_pipeline_t **out
) {
    return da4ml_cmvm_solve_seeded(kernel, n_in, n_out, method0, method1, hard_dc, decompose_dc, qintervals, latencies, adder_size, carry_size, search_all, 0, out);
}

int da4ml_cmvm_solve_single(
    const float *kernel, int64_t n_in, int64_t n_out, const char *method, const float *qintervals, const float *latencies,
    int adder_size, int carry_size, int32_t *trace, int64_t trace_cap, da4ml_pipeline_t **out
) {
    return da4ml_cmvm_solve_single_seeded(kernel, n_in, n_out, method, qintervals, latencies, adder_size, carry_size, trace, trace_cap, 0, out);
}

int da4ml_cmvm_solve_single_seeded(
    const float *kernel, int64_t n_in, int64_t n_out, const char *method, const float *qintervals, const float *latencies,
    int adder_size, int carry_size, int32_t *trace, int64_t trace_cap, uint64_t seed, da4ml_pipeline_t **out
) {
    return guarded([&] {
        if (!kernel || n_in <= 0 || n_out <= 0 || !method || !out)
            throw ApiError(DA4ML_E_INVALID, "invalid argument");
        init_device();
        static DevBuf kbuf;
        static PinBuf kpin;
        size_t bytes = sizeof(float) * (size_t)n_in * n_out;
        kbuf.ensure(bytes, false);
        kpin.ensure(bytes);
        memcpy(kpin.p, kernel, bytes);
        CK(cudaMemcpyAsync(kbuf.p, kpin.p, bytes, cudaMemcpyHostToDevice, g_stream));
        StageJob j;
        j.n_in = (int)n_in;
        j.n_out = (int)n_out;
        j.method = parse_method(method);
        j.adder_size = adder_size;
        j.carry_size = carry_size;
        j.seed = seed;
        j.d_kernel = (const float *)kbuf.p;
        j.qint.resize(3 * (size_t)n_in);
        j.lat.resize(n_in);
        for (int64_t i = 0; i < n_in; ++i) { // cmvm_core.cc:18-32 defaults
            j.qint[3 * i + 0] = qintervals ? qintervals[3 * i + 0] : -128.0f;
            j.qint[3 * i + 1] = qintervals ? qintervals[3 * i + 1] : 127.0f;
            j.qint[3 * i + 2] = qintervals ? qintervals[3 * i + 2] : 1.0f;
            j.lat[i] = latencies ? latencies[i] : 0.0f;
        }
        j.trace = trace;
        j.trace_cap = trace ? trace_cap : 0;
        Timing tm;
        std::vector<StageJob *> jobs{&j};
        g_out_arena2.reset();
        run_stage_jobs(jobs, tm, true);
        auto pl = std::make_unique<PipelineImpl>();
        pl->stages.push_back(std::move(j.res));
        pl->device_ms = tm.device_ms;
        pl->launches = tm.launches;
        pl->solve_ms = tm.solve_ms;
        pl->solve_launches = tm.solve_launches;
        pl->algo_bytes = tm.algo_bytes;
        *out = new da4ml_pipeline();
        (*out)->impl = std::move(pl);
    });
}

// ---- sweep: many matrices under many option sets ---------------------------------------------------
int da4ml_cmvm_solve_sweep_batch(
    int64_t n_problems, const float *const *kernels, const int64_t *n_in, const int64_t *n_out, const float *const *qintervals,
    const float *const *latencies, int adder_size, int carry_size, int64_t n_sets, const char *const *method0, const char *const *method1,
    const int32_t *hard_dc, const int32_t *decompose_dc, const int32_t *search_all, int keep_all, da4ml_sweep_t **out
) {
    return da4ml_cmvm_solve_sweep_batch_seeded(n_problems, kernels, n_in, n_out, qintervals, latencies, adder_size, carry_size, n_sets, method0, method1, hard_dc,
                                               decompose_dc, search_all, nullptr, keep_all, out);
}

int da4ml_cmvm_solve_sweep_batch_seeded(
    int64_t n_problems, const float *const *kernels, const int64_t *n_in, const int64_t *n_out, const float *const *qintervals,
    const float *const *latencies, int adder_size, int carry_size, int64_t n_sets, const char *const *method0, const char *const *method1,
    const int32_t *hard_dc, const int32_t *decompose_dc, const int32_t *search_all, const uint64_t *seed, int keep_all, da4ml_sweep_t **out
) {
    return guarded([&] {
        if (n_problems <= 0)
            throw ApiError(DA4ML_E_INVALID, "solve_sweep: n_problems must be positive (got " + std::to_string(n_problems) + ")");
        if (!kernels || !n_in || !n_out)
            throw ApiError(DA4ML_E_INVALID, "solve_sweep: a kernel array is null");
        for (int64_t p = 0; p < n_problems; ++p) // (a lone matrix needs no name)
            if (!kernels[p] || n_in[p] <= 0 || n_out[p] <= 0)
                throw ApiError(DA4ML_E_INVALID, n_problems == 1 ? std::string("solve_sweep: kernel must be a non-empty 2D array")
                                                                : "solve_sweep: kernel " + std::to_string(p) + " must be a non-empty 2D array");
        if (n_sets <= 0)
            throw ApiError(DA4ML_E_INVALID, "solve_sweep: n_sets must be positive (got " + std::to_string(n_sets) + ")");
        if (!method0 || !method1 || !hard_dc || !decompose_dc || !search_all)
            throw ApiError(DA4ML_E_INVALID, "solve_sweep: an option array is null");
        if (!out)
            throw ApiError(DA4ML_E_INVALID, "solve_sweep: out is null");
        std::vector<SolveOptions> sets((size_t)n_sets);
        for (int64_t s = 0; s < n_sets; ++s) {
            if (!method0[s] || !method1[s])
                throw ApiError(DA4ML_E_INVALID, "solve_sweep: a method of option set " + std::to_string(s) + " is null");
            sets[s] = SolveOptions{method0[s], method1[s], hard_dc[s], decompose_dc[s], search_all[s] != 0};
            sets[s].seed = seed ? seed[s] : 0;
            parse_method(sets[s].method0); // "Unknown method: ..." before any device call
            if (sets[s].method1 != "auto")
                parse_method(sets[s].method1);
        }
        std::vector<SweepImpl> sweeps;
        std::vector<std::unique_ptr<PipelineImpl>> winners;
        solve_many(n_problems, kernels, n_in, n_out, sets, qintervals, latencies, adder_size, carry_size, winners, false, &sweeps, keep_all != 0);
        std::vector<std::unique_ptr<da4ml_sweep>> res((size_t)n_problems); // (all results exist before any is handed out)
        for (int64_t p = 0; p < n_problems; ++p)
            res[p].reset(new da4ml_sweep{std::make_unique<SweepImpl>(std::move(sweeps[p]))});
        for (int64_t p = 0; p < n_problems; ++p)
            out[p] = res[p].release();
    });
}

int da4ml_cmvm_solve_sweep(
    const float *kernel, int64_t n_in, int64_t n_out, const float *qintervals, const float *latencies, int adder_size, int carry_size, int64_t n_sets,
    const char *const *method0, const char *const *method1, const int32_t *hard_dc, const int32_t *decompose_dc, const int32_t *search_all, int keep_all,
    da4ml_sweep_t **out
) {
    return da4ml_cmvm_solve_sweep_batch(1, &kernel, &n_in, &n_out, &qintervals, &latencies, adder_size, carry_size, n_sets, method0, method1, hard_dc,
                                        decompose_dc, search_all, keep_all, out);
}

int da4ml_sweep_counts(const da4ml_sweep_t *s, int64_t out[4]) {
    if (!s || !out)
        return DA4ML_E_INVALID;
    out[0] = s->impl->n_sets;
    out[1] = (int64_t)s->impl->cands.size();
    out[2] = (int64_t)std::count_if(s->impl->kept.begin(), s->impl->kept.end(), [](const std::unique_ptr<PipelineImpl> &p) { return p != nullptr; });
    out[3] = s->impl->n_solved;
    return DA4ML_OK;
}

int da4ml_sweep_profile(const da4ml_sweep_t *s, double out[8]) {
    if (!s || !out)
        return DA4ML_E_INVALID;
    const PipelineImpl &t = s->impl->totals;
    const double row[8] = {t.device_ms, (double)t.launches, t.solve_ms, (double)t.solve_launches, t.algo_bytes, (double)t.jobs_total, (double)t.jobs_run, 0.0};
    std::copy(row, row + 8, out);
    return DA4ML_OK;
}

int da4ml_sweep_summary(const da4ml_sweep_t *s, int64_t *ints, float *floats) {
    if (!s)
        return DA4ML_E_INVALID;
    for (size_t i = 0; i < s->impl->cands.size(); ++i) {
        const CandidateSummary &c = s->impl->cands[i];
        if (ints) {
            const int64_t row[12] = {c.set, c.hard_dc, c.decompose_dc_start, c.method0, c.method1, c.decompose_dc, c.n_adders, c.n_ops0, c.n_ops1, c.winner, c.front,
                                     s->impl->kept[i] != nullptr};
            std::copy(row, row + 12, ints + 12 * i);
        }
        if (floats) {
            floats[3 * i + 0] = c.cost;
            floats[3 * i + 1] = c.latency_min;
            floats[3 * i + 2] = c.latency_max;
        }
    }
    return DA4ML_OK;
}

int da4ml_sweep_pipeline(const da4ml_sweep_t *s, int64_t candidate, da4ml_pipeline_t **out) {
    return guarded([&] {
        if (!s || !out)
            throw ApiError(DA4ML_E_INVALID, "sweep_pipeline: invalid argument");
        const int64_t n = (int64_t)s->impl->cands.size();
        if (candidate < 0 || candidate >= n)
            throw ApiError(DA4ML_E_INVALID, "sweep_pipeline: candidate " + std::to_string(candidate) + " is out of range [0, " + std::to_string(n) + ")");
        if (!s->impl->kept[candidate])
            throw ApiError(DA4ML_E_INVALID, "sweep_pipeline: the op tables of candidate " + std::to_string(candidate) +
                                                " were not kept (only the winners and the front are, unless the sweep was run with keep_all)");
        *out = new da4ml_pipeline{std::make_unique<PipelineImpl>(*s->impl->kept[candidate])};
    });
}

void da4ml_sweep_free(da4ml_sweep_t *s) { delete s; }

int da4ml_sweep_front(const float *cost, const float *latency_max, int64_t n, int8_t *front) {
    if (n < 0 || (n > 0 && (!cost || !latency_max || !front)))
        return DA4ML_E_INVALID;
    pareto_front(cost, latency_max, n, front);
    return DA4ML_OK;
}

namespace {
// ps_split's device: the call's three cached buffers, launches on the library stream with CUDA-event timing
struct CudaSplitDev {
    int threads = 256;
    Timing *tm = nullptr;
    size_t bytes_down = 0;
    char *buffer(int which, size_t bytes) {
        static DevBuf bufs[3];
        bufs[which].ensure(bytes, false);
        return (char *)bufs[which].p;
    }
    void up(void *dst, const void *src, size_t bytes) {
        if (bytes)
            CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, g_stream));
    }
    void down(void *dst, const void *src, size_t bytes) {
        if (bytes)
            CK(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, g_stream));
        CK(cudaStreamSynchronize(g_stream));
    }
    void count(const PsDesign *d, const PsTask *t, int n) {
        tm->begin();
        pipeline_split_kernel<<<(unsigned)n, threads, 0, g_stream>>>(d, t);
        CK(cudaGetLastError());
        tm->end(1);
    }
    void write(const PsDesign *d, const PsTask *t, int n) {
        tm->begin();
        pipeline_split_write_kernel<<<(unsigned)n, threads, 0, g_stream>>>(d, t);
        CK(cudaGetLastError());
        tm->end(1);
    }
};
} // namespace

// da4ml_pipeline_price, and with `split` non-null da4ml_pipeline_split (profile then has 4 entries)
static int pipeline_price_impl(
    int64_t n_designs, const int64_t *n_stages, const int64_t *stage_meta, const int64_t *inp_shifts, const int64_t *out_idxs, const int64_t *out_shifts,
    const int64_t *out_negs, const int64_t *ops_i, const float *ops_f, const double *latencies, const double *cutoffs, int64_t n_cutoffs, int retiming,
    int32_t *status, int64_t *stages, int64_t *reg_bits, double *latency_max, double *cutoff_out, double *out_latency, double *profile, da4ml_split_t **split
) {
    return guarded([&] {
        if (n_designs < 1 || n_designs > (1 << 24) || !n_stages || !stage_meta)
            throw ApiError(DA4ML_E_INVALID, "pipeline_price: n_designs must be positive and the design arrays non-null");
        if (n_cutoffs < 1 || n_cutoffs > (1 << 16) || !cutoffs)
            throw ApiError(DA4ML_E_INVALID, "pipeline_price: at least one latency cutoff is needed");
        if (!status || !stages || !reg_bits || !latency_max || !cutoff_out)
            throw ApiError(DA4ML_E_INVALID, "pipeline_price: an output array is null");
        if (n_designs * n_cutoffs > (1 << 24))
            throw ApiError(DA4ML_E_INVALID, "pipeline_price: too many (design, cutoff) tasks");
        for (int64_t j = 0; j < n_cutoffs; ++j)
            if (!(cutoffs[j] > 0) || !std::isfinite(cutoffs[j]))
                throw ApiError(DA4ML_E_INVALID, "pipeline_price: latency cutoff " + std::to_string(j) + " is " + std::to_string(cutoffs[j]) +
                                                    "; it must be positive and finite (cutoff 0 is the unpipelined design the solver reports)");
        // host preparation of every design (all argument checks happen here, before the device is touched)
        std::vector<PpPrepared> prep(n_designs);
        std::vector<PpSplitInfo> info(split ? n_designs : 0);
        std::vector<int64_t> lat_off(n_designs);
        int64_t s0 = 0, o_in = 0, o_out = 0, o_ops = 0, lat_n = 0;
        for (int64_t d = 0; d < n_designs; ++d) {
            if (n_stages[d] < 1 || n_stages[d] > (1 << 16))
                throw ApiError(DA4ML_E_INVALID, "pipeline_price: design " + std::to_string(d) + " has " + std::to_string(n_stages[d]) + " stages");
            std::vector<PpStageIn> st(n_stages[d]);
            for (int64_t k = 0; k < n_stages[d]; ++k, ++s0) {
                const int64_t *m = stage_meta + 5 * s0;
                PpStageIn &S = st[k];
                S.n_in = m[0], S.n_out = m[1], S.n_ops = m[2], S.carry_size = m[3], S.adder_size = m[4];
                if (S.n_in < 0 || S.n_out < 0 || S.n_ops < 0)
                    throw ApiError(DA4ML_E_INVALID, "pipeline_price: design " + std::to_string(d) + " stage " + std::to_string(k) + " has a negative size");
                S.inp_shifts = inp_shifts ? inp_shifts + o_in : nullptr;
                S.out_idxs = out_idxs ? out_idxs + o_out : nullptr;
                S.out_shifts = out_shifts ? out_shifts + o_out : nullptr;
                S.out_negs = out_negs ? out_negs + o_out : nullptr;
                S.ops_i = ops_i ? ops_i + 4 * o_ops : nullptr;
                S.ops_f = ops_f ? ops_f + 5 * o_ops : nullptr;
                o_in += S.n_in, o_out += S.n_out, o_ops += S.n_ops;
            }
            try {
                prep[d] = pp_prepare(st.data(), n_stages[d], split ? &info[d] : nullptr);
            }
            catch (const std::invalid_argument &e) {
                throw ApiError(DA4ML_E_INVALID, std::string(e.what()) + " (design " + std::to_string(d) + ")");
            }
            lat_off[d] = lat_n;
            lat_n += prep[d].n_in;
        }
        if (latencies)
            for (int64_t i = 0; i < lat_n; ++i)
                if (!std::isfinite(latencies[i]) || latencies[i] < 0)
                    throw ApiError(DA4ML_E_INVALID, "pipeline_price: input latency " + std::to_string(i) + " is not a finite non-negative number");
        init_device();
        // one device buffer: the prepared designs, the input latencies, per task its workspace and output latencies,
        // the task list and the results
        const int64_t n_tasks = n_designs * n_cutoffs;
        Carver c;
        std::vector<size_t> o_add(n_designs), o_lvl(n_designs), o_bits(n_designs), o_onode(n_designs), o_ws(n_tasks), o_olat(n_tasks);
        for (int64_t d = 0; d < n_designs; ++d) {
            o_add[d] = c.take(sizeof(PpAdd) * prep[d].adds.size());
            o_lvl[d] = c.take(sizeof(int) * prep[d].lvl_begin.size());
            o_bits[d] = c.take(sizeof(int) * prep[d].node_bits.size());
            o_onode[d] = c.take(sizeof(int) * prep[d].out_node.size());
        }
        const size_t o_desc = c.take(sizeof(PpDesign) * n_designs), o_lat = c.take(sizeof(double) * lat_n);
        for (int64_t t = 0; t < n_tasks; ++t) {
            const PpPrepared &P = prep[t / n_cutoffs];
            o_ws[t] = c.take((sizeof(double) + sizeof(int)) * P.n_nodes);
            o_olat[t] = c.take(out_latency ? sizeof(double) * P.n_out : 0);
        }
        const size_t o_task = c.take(sizeof(PpTask) * n_tasks), o_res = c.take(sizeof(PpResult) * n_tasks);
        static DevBuf buf;
        buf.ensure(c.off, false);
        char *b = (char *)buf.p;
        std::vector<PpDesign> desc(n_designs);
        auto up = [&](size_t off, const void *src, size_t bytes) {
            if (bytes)
                CK(cudaMemcpyAsync(b + off, src, bytes, cudaMemcpyHostToDevice, g_stream));
        };
        for (int64_t d = 0; d < n_designs; ++d) {
            const PpPrepared &P = prep[d];
            up(o_add[d], P.adds.data(), sizeof(PpAdd) * P.adds.size());
            up(o_lvl[d], P.lvl_begin.data(), sizeof(int) * P.lvl_begin.size());
            up(o_bits[d], P.node_bits.data(), sizeof(int) * P.node_bits.size());
            up(o_onode[d], P.out_node.data(), sizeof(int) * P.out_node.size());
            desc[d] = PpDesign{(const PpAdd *)(b + o_add[d]), (const int *)(b + o_lvl[d]), (const int *)(b + o_bits[d]), (const int *)(b + o_onode[d]),
                               P.n_in, P.n_nodes, (int)P.adds.size(), (int)P.lvl_begin.size() - 1, P.n_out, P.adder_size, P.carry_size, 0, P.out_bits};
        }
        up(o_desc, desc.data(), sizeof(PpDesign) * n_designs);
        if (latencies)
            up(o_lat, latencies, sizeof(double) * lat_n);
        Timing tm;
        auto run = [&](const std::vector<PpRequest> &req, std::vector<PpResult> &res) {
            std::vector<PpTask> tasks(req.size());
            for (size_t k = 0; k < req.size(); ++k) {
                const PpRequest &q = req[k];
                const PpPrepared &P = prep[q.design];
                PpTask &T = tasks[k];
                T.design = q.design;
                T.pad = 0;
                T.cutoff = q.cutoff;
                T.in_lat = latencies && !q.zero_latency ? (const double *)(b + o_lat) + lat_off[q.design] : nullptr;
                T.lat = (double *)(b + o_ws[q.slot]);
                T.last_use = (int *)(T.lat + P.n_nodes);
                T.out_lat = out_latency && !q.zero_latency ? (double *)(b + o_olat[q.slot]) : nullptr;
            }
            up(o_task, tasks.data(), sizeof(PpTask) * tasks.size());
            tm.begin();
            pipeline_price_kernel<<<(unsigned)tasks.size(), 256, 0, g_stream>>>((const PpDesign *)(b + o_desc), (const PpTask *)(b + o_task), (PpResult *)(b + o_res));
            CK(cudaGetLastError());
            tm.end(1);
            res.resize(req.size());
            CK(cudaMemcpyAsync(res.data(), b + o_res, sizeof(PpResult) * req.size(), cudaMemcpyDeviceToHost, g_stream));
            CK(cudaStreamSynchronize(g_stream));
        };
        bool first = true;
        auto run_first = [&](const std::vector<PpRequest> &req, std::vector<PpResult> &res) {
            run(req, res);
            if (first && out_latency) { // the traced output latencies of the first pass (the tasks' own latencies)
                int64_t off = 0;
                for (int64_t t = 0; t < n_tasks; ++t) {
                    const int n_out = prep[t / n_cutoffs].n_out;
                    if (n_out)
                        CK(cudaMemcpyAsync(out_latency + off, b + o_olat[t], sizeof(double) * n_out, cudaMemcpyDeviceToHost, g_stream));
                    off += n_out;
                }
                CK(cudaStreamSynchronize(g_stream));
                for (int64_t t = 0, o = 0; t < n_tasks; ++t)
                    for (int k = 0; k < prep[t / n_cutoffs].n_out; ++k, ++o)
                        if (res[t].status != PP_OK)
                            out_latency[o] = nan("");
            }
            first = false;
        };
        const std::vector<PpAnswer> ans = pp_price((int)n_designs, cutoffs, (int)n_cutoffs, retiming != 0, run_first);
        std::unique_ptr<da4ml_split> sp_out;
        int64_t split_launches = 0;
        size_t split_bytes = 0;
        if (split) { // every ok task's split, at the (cutoff, latencies) it comes from
            std::vector<PsPrep> sp(n_designs);
            for (int64_t d = 0; d < n_designs; ++d)
                sp[d] = ps_prepare(prep[d], info[d]);
            CudaSplitDev dev;
            dev.tm = &tm;
            sp_out.reset(new da4ml_split{ps_split(prep, sp, desc, ans, cutoffs, n_cutoffs, retiming != 0, latencies, latencies ? (const double *)(b + o_lat) : nullptr,
                                                  lat_off, dev)});  // fmt: skip
            split_launches = sp_out->r.launches;
            split_bytes = sp_out->r.tables.size();
        }
        tm.collect();
        for (int64_t t = 0; t < n_tasks; ++t) {
            status[t] = ans[t].status;
            stages[t] = ans[t].stages;
            reg_bits[t] = ans[t].reg_bits;
            latency_max[t] = ans[t].latency_max;
            cutoff_out[t] = ans[t].status == PP_OK ? ans[t].cutoff : nan("");
        }
        if (profile) {
            profile[0] = tm.device_ms;
            profile[1] = (double)tm.launches;
            if (split)
                profile[2] = (double)split_launches, profile[3] = (double)split_bytes;
        }
        if (split)
            *split = sp_out.release();
    });
}

int da4ml_pipeline_price(
    int64_t n_designs, const int64_t *n_stages, const int64_t *stage_meta, const int64_t *inp_shifts, const int64_t *out_idxs, const int64_t *out_shifts,
    const int64_t *out_negs, const int64_t *ops_i, const float *ops_f, const double *latencies, const double *cutoffs, int64_t n_cutoffs, int retiming,
    int32_t *status, int64_t *stages, int64_t *reg_bits, double *latency_max, double *cutoff_out, double *out_latency, double profile[2]
) {
    return pipeline_price_impl(n_designs, n_stages, stage_meta, inp_shifts, out_idxs, out_shifts, out_negs, ops_i, ops_f, latencies, cutoffs, n_cutoffs, retiming, status,
                               stages, reg_bits, latency_max, cutoff_out, out_latency, profile, nullptr);
}

int da4ml_pipeline_split(
    int64_t n_designs, const int64_t *n_stages, const int64_t *stage_meta, const int64_t *inp_shifts, const int64_t *out_idxs, const int64_t *out_shifts,
    const int64_t *out_negs, const int64_t *ops_i, const float *ops_f, const double *latencies, const double *cutoffs, int64_t n_cutoffs, int retiming,
    int32_t *status, int64_t *stages, int64_t *reg_bits, double *latency_max, double *cutoff_out, double *out_latency, double profile[4], da4ml_split_t **out
) {
    if (!out)
        return guarded([] { throw ApiError(DA4ML_E_INVALID, "pipeline_split: the handle pointer is null"); });
    *out = nullptr;
    return pipeline_price_impl(n_designs, n_stages, stage_meta, inp_shifts, out_idxs, out_shifts, out_negs, ops_i, ops_f, latencies, cutoffs, n_cutoffs, retiming, status,
                               stages, reg_bits, latency_max, cutoff_out, out_latency, profile, out);
}

int da4ml_split_info(const da4ml_split_t *s, int64_t task, int64_t out[4]) {
    return guarded([&] {
        if (!s || !out)
            throw ApiError(DA4ML_E_INVALID, "split_info: the handle or the output array is null");
        if (task < 0 || task >= (int64_t)s->r.tasks.size())
            throw ApiError(DA4ML_E_INVALID, "split_info: task " + std::to_string(task) + " is out of range [0, " + std::to_string(s->r.tasks.size()) + ")");
        ps_info(s->r, task, out);
    });
}

int da4ml_split_copy(const da4ml_split_t *s, int64_t task, int64_t *stage_meta, int64_t *out_idxs, int64_t *out_shifts, int64_t *out_negs, int64_t *ops_i, double *ops_f) {
    return guarded([&] {
        if (!s)
            throw ApiError(DA4ML_E_INVALID, "split_copy: the handle is null");
        if (task < 0 || task >= (int64_t)s->r.tasks.size())
            throw ApiError(DA4ML_E_INVALID, "split_copy: task " + std::to_string(task) + " is out of range [0, " + std::to_string(s->r.tasks.size()) + ")");
        const PsSplit &S = s->r.tasks[task];
        if (S.status != PS_SPLIT)
            throw ApiError(DA4ML_E_INVALID, "split_copy: task " + std::to_string(task) + " has no split (da4ml_split_info status " + std::to_string(S.status) + ")");
        if (!stage_meta || !out_idxs || !out_shifts || !out_negs || (S.n_rows && (!ops_i || !ops_f)))
            throw ApiError(DA4ML_E_INVALID, "split_copy: an output array is null");
        ps_copy(s->r, task, stage_meta, out_idxs, out_shifts, out_negs, ops_i, ops_f);
    });
}

void da4ml_split_free(da4ml_split_t *s) { delete s; }

void da4ml_pipeline_free(da4ml_pipeline_t *p) { delete p; }
int64_t da4ml_pipeline_n_stages(const da4ml_pipeline_t *p) { return p ? (int64_t)p->impl->stages.size() : 0; }
int da4ml_pipeline_stage_meta(const da4ml_pipeline_t *p, int64_t s, int64_t meta[5]) {
    if (!p || s < 0 || s >= (int64_t)p->impl->stages.size())
        return DA4ML_E_INVALID;
    const StageResult &r = p->impl->stages[s];
    meta[0] = r.n_in;
    meta[1] = r.n_out;
    meta[2] = r.n_ops();
    meta[3] = r.carry_size;
    meta[4] = r.adder_size;
    return DA4ML_OK;
}
int da4ml_pipeline_stage_copy(
    const da4ml_pipeline_t *p, int64_t s, int64_t *inp_shifts, int64_t *out_idxs, int64_t *out_shifts, int64_t *out_negs,
    int64_t *ops_i, float *ops_f
) {
    if (!p || s < 0 || s >= (int64_t)p->impl->stages.size())
        return DA4ML_E_INVALID;
    const StageResult &r = p->impl->stages[s];
    if (inp_shifts)
        std::copy(r.inp_shifts.begin(), r.inp_shifts.end(), inp_shifts);
    if (out_idxs)
        std::copy(r.out_idxs.begin(), r.out_idxs.end(), out_idxs);
    if (out_shifts)
        std::copy(r.out_shifts.begin(), r.out_shifts.end(), out_shifts);
    if (out_negs)
        std::copy(r.out_negs.begin(), r.out_negs.end(), out_negs);
    const size_t n_ops = r.op_misc.size();
    if (ops_i)
        for (size_t k = 0; k < n_ops; ++k) {
            ops_i[4 * k + 0] = r.op_misc[k].x;
            ops_i[4 * k + 1] = r.op_misc[k].y;
            ops_i[4 * k + 2] = r.op_misc[k].z;
            ops_i[4 * k + 3] = r.op_misc[k].w;
        }
    if (ops_f)
        for (size_t k = 0; k < n_ops; ++k) {
            ops_f[5 * k + 0] = r.op_q[k].x;
            ops_f[5 * k + 1] = r.op_q[k].y;
            ops_f[5 * k + 2] = r.op_q[k].z;
            ops_f[5 * k + 3] = r.op_q[k].w;
            ops_f[5 * k + 4] = r.op_cost[k];
        }
    return DA4ML_OK;
}
int da4ml_pipeline_stage_counters(const da4ml_pipeline_t *p, int64_t s, int64_t counters[32]) {
    if (!p || s < 0 || s >= (int64_t)p->impl->stages.size())
        return DA4ML_E_INVALID;
    std::copy(p->impl->stages[s].counters, p->impl->stages[s].counters + 32, counters);
    return DA4ML_OK;
}
int da4ml_pipeline_stage_milestones(const da4ml_pipeline_t *p, int64_t s, int64_t out[63]) {
    if (!p || s < 0 || s >= (int64_t)p->impl->stages.size())
        return DA4ML_E_INVALID;
    std::copy(p->impl->stages[s].counters + META_MILESTONES, p->impl->stages[s].counters + META_MILESTONES + 63, out);
    return DA4ML_OK;
}
double da4ml_pipeline_device_ms(const da4ml_pipeline_t *p) { return p ? p->impl->device_ms : 0.0; }
int64_t da4ml_pipeline_launches(const da4ml_pipeline_t *p) { return p ? p->impl->launches : 0; }
int da4ml_pipeline_profile(const da4ml_pipeline_t *p, double out[8]) {
    if (!p)
        return DA4ML_E_INVALID;
    out[0] = p->impl->device_ms;
    out[1] = (double)p->impl->launches;
    out[2] = p->impl->solve_ms;
    out[3] = (double)p->impl->solve_launches;
    out[4] = p->impl->algo_bytes;
    out[5] = (double)p->impl->jobs_total;
    out[6] = (double)p->impl->jobs_run;
    out[7] = 0.0;
    return DA4ML_OK;
}

// ---- helpers -------------------------------------------------------------------------------------
int da4ml_cmvm_csd_decompose(const float *kernel, int64_t n_in, int64_t n_out, int center, int8_t *csd, int8_t *shift0, int8_t *shift1, int64_t *n_bits) {
    return guarded([&] {
        if (!kernel || n_in <= 0 || n_out <= 0 || !csd || !shift0 || !shift1 || !n_bits)
            throw ApiError(DA4ML_E_INVALID, "csd_decompose only supports 2D arrays."); // bit_decompose.cc:48
        init_device();
        const size_t ne = (size_t)n_in * n_out;
        static DevBuf buf;
        Carver c;
        size_t ok = c.take(sizeof(float) * ne), oq = c.take(sizeof(float) * 3 * n_in), ol = c.take(sizeof(float) * n_in), om = c.take(sizeof(uint2) * ne),
               os0 = c.take(n_in), os1 = c.take(n_out), ocd = c.take(sizeof(int) * n_out), opm = c.take(sizeof(int) * PM_WORDS), od = c.take(sizeof(ProblemDesc)),
               ocsd = c.take(ne * 32), oint = c.take(sizeof(int) * (ne + 1));
        buf.ensure(c.off, false);
        char *b = (char *)buf.p;
        CK(cudaMemcpyAsync(b + ok, kernel, sizeof(float) * ne, cudaMemcpyHostToDevice, g_stream));
        int nbits = 0;
        if (center) {
            std::vector<float> q(3 * (size_t)n_in, 1.0f); // non-zero ranges: no row is blanked
            CK(cudaMemcpyAsync(b + oq, q.data(), sizeof(float) * 3 * n_in, cudaMemcpyHostToDevice, g_stream));
            ProblemDesc d;
            memset(&d, 0, sizeof(d));
            d.n_in = (int)n_in;
            d.n_out = (int)n_out;
            d.kernel = (const float *)(b + ok);
            d.qint = (const float *)(b + oq);
            d.lat = (const float *)(b + ol);
            d.masks0 = (uint2 *)(b + om);
            d.shift0 = (int8_t *)(b + os0);
            d.shift1 = (int8_t *)(b + os1);
            d.col_digits = (int *)(b + ocd);
            d.prep_meta = (int *)(b + opm);
            CK(cudaMemcpyAsync(b + od, &d, sizeof(d), cudaMemcpyHostToDevice, g_stream));
            cmvm_prep_kernel<<<1, 256, 0, g_stream>>>((ProblemDesc *)(b + od));
            CK(cudaGetLastError());
            int pm[PM_WORDS];
            CK(cudaMemcpyAsync(pm, b + opm, sizeof(pm), cudaMemcpyDeviceToHost, g_stream));
            CK(cudaStreamSynchronize(g_stream));
            nbits = pm[PM_NBITS];
            csd_export_kernel<<<(unsigned)((ne + 255) / 256), 256, 0, g_stream>>>((const uint2 *)(b + om), (int)ne, nbits, (int8_t *)(b + ocsd));
            CK(cudaMemcpyAsync(shift0, b + os0, n_in, cudaMemcpyDeviceToHost, g_stream));
            CK(cudaMemcpyAsync(shift1, b + os1, n_out, cudaMemcpyDeviceToHost, g_stream));
        }
        else {
            int *xi = (int *)(b + oint);
            float_to_int_kernel<<<(unsigned)((ne + 255) / 256), 256, 0, g_stream>>>((const float *)(b + ok), (int)ne, xi);
            CK(cudaMemsetAsync(xi + ne, 0, sizeof(int), g_stream));
            int_absmax_kernel<<<(unsigned)((ne + 255) / 256), 256, 0, g_stream>>>(xi, (int)ne, xi + ne);
            int mx = 0;
            CK(cudaMemcpyAsync(&mx, xi + ne, sizeof(int), cudaMemcpyDeviceToHost, g_stream));
            CK(cudaStreamSynchronize(g_stream));
            nbits = csd_nbits(mx);
            int_csd_kernel<<<(unsigned)((ne + 255) / 256), 256, 0, g_stream>>>(xi, (int)ne, nbits, (int8_t *)(b + ocsd));
            memset(shift0, 0, n_in);
            memset(shift1, 0, n_out);
        }
        CK(cudaGetLastError());
        CK(cudaMemcpyAsync(csd, b + ocsd, ne * nbits, cudaMemcpyDeviceToHost, g_stream));
        CK(cudaStreamSynchronize(g_stream));
        *n_bits = nbits;
    });
}

int da4ml_cmvm_int_arr_to_csd(const int32_t *x, int64_t n, int8_t *csd, int64_t *n_bits) {
    return guarded([&] {
        if (!x || n <= 0 || !csd || !n_bits)
            throw ApiError(DA4ML_E_INVALID, "invalid argument");
        init_device();
        static DevBuf buf;
        Carver c;
        size_t ox = c.take(sizeof(int) * (n + 1)), oc = c.take((size_t)n * 32);
        buf.ensure(c.off, false);
        char *b = (char *)buf.p;
        int *xi = (int *)(b + ox);
        CK(cudaMemcpyAsync(xi, x, sizeof(int) * n, cudaMemcpyHostToDevice, g_stream));
        CK(cudaMemsetAsync(xi + n, 0, sizeof(int), g_stream));
        int_absmax_kernel<<<(unsigned)((n + 255) / 256), 256, 0, g_stream>>>(xi, (int)n, xi + n);
        int mx = 0;
        CK(cudaMemcpyAsync(&mx, xi + n, sizeof(int), cudaMemcpyDeviceToHost, g_stream));
        CK(cudaStreamSynchronize(g_stream));
        int nbits = csd_nbits(mx);
        int_csd_kernel<<<(unsigned)((n + 255) / 256), 256, 0, g_stream>>>(xi, (int)n, nbits, (int8_t *)(b + oc));
        CK(cudaGetLastError());
        CK(cudaMemcpyAsync(csd, b + oc, (size_t)n * nbits, cudaMemcpyDeviceToHost, g_stream));
        CK(cudaStreamSynchronize(g_stream));
        *n_bits = nbits;
    });
}

int da4ml_cmvm_kernel_decompose(const float *kernel, int64_t n_in, int64_t n_out, int dc, float *m0, float *m1) {
    return guarded([&] {
        if (!kernel || n_in <= 0 || n_out <= 0 || !m0 || !m1)
            throw ApiError(DA4ML_E_INVALID, "csd_decompose only supports 2D arrays.");
        init_device();
        const size_t n = (size_t)n_out + 1;
        static DevBuf buf;
        Carver c;
        size_t ok = c.take(sizeof(float) * n_in * n_out), oa = c.take(sizeof(float) * n_in * n), od = c.take(sizeof(int) * n * n), os = c.take(n * n), os0 = c.take(n_in),
               os1 = c.take(n_out), om0 = c.take(sizeof(float) * n_in * n_out), om1 = c.take(sizeof(float) * n_out * n_out), omap = c.take(sizeof(int) * 2 * n), oj = c.take(sizeof(DecompJob));
        buf.ensure(c.off, false);
        char *b = (char *)buf.p;
        CK(cudaMemcpyAsync(b + ok, kernel, sizeof(float) * n_in * n_out, cudaMemcpyHostToDevice, g_stream));
        center_kernel<<<1, 256, 0, g_stream>>>((const float *)(b + ok), (int)n_in, (int)n_out, (float *)(b + oa), (int8_t *)(b + os0), (int8_t *)(b + os1));
        long long tot = (long long)n * n;
        dist_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, g_stream>>>((const float *)(b + oa), (int)n_in, (int)n, (int *)(b + od), (int8_t *)(b + os));
        DecompJob j{dc, (float *)(b + om0), (float *)(b + om1), (int *)(b + omap)};
        CK(cudaMemcpyAsync(b + oj, &j, sizeof(j), cudaMemcpyHostToDevice, g_stream));
        const int threads = std::min(1024, std::max(64, (int)((n + 31) / 32 * 32)));
        const size_t smem = n * 17 + 64;
        if (smem > 48 * 1024)
            CK(cudaFuncSetAttribute(mst_build_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        mst_build_kernel<<<1, threads, smem, g_stream>>>((const float *)(b + oa), (const int *)(b + od), (const int8_t *)(b + os), (const int8_t *)(b + os0), (const int8_t *)(b + os1), (int)n_in, (int)n_out, (const DecompJob *)(b + oj));
        CK(cudaGetLastError());
        CK(cudaMemcpyAsync(m0, b + om0, sizeof(float) * n_in * n_out, cudaMemcpyDeviceToHost, g_stream));
        CK(cudaMemcpyAsync(m1, b + om1, sizeof(float) * n_out * n_out, cudaMemcpyDeviceToHost, g_stream));
        CK(cudaStreamSynchronize(g_stream));
    });
}

// ---- DAIS interpreter (reference dais/bindings.cc `run_interp`) ------------------------------------------------------
int da4ml_dais_program_load(const int32_t *words, int64_t n_words, da4ml_dais_program_t **out) {
    return guarded([&] {
        if (!out)
            throw ApiError(DA4ML_E_INVALID, "invalid argument");
        auto p = std::make_unique<da4ml_dais_program>();
        dais_parse(words, n_words, p->h);
        dais_validate(p->h);
        dais_levelise(p->h);
        *out = p.release();
    });
}

int da4ml_dais_program_info(const da4ml_dais_program_t *p, int64_t info[6]) {
    if (!p || !info)
        return DA4ML_E_INVALID;
    info[0] = p->h.n_in;
    info[1] = p->h.n_out;
    info[2] = p->h.n_ops;
    info[3] = p->h.n_tables;
    info[4] = p->h.n_levels;
    info[5] = p->h.max_width;
    return DA4ML_OK;
}

int da4ml_dais_program_run_stream(da4ml_dais_program_t *p, const double *inputs, int64_t n_samples, double *outputs, int device_ptrs, void *stream) {
    return guarded([&] {
        if (!p || n_samples < 0 || (n_samples > 0 && ((!inputs && p->h.n_in) || (!outputs && p->h.n_out))))
            throw ApiError(DA4ML_E_INVALID, "invalid argument");
        dais_execute(*p, inputs, n_samples, outputs, device_ptrs != 0, (cudaStream_t)stream);
    });
}

int da4ml_dais_program_run(da4ml_dais_program_t *p, const double *inputs, int64_t n_samples, double *outputs, int device_ptrs) {
    return da4ml_dais_program_run_stream(p, inputs, n_samples, outputs, device_ptrs, g_stream);
}

int da4ml_dais_program_profile(da4ml_dais_program_t *p, const double *inputs, int64_t n_samples, int device_ptrs, void *cuda_stream, int64_t *stats) {
    return guarded([&] {
        if (!p)
            throw ApiError(DA4ML_E_INVALID, "profile: the program handle is null");
        if (n_samples < 0)
            throw ApiError(DA4ML_E_INVALID, "profile: n_samples is negative (" + std::to_string(n_samples) + ")");
        if (n_samples > 0 && p->h.n_in && !inputs)
            throw ApiError(DA4ML_E_INVALID, "profile: inputs is null");
        if (p->h.n_ops && !stats)
            throw ApiError(DA4ML_E_INVALID, "profile: stats is null");
        DaisRequest req;
        req.pass = DaisPass::profile;
        req.stats = (long long *)stats;
        dais_execute(*p, inputs, n_samples, nullptr, device_ptrs != 0, (cudaStream_t)cuda_stream, req);
    });
}

int da4ml_dais_program_dump(da4ml_dais_program_t *p, const double *inputs, int64_t n_samples, const int32_t *op_ids, int64_t n_sel, int64_t *values, int device_ptrs,
                            void *cuda_stream) {
    return guarded([&] {
        if (!p)
            throw ApiError(DA4ML_E_INVALID, "dump: the program handle is null");
        if (n_samples < 0)
            throw ApiError(DA4ML_E_INVALID, "dump: n_samples is negative (" + std::to_string(n_samples) + ")");
        if (n_sel < 0)
            throw ApiError(DA4ML_E_INVALID, "dump: n_sel is negative (" + std::to_string(n_sel) + ")");
        if (n_sel > 0 && !op_ids)
            throw ApiError(DA4ML_E_INVALID, "dump: op_ids is null");
        for (int64_t k = 0; k < n_sel; ++k)
            if (op_ids[k] < 0 || op_ids[k] >= p->h.n_ops)
                throw ApiError(DA4ML_E_INVALID, "dump: op id " + std::to_string(op_ids[k]) + " at position " + std::to_string(k) + " is out of range [0, " +
                                                    std::to_string(p->h.n_ops) + ")");
        if (n_samples > 0 && p->h.n_in && !inputs)
            throw ApiError(DA4ML_E_INVALID, "dump: inputs is null");
        if (n_samples > 0 && n_sel > 0 && !values)
            throw ApiError(DA4ML_E_INVALID, "dump: values is null");
        DaisRequest req;
        req.pass = DaisPass::dump;
        req.sel = op_ids;
        req.n_sel = n_sel;
        dais_execute(*p, inputs, n_samples, values, device_ptrs != 0, (cudaStream_t)cuda_stream, req);
    });
}

void da4ml_dais_program_free(da4ml_dais_program_t *p) {
    std::lock_guard<std::mutex> lock(g_mutex);
    delete p;
}

// Adder-graph programs only (opcodes -1/0/1, no tables): the checks and messages of the CMVM path, then the engine above.
int da4ml_dais_run(const int32_t *program, int64_t n_words, const double *inputs, int64_t n_samples, double *outputs) {
    return guarded([&] {
        if (!program || n_words < 6 || !inputs || !outputs || n_samples < 0)
            throw ApiError(DA4ML_E_RUNTIME, "Binary data too small to contain valid DAIS model file"); // DAISInterpreter.cc:11-15
        if (program[0] != 1)
            throw ApiError(DA4ML_E_RUNTIME, "DAIS version mismatch: expected version 1, got version " + std::to_string(program[0]));
        const int n_in = program[2], n_out = program[3], n_ops = program[4], n_tables = program[5];
        if (n_in < 0 || n_out < 0 || n_ops < 0)
            throw ApiError(DA4ML_E_RUNTIME, "Binary data header holds a negative count");
        if (n_tables != 0 || n_words != 6 + (int64_t)n_in + 3LL * n_out + 8LL * n_ops)
            throw ApiError(DA4ML_E_RUNTIME, "Binary data size mismatch (lookup tables are not produced by the CMVM path)");
        if (n_samples == 0)
            return;
        da4ml_dais_program prog;
        dais_parse(program, n_words, prog.h); // (index and shift ranges of the header arrays)
        for (int i = 0; i < n_ops; ++i) {
            const DaisOp &op = prog.h.ops[i];
            if (op.opcode == -1) {
                if (op.id0 < 0 || op.id0 >= n_in)
                    throw ApiError(DA4ML_E_RUNTIME, "input index out of range at operation " + std::to_string(i));
                continue;
            }
            if (op.opcode != 0 && op.opcode != 1)
                throw ApiError(DA4ML_E_RUNTIME, "Unknown opcode: " + std::to_string(op.opcode) + " at index " + std::to_string(i) + " (only adder graphs are replayed on this path)");
            if (op.id0 < 0 || op.id0 >= i || op.id1 < 0 || op.id1 >= i)
                throw ApiError(DA4ML_E_RUNTIME, "Operation " + std::to_string(i) + " violating causality");
        }
        dais_levelise(prog.h);
        dais_execute(prog, inputs, n_samples, outputs, false, g_stream);
    });
}

int da4ml_cmvm_get_lsb_loc(float x) { return get_lsb_loc(x); }
int da4ml_cmvm_iceil_log2(float x) { return iceil_log2(x); }
int da4ml_cmvm_cost_add(const float q0[3], const float q1[3], int64_t shift, int sub, int adder_size, int carry_size, float out[2]) {
    cost_add(QInt{q0[0], q0[1], q0[2]}, QInt{q1[0], q1[1], q1[2]}, shift, sub != 0, adder_size, carry_size, out[0], out[1]);
    return DA4ML_OK;
}

} // extern "C"
