// pipeline_price.cuh -- price solver results as they will be pipelined: re-trace an adder graph under a latency cutoff,
// split it into register stages, and count its stages and register bits (reference: the symbolic tracer's latency rule,
// trace/fixed_variable.py:347-379; comb_trace with its dead-statement elimination, trace/tracer.py; to_pipeline with
// retiming=False, trace/pipeline.py:63-167; Pipeline.reg_bits, types.py:695-703; retime_pipeline, trace/pipeline.py:8-31).
//
// A *design* is one solver result (the stages of a RawPipeline, opcodes -1/0/1).  Everything that does not depend on the
// cutoff is prepared once per design on the host (pp_prepare): every value the replay creates is a *node* (a network
// input, one adder, or the constant zero a dead output column becomes), every op is a view of a node scaled by +-2^k, the
// adders are ordered by dependency level, the liveness of every node (comb_trace drops what reaches no output) and the
// minimal_kif bits of its interval are known, and so are the float32 operands the tracer hands cost_add.  A *task* is
// (design, cutoff, input latencies); pipeline_price_kernel runs one CTA per task: the adders of one level at a time get
// their traced latency in double with the tracer's own expressions, then every live node gets its producer stage
// floor(lat / (c + 1e-9)) and, by a max over its consumers, its last consumer stage, and the stage count, the register
// bits and retime_pipeline's bisection bounds are reduced over the nodes.  pp_price drives it, including the bisection.
#pragma once
#include "cmvm_num.cuh"
#include "cmvm_types.cuh"

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <functional>
#include <stdexcept>
#include <string>
#include <vector>

namespace da {

enum PpStatus : int { PP_OK = 0, PP_SLOW_ADDER = 1 /* the tracer's AssertionError */, PP_UNSUPPORTED = 2 /* a constant intermediate value */ };

// One adder of a design, in dependency-level order.  `node` is its own node id; n0 / n1 the nodes its operands view; q0 /
// q1 the operand intervals cost_add receives (after FixedVariable.__add__'s sign normalisation, as float32); `flag` 2: an
// operand is a constant (refused before the latency), 1: the sum is a constant (refused after the latency), 0: neither.
struct PpAdd {
    int node, n0, n1, flag;
    float q0[3], q1[3];
};

// Device view of a prepared design.  Node ids: [0, n_in) the network inputs, n_in the constant zero, then the adders.
struct PpDesign {
    const PpAdd *adds;     // [n_adds] in level order
    const int *lvl_begin;  // [n_levels + 1]
    const int *node_bits;  // [n_nodes] bits of the node's own interval (minimal_kif); -1: not in the traced graph
    const int *out_node;   // [n_out]
    int n_in, n_nodes, n_adds, n_levels, n_out, adder_size, carry_size, pad;
    long long out_bits;    // bits of the last stage's outputs (their intervals do not depend on the cutoff)
};

struct PpTask {
    int design, pad;
    double cutoff;          // 0: unpipelined (only the bisection asks for it)
    const double *in_lat;   // [n_in] or nullptr (zeros)
    double *lat;            // workspace [n_nodes]
    int *last_use;          // workspace [n_nodes]
    double *out_lat;        // [n_out] or nullptr
};

struct PpResult {
    int status, stages;
    long long reg_bits;
    double latency_max, retime_hi, retime_lo; // retime_pipeline's starting cutoff_high / cutoff_low for this split
};

// IEEE double ops the compiler may not contract into FMAs (the tracer's expressions are separate Python float ops)
DA_HD double pp_add(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dadd_rn(a, b);
#else
    volatile double r = a + b;
    return r;
#endif
}
DA_HD double pp_mul(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __dmul_rn(a, b);
#else
    volatile double r = a * b;
    return r;
#endif
}
DA_HD double pp_div(double a, double b) {
#if defined(__CUDA_ARCH__)
    return __ddiv_rn(a, b);
#else
    volatile double r = a / b;
    return r;
#endif
}
// to_pipeline's get_stage
DA_HD int pp_stage(double lat, double c) { return c > 0 ? (int)floor(pp_div(lat, pp_add(c, 1e-9))) : 0; }
// non-negative doubles order like their bit patterns: max-reductions through integer atomics
DA_HD unsigned long long pp_dbits(double x) {
    unsigned long long u;
    memcpy(&u, &x, 8);
    return u;
}
DA_HD double pp_bitsd(unsigned long long u) {
    double x;
    memcpy(&x, &u, 8);
    return x;
}

// The tracer's latency of every adder node of task `t`, level by level, with the tracer's own expressions (t.lat holds the
// inputs' latencies on entry); the first failing adder goes to `s_fail` as (node << 2 | status).  With COST, cost_add's
// cost of every adder node goes to cost[node] as well (the split needs it, pricing drops it).  Every thread of the CTA
// calls it; it ends with a barrier.  Shared by pipeline_price_kernel and pipeline_split_kernel.
template <bool COST> __device__ __forceinline__ void pp_replay(const PpDesign &d, const PpTask &t, unsigned long long &s_fail, float *cost_out) {
    const double c = t.cutoff;
    const int tid = threadIdx.x, nt = blockDim.x;
    for (int l = 0; l < d.n_levels; ++l) {
        for (int k = d.lvl_begin[l] + tid; k < d.lvl_begin[l + 1]; k += nt) {
            const PpAdd a = d.adds[k];
            float dl = 0.f, cost = 0.f;
            cost_add(QInt{a.q0[0], a.q0[1], a.q0[2]}, QInt{a.q1[0], a.q1[1], a.q1[2]}, 0, false, d.adder_size, d.carry_size, dl, cost);
            const double dlat = (double)dl, base = fmax(t.lat[a.n0], t.lat[a.n1]);
            double lat = pp_add(dlat, base);
            bool slow = false;
            if (c > 0 && ceil(pp_div(lat, c)) > ceil(pp_div(base, c))) { // would straddle a register boundary
                slow = !(dlat <= c);
                lat = pp_add(pp_mul(ceil(pp_div(base, c)), c), dlat);
            }
            t.lat[a.node] = lat;
            if (COST)
                cost_out[a.node] = cost;
            const int st = a.flag == 2 ? PP_UNSUPPORTED : slow ? PP_SLOW_ADDER : a.flag == 1 ? PP_UNSUPPORTED : PP_OK;
            if (st != PP_OK)
                atomicMin(&s_fail, ((unsigned long long)a.node << 2) | (unsigned long long)st);
        }
        __syncthreads();
    }
}

__global__ void __launch_bounds__(256) pipeline_price_kernel(const PpDesign *designs, const PpTask *tasks, PpResult *results) {
    DA_SHARED_VAR(unsigned long long, s_fail);  // (replay order << 2 | status) of the first failing adder
    DA_SHARED_VAR(unsigned long long, s_latmax);
    DA_SHARED_VAR(unsigned long long, s_hi);
    DA_SHARED_VAR(unsigned long long, s_lo);
    DA_SHARED_VAR(unsigned long long, s_bits);
    const PpTask t = tasks[blockIdx.x];
    const PpDesign d = designs[t.design];
    const double c = t.cutoff;
    const int tid = threadIdx.x, nt = blockDim.x;
    if (tid == 0) {
        s_fail = ~0ull;
        s_latmax = s_hi = s_lo = 0ull;
        s_bits = 0ull;
    }
    for (int v = tid; v < d.n_nodes; v += nt) {
        // (an input with a point interval is a constant to the tracer: no op views it, see pp_prepare)
        t.lat[v] = v < d.n_in && t.in_lat ? t.in_lat[v] : 0.0;
        t.last_use[v] = -1;
    }
    __syncthreads();
    pp_replay<false>(d, t, s_fail, nullptr);
    PpResult r{};
    if (s_fail != ~0ull) {
        if (tid == 0) {
            r.status = (int)(s_fail & 3ull);
            r.stages = -1;
            r.reg_bits = -1;
            r.latency_max = r.retime_hi = r.retime_lo = nan("");
            results[blockIdx.x] = r;
        }
        return;
    }
    for (int o = tid; o < d.n_out; o += nt) {
        const double lo = t.lat[d.out_node[o]];
        atomicMax(&s_latmax, pp_dbits(lo));
        if (t.out_lat)
            t.out_lat[o] = lo;
    }
    __syncthreads();
    const double lat_max = pp_bitsd(s_latmax);
    const int s_out = pp_stage(lat_max, c), n_st = s_out + 1;
    // last consumer stage of every live node: the stage of each live adder reading it, and the output stage
    for (int k = tid; k < d.n_adds; k += nt) {
        const PpAdd a = d.adds[k];
        if (d.node_bits[a.node] < 0)
            continue;
        const int s = pp_stage(t.lat[a.node], c);
        atomicMax(&t.last_use[a.n0], s);
        atomicMax(&t.last_use[a.n1], s);
    }
    for (int o = tid; o < d.n_out; o += nt)
        atomicMax(&t.last_use[d.out_node[o]], s_out);
    __syncthreads();
    // a value produced in stage p and last read in stage q > p is an output of stages p .. q-1: its bits count q - p
    // times; its latency as an output of stage p is its own, as an output of a later stage i the copy's c * i
    unsigned long long bits = 0ull, hi = 0ull;
    for (int v = tid; v < d.n_nodes; v += nt) {
        const int b = d.node_bits[v], q = t.last_use[v];
        if (b < 0 || q < 0)
            continue;
        const double lv = t.lat[v];
        const int p = pp_stage(lv, c);
        bits += (unsigned long long)b * (unsigned long long)(q - p) + (v < d.n_in && p == 0 ? (unsigned long long)b : 0ull);
        if (q > p)
            hi = max(hi, pp_dbits(pp_div(lv, (double)(p + 1))));
        if (q - 1 > p)
            hi = max(hi, pp_dbits(pp_div(pp_mul(c, (double)(q - 1)), (double)q)));
    }
    unsigned long long lo = 0ull;
    for (int o = tid; o < d.n_out; o += nt) { // the last stage's outputs
        const double lv = t.lat[d.out_node[o]];
        const double x = pp_stage(lv, c) == s_out ? lv : pp_mul(c, (double)s_out);
        lo = max(lo, pp_dbits(x));
    }
    atomicAdd(&s_bits, bits);
    atomicMax(&s_hi, hi);
    atomicMax(&s_lo, lo);
    __syncthreads();
    if (tid == 0) {
        const double lo_lat = pp_bitsd(s_lo);
        r.status = PP_OK;
        r.stages = n_st;
        r.reg_bits = (long long)s_bits + d.out_bits;
        r.latency_max = lat_max;
        r.retime_hi = fmax(pp_bitsd(s_hi), pp_div(lo_lat, (double)n_st));
        r.retime_lo = pp_div(lo_lat, (double)n_st);
        results[blockIdx.x] = r;
    }
}

// ---- host side: per-design preparation and the retiming bisection --------------------------------------------------

// One stage of a design in the flat layout of da4ml_pipeline_stage_copy.
struct PpStageIn {
    int64_t n_in, n_out, n_ops, carry_size, adder_size;
    const int64_t *inp_shifts, *out_idxs, *out_shifts, *out_negs, *ops_i; // ops_i [n_ops][4]
    const float *ops_f;                                                     // [n_ops][5]
};

// What a split needs beyond pricing, recorded by pp_prepare only when asked for (pipeline_split.cuh).  Node ids as in
// PpDesign; the constant node stands for every all-zero output column.
struct PpSplitInfo {
    std::vector<double> own_q;          // [n_nodes][3] the node's own (unscaled) interval; the constant: (0, 0, 2^32)
    std::vector<int> x, y, opc, data;   // per adder node - n_in - 1: FixedVariable.__add__'s operand order (the operand
                                        // with a positive factor first) and the op it becomes: opcode = (factor of y < 0),
                                        // data = log2|factor of y / factor of x|
    std::vector<int64_t> out_shift;     // [n_out] log2|factor| of each output's view
    std::vector<char> out_neg;          // [n_out] factor < 0
};

struct PpPrepared {
    std::vector<PpAdd> adds;
    std::vector<int> lvl_begin, node_bits, out_node;
    int n_in = 0, n_nodes = 0, n_out = 0, adder_size = -1, carry_size = -1;
    long long out_bits = 0;
};

// sum of minimal_kif (types.py:86-114) of an interval
inline int pp_kif_bits(double lo, double hi, double step) {
    if (lo == 0.0 && hi == 0.0)
        return 0;
    const int keep_neg = lo < 0;
    const int frac = (int)(-std::log2(step));
    const double imin = std::nearbyint(lo / step), imax = std::nearbyint(hi / step);
    const int bits = (int)std::ceil(std::log2(std::max(std::fabs(imin), imax + 1)));
    return keep_neg + bits;
}

// Check one design's arrays (DA4ML_E_INVALID-class errors are thrown as std::invalid_argument) and prepare it.
inline PpPrepared pp_prepare(const PpStageIn *st, int64_t n_stages, PpSplitInfo *split = nullptr) {
    struct View { // a node seen through a scaling: interval of the scaled value and its factor (+-2^k)
        int node;
        double lo, hi, step, f;
    };
    auto scaled = [](View v, double s) {
        const double a = v.lo * s, b = v.hi * s;
        return View{v.node, std::min(a, b), std::max(a, b), std::fabs(v.step * s), v.f * s};
    };
    auto bad = [](const std::string &m) { throw std::invalid_argument("pipeline_price: " + m); };
    if (n_stages < 1)
        bad("a design needs at least one stage");
    PpPrepared P;
    P.n_in = (int)st[0].n_in;
    P.adder_size = (int)st[0].adder_size;
    P.carry_size = (int)st[0].carry_size;
    const int CONST = P.n_in;
    std::vector<View> node_view; // the view an adder node was created with
    std::vector<double> in_q(3 * (size_t)P.n_in);
    for (int k = 0; k < P.n_in; ++k)
        in_q[3 * k] = 0.0, in_q[3 * k + 1] = 0.0, in_q[3 * k + 2] = 1.0;
    for (int64_t s = 0; s < n_stages; ++s) {
        const PpStageIn &S = st[s];
        if (S.n_in < 0 || S.n_out < 0 || S.n_ops < 0 || (s > 0 && S.n_in != st[s - 1].n_out))
            bad("stage " + std::to_string(s) + " has a bad shape");
        if (S.n_in > (1 << 24) || S.n_ops > (1 << 26))
            bad("stage " + std::to_string(s) + " is too large");
        if ((S.n_in && !S.inp_shifts) || (S.n_out && (!S.out_idxs || !S.out_shifts || !S.out_negs)) || (S.n_ops && (!S.ops_i || !S.ops_f)))
            bad("a stage array is null");
        for (int64_t i = 0; i < S.n_ops; ++i) {
            const int64_t *o = S.ops_i + 4 * i;
            const bool ok = o[2] == -1 ? (o[0] >= 0 && o[0] < S.n_in && std::abs(S.inp_shifts[o[0]]) <= 512) : (o[2] == 0 || o[2] == 1) ? (o[0] >= 0 && o[0] < i && o[1] >= 0 && o[1] < i && std::abs(o[3]) <= 512) : false;
            if (!ok)
                bad("stage " + std::to_string(s) + " op " + std::to_string(i) + ": opcode " + std::to_string(o[2]) + " with operands (" + std::to_string(o[0]) + ", " +
                    std::to_string(o[1]) + ") is not an adder-graph op (opcodes -1, 0, 1; operands earlier ops, inputs in range)");
        }
        for (int64_t k = 0; k < S.n_out; ++k)
            if (S.out_idxs[k] < -1 || S.out_idxs[k] >= S.n_ops || std::abs(S.out_shifts[k]) > 512)
                bad("stage " + std::to_string(s) + " output " + std::to_string(k) + " is out of range");
    }
    for (int64_t i = 0; i < st[0].n_ops; ++i) // the design's input intervals (CombLogic.inp_qint)
        if (st[0].ops_i[4 * i + 2] == -1)
            for (int j = 0; j < 3; ++j)
                in_q[3 * st[0].ops_i[4 * i] + j] = st[0].ops_f[5 * i + j];
    auto view_of = [&](int node) -> View {
        if (node == CONST)
            return View{CONST, 0.0, 0.0, 4294967296.0, 1.0};
        if (node < P.n_in)
            return View{node, in_q[3 * node], in_q[3 * node + 1], in_q[3 * node + 2], 1.0};
        return node_view[node - P.n_in - 1];
    };
    // replay: cur = the views entering the stage
    std::vector<View> cur(P.n_in);
    for (int k = 0; k < P.n_in; ++k)
        cur[k] = in_q[3 * k] == in_q[3 * k + 1] ? View{CONST, in_q[3 * k], in_q[3 * k + 1], in_q[3 * k + 2], 1.0} : view_of(k);
    std::vector<int> lvl(P.n_in + 1, 0);
    std::vector<PpAdd> adds;
    for (int64_t s = 0; s < n_stages; ++s) {
        const PpStageIn &S = st[s];
        std::vector<View> buf(S.n_ops);
        for (int64_t i = 0; i < S.n_ops; ++i) {
            const int64_t *o = S.ops_i + 4 * i;
            if (o[2] == -1) {
                buf[i] = scaled(cur[o[0]], std::ldexp(1.0, (int)S.inp_shifts[o[0]]));
                continue;
            }
            View A = buf[o[0]], B = scaled(buf[o[1]], std::ldexp(1.0, (int)o[3]));
            if (o[2] == 1)
                B = scaled(B, -1.0);
            PpAdd a{};
            a.node = P.n_in + 1 + (int)adds.size();
            a.n0 = A.node;
            a.n1 = B.node;
            a.flag = (A.lo == A.hi || B.lo == B.hi) ? 2 : 0;
            const double lo = A.lo + B.lo, hi = A.hi + B.hi, step = std::min(A.step, B.step);
            double f = A.f;
            View X = A, Y = B; // FixedVariable.__add__: the operand with a positive factor first; both negative: negate both
            if (A.f < 0) {
                if (B.f > 0)
                    X = B, Y = A, f = B.f;
                else
                    X = scaled(A, -1.0), Y = scaled(B, -1.0);
            }
            a.q0[0] = (float)X.lo, a.q0[1] = (float)X.hi, a.q0[2] = (float)X.step;
            a.q1[0] = (float)Y.lo, a.q1[1] = (float)Y.hi, a.q1[2] = (float)Y.step;
            if (split) {
                split->x.push_back(X.node);
                split->y.push_back(Y.node);
                split->opc.push_back(Y.f < 0);
                split->data.push_back((int)std::log2(std::fabs(Y.f / X.f)));
            }
            if (a.flag == 0 && lo == hi)
                a.flag = 1;
            node_view.push_back(View{a.node, lo, hi, step, f});
            lvl.push_back(1 + std::max(lvl[A.node], lvl[B.node]));
            adds.push_back(a);
            buf[i] = node_view.back();
        }
        std::vector<View> next(S.n_out);
        for (int64_t k = 0; k < S.n_out; ++k) {
            const int64_t i = S.out_idxs[k];
            if (i < 0)
                next[k] = view_of(CONST);
            else
                next[k] = scaled(scaled(buf[i], std::ldexp(1.0, (int)S.out_shifts[k])), S.out_negs[k] ? -1.0 : 1.0);
        }
        cur.swap(next);
    }
    P.n_nodes = P.n_in + 1 + (int)adds.size();
    P.n_out = (int)cur.size();
    if (split) {
        split->own_q.resize(3 * (size_t)P.n_nodes);
        for (int v = 0; v < P.n_nodes; ++v) {
            View w = view_of(v);
            w = scaled(w, 1.0 / w.f); // FixedVariable.unscaled
            split->own_q[3 * v] = w.lo, split->own_q[3 * v + 1] = w.hi, split->own_q[3 * v + 2] = w.step;
        }
        for (const View &v : cur) {
            split->out_shift.push_back((int64_t)std::log2(std::fabs(v.f)));
            split->out_neg.push_back(v.f < 0);
        }
    }
    // liveness (comb_trace's dead-statement elimination) and bits
    std::vector<char> live(P.n_nodes, 0);
    for (const View &v : cur) {
        P.out_node.push_back(v.node);
        live[v.node] = 1;
        P.out_bits += v.node == CONST ? 0 : pp_kif_bits(v.lo, v.hi, v.step);
    }
    for (size_t k = adds.size(); k-- > 0;)
        if (live[adds[k].node])
            live[adds[k].n0] = live[adds[k].n1] = 1;
    P.node_bits.assign(P.n_nodes, -1);
    for (int v = 0; v < P.n_nodes; ++v) {
        if (!live[v])
            continue;
        if (v == CONST) {
            P.node_bits[v] = 0;
            continue;
        }
        View w = view_of(v);
        if (w.f < 0)
            w = scaled(w, -1.0); // the node's own interval (the op's qint in the traced graph)
        P.node_bits[v] = pp_kif_bits(w.lo, w.hi, w.step);
    }
    // adders by level (stable: replay order within a level); level l + 1 is adds[lvl_begin[l], lvl_begin[l + 1])
    int n_lv = 0;
    for (const PpAdd &a : adds)
        n_lv = std::max(n_lv, lvl[a.node]);
    P.lvl_begin.assign(n_lv + 1, 0);
    for (const PpAdd &a : adds)
        ++P.lvl_begin[lvl[a.node]];
    for (int l = 1; l <= n_lv; ++l)
        P.lvl_begin[l] += P.lvl_begin[l - 1];
    std::vector<int> pos(P.lvl_begin.begin(), P.lvl_begin.end() - 1);
    P.adds.resize(adds.size());
    for (const PpAdd &a : adds)
        P.adds[pos[lvl[a.node] - 1]++] = a;
    return P;
}

// Per (design, cutoff) answer of pp_price.
struct PpAnswer {
    int status = PP_OK, stages = -1;
    long long reg_bits = -1;
    double latency_max = 0, cutoff = 0;
    int first_stages = -1; // stages of the first split (the task's own cutoff and latencies)
    bool retimed = false;  // a bisection round succeeded: the kept split is the last such round's (`cutoff`, latency 0)
};

// `run(tasks, results)`: one launch of pipeline_price_kernel over `tasks` (design, cutoff, latencies: nullptr = zeros).
// Pricing of every design under every cutoff, then (retiming) retime_pipeline's bisection for all tasks together: one
// launch per round over the tasks still bisecting, each re-traced with its inputs at latency 0.
struct PpRequest {
    int design;
    double cutoff;
    bool zero_latency;
    int slot; // the (design, cutoff) task it belongs to: design * n_cutoffs + cutoff index
};
inline std::vector<PpAnswer> pp_price(int n_designs, const double *cutoffs, int n_cutoffs, bool retiming,
                                      const std::function<void(const std::vector<PpRequest> &, std::vector<PpResult> &)> &run) {
    std::vector<PpRequest> req;
    for (int d = 0; d < n_designs; ++d)
        for (int j = 0; j < n_cutoffs; ++j)
            req.push_back(PpRequest{d, cutoffs[j], false, (int)req.size()});
    std::vector<PpResult> res;
    run(req, res);
    std::vector<PpAnswer> ans(req.size());
    std::vector<double> hi(req.size()), lo(req.size());
    for (size_t t = 0; t < req.size(); ++t) {
        ans[t].status = res[t].status;
        ans[t].stages = res[t].stages;
        ans[t].reg_bits = res[t].reg_bits;
        ans[t].latency_max = res[t].latency_max;
        ans[t].cutoff = req[t].cutoff;
        hi[t] = res[t].retime_hi;
        lo[t] = res[t].retime_lo;
    }
    std::vector<int> n_stages(req.size());
    for (size_t t = 0; t < req.size(); ++t)
        n_stages[t] = ans[t].first_stages = ans[t].stages;
    while (retiming) {
        std::vector<size_t> open;
        std::vector<PpRequest> round;
        for (size_t t = 0; t < req.size(); ++t)
            if (ans[t].status == PP_OK && hi[t] - lo[t] > 1) {
                open.push_back(t);
                round.push_back(PpRequest{req[t].design, std::floor((hi[t] + lo[t]) / 2), true, (int)t});
            }
        if (open.empty())
            break;
        run(round, res);
        for (size_t k = 0; k < open.size(); ++k) {
            const size_t t = open[k];
            if (res[k].status != PP_OK || res[k].stages > n_stages[t]) { // an adder slower than the cutoff, or too many stages
                lo[t] = round[k].cutoff;
                continue;
            }
            hi[t] = round[k].cutoff;
            ans[t].retimed = true;
            ans[t].stages = res[k].stages;
            ans[t].reg_bits = res[k].reg_bits;
        }
    }
    for (size_t t = 0; t < req.size(); ++t)
        if (retiming && ans[t].status == PP_OK)
            ans[t].cutoff = hi[t];
    return ans;
}

} // namespace da
