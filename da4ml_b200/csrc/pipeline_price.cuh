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

// What the node of a PpAdd is.  The order matters: no flag from PP_ONE_OPERAND on is an adder (no cost_add, no
// register-boundary rule), and pp_replay tests that as `flag >= PP_ONE_OPERAND`.
enum PpFlag : int {
    PP_ADDER = 0,          // an adder
    PP_CONST_SUM = 1,      // an adder whose sum is a constant (refused after the latency)
    PP_CONST_OPERAND = 2,  // an adder with a constant operand (refused before the latency)
    PP_ONE_OPERAND = 3,    // an activation (relu / quantize, opcodes +-2 / +-3) or a constant addition (opcode 4) of
                           // node n0 == n1: its operand's latency (trace/fixed_variable.py:353-359, 381-384); tracer
                           // cost q0[0]
    PP_CONST_CADD = 4,     // a constant addition of a constant (refused like PP_CONST_OPERAND, after the latency)
    PP_LOOKUP = 5,         // a lookup (opcode 8) of node n0 == n1: its operand's latency plus q0[1] (max(b_in - 6, 1),
                           // no register-boundary rule: trace/fixed_variable.py:331-340); tracer cost q0[0]
    PP_MUX = 6,            // an MSB mux (opcode +-6) of the data nodes n0 / n1 on the condition node nc: the largest of
                           // its three operands' latencies plus q0[1] (cost_add's latency of its data operands; msb_mux
                           // is built with an explicit latency, so no register-boundary rule:
                           // trace/fixed_variable.py:841-859); tracer cost q0[0]
};

// One node an op of a design creates, in dependency-level order.  `node` is its own node id; n0 / n1 the nodes its operands
// view; for an adder, q0 / q1 the operand intervals cost_add receives (after FixedVariable.__add__'s sign normalisation, as
// float32); nc the condition node of an MSB mux, -1 for every other flag.
struct PpAdd {
    int node, n0, n1;
    PpFlag flag;
    float q0[3], q1[3];
    int nc;
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
            if (a.flag == PP_MUX) { // no adder, no boundary rule
                t.lat[a.node] = pp_add(fmax(fmax(t.lat[a.n0], t.lat[a.n1]), t.lat[a.nc]), (double)a.q0[1]);
                if (COST)
                    cost_out[a.node] = a.q0[0];
                continue;
            }
            if (a.flag >= PP_ONE_OPERAND) { // an activation, a constant addition or a lookup: no adder
                t.lat[a.node] = a.flag == PP_LOOKUP ? pp_add((double)a.q0[1], t.lat[a.n0]) : t.lat[a.n0];
                if (COST)
                    cost_out[a.node] = a.q0[0];
                if (a.flag == PP_CONST_CADD)
                    atomicMin(&s_fail, ((unsigned long long)a.node << 2) | (unsigned long long)PP_UNSUPPORTED);
                continue;
            }
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
            const int st = a.flag == PP_CONST_OPERAND ? PP_UNSUPPORTED : slow ? PP_SLOW_ADDER : a.flag == PP_CONST_SUM ? PP_UNSUPPORTED : PP_OK;
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
        if (a.flag == PP_MUX)
            atomicMax(&t.last_use[a.nc], s);
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

// A node seen through a scaling: the interval of the scaled value and its factor (+-2^k).
struct PpView {
    int node;
    double lo, hi, step, f;
};

// What a split needs of one node an op creates: its operands as views of their nodes, and the op it becomes.  An adder: x
// and y in FixedVariable.__add__'s operand order (the operand with a positive factor first), opcode = (factor of y < 0),
// data = log2|factor of y / factor of x|.  A one-operand op: x its operand, y none; relu / quantize: opcode +-2 / +-3 by
// the sign of the operand's factor, data 0; a constant addition: opcode 4, data the addend in steps; a lookup: opcode 8,
// data the table index.  An MSB mux: x / y its data operands a / b, opcode 6 or -6 by the sign of b's factor, data
// log2|factor of b / factor of a|.  z is the mux's condition, none for every other op.  None: node -1, zeros.
struct PpSplitOp {
    PpView x, y, z;
    int opc, data;
};

// What a split needs beyond pricing, recorded by pp_prepare only when asked for (pipeline_split.cuh).  Node ids as in
// PpDesign; the constant node stands for every all-zero output column.
struct PpSplitInfo {
    std::vector<double> own_q;          // [n_nodes][3] the node's own (unscaled) interval; the constant: (0, 0, 2^32)
    std::vector<PpSplitOp> ops;         // [node - n_in - 1] per node an op creates
    std::vector<PpView> out_v;          // [n_out] each output's view
    std::vector<int64_t> out_shift;     // [n_out] log2|factor| of each output's view
    std::vector<char> out_neg;          // [n_out] factor < 0
};

struct PpPrepared {
    std::vector<PpAdd> adds;
    std::vector<int> lvl_begin, node_bits, out_node;
    int n_in = 0, n_nodes = 0, n_out = 0, adder_size = -1, carry_size = -1;
    long long out_bits = 0;
};

// minimal_kif (types.py:86-114) of an interval
inline void pp_minimal_kif(double lo, double hi, double step, int &k, int &i, int &f) {
    if (lo == 0.0 && hi == 0.0) {
        k = i = f = 0;
        return;
    }
    k = lo < 0;
    f = (int)(-std::log2(step));
    const double imin = std::nearbyint(lo / step), imax = std::nearbyint(hi / step);
    i = (int)std::ceil(std::log2(std::max(std::fabs(imin), imax + 1))) - f;
}

// What relu / quantize make of a value (the interval [lo, hi] of its scaled view, step > 0), as CombLogic.__call__ replays
// opcodes +-2 / +-3 (types.py:259-266): FixedVariable.relu(i, f) with TRN (trace/fixed_variable.py:645-686) and
// FixedVariable.quantize(k, i, f) with WRAP / TRN and _force_factor_clear (:688-779), (k, i, f) the minimal_kif of the op's
// interval.  kind 0: the value itself (relu changed nothing), 1: the constant `lo`, 2: a new value [lo, hi] / step.
struct PpAct {
    int kind;
    double lo, hi, step;
};
// FixedVariable.kif (trace/fixed_variable.py:418-428) of a non-constant value: k + i + f
inline int pp_kif_prop_bits(double lo, double hi, double step) {
    const int f = -(int)std::log2(step);
    const int i = (int)std::ceil(std::log2(std::max(-lo, hi + step)));
    return (lo < 0) + i + f;
}
inline PpAct pp_relu(double lo, double hi, double step, int i, int f) {
    const double st = std::max(std::ldexp(1.0, -f), step);
    double l = (std::floor(std::max(0.0, lo) / st) + 0.0) * st, h = (std::floor(hi / st) + 0.0) * st; // (floor: an int, no -0)
    const double top = std::ldexp(1.0, i) - st;
    if (top < h)
        l = 0.0, h = top;
    h = std::max(0.0, h);
    if (l == lo && h == hi && st == step)
        return PpAct{0, lo, hi, step};
    return l == h ? PpAct{1, l, l, st} : PpAct{2, l, h, st};
}
inline PpAct pp_quantize(double lo, double hi, double step, int k, int i, int f) {
    if (k + i + f <= 0)
        return PpAct{1, 0.0, 0.0, 1.0};
    const int f0 = -(int)std::log2(step), k0 = lo < 0;
    int i0 = (int)std::ceil(std::log2(std::max(-lo, hi + step)));
    f = std::min(f, f0);
    k = i >= i0 ? std::min(k, k0) : k;
    const double st = std::ldexp(1.0, -f);
    if (lo < 0)
        i0 = std::max(i0, (int)std::ceil(std::log2(-std::floor(lo / st) * st)));
    i = std::min(i, i0 + (k == 0 && k0 == 1));
    if (i + k + f <= 0)
        return PpAct{1, 0.0, 0.0, 1.0};
    double l = k ? -std::ldexp(1.0, i) : 0.0, h = std::ldexp(1.0, i) - st; // (+0.0, as the tracer's Decimal)
    if (lo >= l && hi <= h)
        l = (std::floor(lo / st) + 0.0) * st, h = (std::floor(hi / st) + 0.0) * st;
    return l == h ? PpAct{1, l, l, st} : PpAct{2, l, h, st};
}

// _const_f (trace/fixed_variable.py:201-214): the least f in (-32, 32] with c * 2^f an integer; -32 for 0
inline int pp_const_f(double c) {
    if (c == 0.0)
        return -32;
    int lo = -32, hi = 32;
    while (hi - lo > 1) {
        const int mid = (hi + lo) >> 1; // (floor division, as Python's //)
        const double v = std::ldexp(c, mid);
        if (v == std::trunc(v))
            hi = mid;
        else
            lo = mid;
    }
    return hi;
}

// sum of minimal_kif of an interval
inline int pp_kif_bits(double lo, double hi, double step) {
    int k, i, f;
    pp_minimal_kif(lo, hi, step, k, i, f);
    return k + i + f;
}

// Check one design's arrays (DA4ML_E_INVALID-class errors are thrown as std::invalid_argument) and prepare it.
inline PpPrepared pp_prepare(const PpStageIn *st, int64_t n_stages, PpSplitInfo *split = nullptr) {
    auto scaled = [](PpView v, double s) {
        const double a = v.lo * s, b = v.hi * s;
        return PpView{v.node, std::min(a, b), std::max(a, b), std::fabs(v.step * s), v.f * s};
    };
    // FixedVariable.__neg__: Decimal negation, whose zero is +0 (a product with a negative power of two gives -0)
    auto negated = [](PpView v) { return PpView{v.node, 0.0 - v.hi, 0.0 - v.lo, v.step, -v.f}; };
    auto bad = [](const std::string &m) { throw std::invalid_argument("pipeline_price: " + m); };
    if (n_stages < 1)
        bad("a design needs at least one stage");
    PpPrepared P;
    P.n_in = (int)st[0].n_in;
    P.adder_size = (int)st[0].adder_size;
    P.carry_size = (int)st[0].carry_size;
    const int CONST = P.n_in;
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
            const bool act = o[2] == 2 || o[2] == -2 || o[2] == 3 || o[2] == -3;
            const bool cadd = o[2] == 4; // a constant addition: data (!= 0, as the tracer records none of 0) steps of its interval
            // a lookup: data the index of its table.  The tables themselves do not reach the kernels (a lookup's cost and
            // latency depend on intervals only), so the caller checks the index against them: the Python host does
            // (_design_tables), and a direct C ABI caller must.
            const bool lut = o[2] == 8;
            // an MSB mux: data = shift << 32 | the condition's op (types.py:272-281)
            const bool mux = o[2] == 6 || o[2] == -6;
            const int64_t mux_c = o[3] & 0xffffffffll;
            const int32_t mux_sh = (int32_t)(uint32_t)((uint64_t)o[3] >> 32);
            const bool ok = o[2] == -1 ? (o[0] >= 0 && o[0] < S.n_in && std::abs(S.inp_shifts[o[0]]) <= 512)
                            : (o[2] == 0 || o[2] == 1) ? (o[0] >= 0 && o[0] < i && o[1] >= 0 && o[1] < i && std::abs(o[3]) <= 512)
                            : act  ? (o[0] >= 0 && o[0] < i && o[1] == -1 && o[3] == 0)
                            : cadd ? (o[0] >= 0 && o[0] < i && o[1] == -1 && o[3] != 0 && std::llabs(o[3]) < (1ll << 31))
                            : lut  ? (o[0] >= 0 && o[0] < i && o[1] == -1 && o[3] >= 0 && o[3] < (1ll << 31))
                            : mux  ? (o[0] >= 0 && o[0] < i && o[1] >= 0 && o[1] < i && mux_c < i && std::abs(mux_sh) <= 512)
                                   : false;
            if (!ok)
                bad("stage " + std::to_string(s) + " op " + std::to_string(i) + ": opcode " + std::to_string(o[2]) + " with operands (" + std::to_string(o[0]) + ", " +
                    std::to_string(o[1]) + ") and data " + std::to_string(o[3]) + " is not an adder-graph op (opcodes -1, 0, 1, the activations +-2, +-3 "
                    "and the constant addition 4 with 0 < |data| < 2^31, the lookup 8 with a table index, the MSB mux +-6 with data shift << 32 | "
                    "condition; operands earlier ops, inputs in range)");
            if (act || cadd || lut || mux) { // the op's interval gives the activation's (k, i, f): a finite interval on a power-of-two grid
                const float *q = S.ops_f + 5 * i;
                const double lo = q[0], hi = q[1], st = q[2];
                int e = 0;
                const bool grid = std::isfinite(lo) && std::isfinite(hi) && st > 0 && std::isfinite(st) && std::frexp(st, &e) == 0.5 && lo <= hi &&
                                  std::fabs(lo / st) < 9.0e15 && std::fabs(hi / st) < 9.0e15 && lo / st == std::trunc(lo / st) && hi / st == std::trunc(hi / st);
                if (!grid)
                    bad("stage " + std::to_string(s) + " op " + std::to_string(i) + ": the interval of an " + (act ? "activation" : cadd ? "opcode 4 constant addition" : lut ? "opcode 8 lookup" : "opcode +-6 MSB mux") +
                        " is not a quantized interval (min <= max, multiples of a power-of-two step)");
            }
        }
        for (int64_t k = 0; k < S.n_out; ++k)
            if (S.out_idxs[k] < -1 || S.out_idxs[k] >= S.n_ops || std::abs(S.out_shifts[k]) > 512)
                bad("stage " + std::to_string(s) + " output " + std::to_string(k) + " is out of range");
    }
    struct Node {
        PpView v;        // the view the node was created with
        int lvl;         // dependency level: 0 for the inputs and the constant
        bool cadd, wrap; // a constant addition / a quantize (FixedVariable.opr == 'cadd' / 'wrap')
    };
    std::vector<Node> nodes(P.n_in + 1); // indexed by node id
    for (int k = 0; k < P.n_in; ++k)
        nodes[k].v = PpView{k, 0.0, 0.0, 1.0, 1.0};
    for (int64_t i = 0; i < st[0].n_ops; ++i) // the design's input intervals (CombLogic.inp_qint)
        if (st[0].ops_i[4 * i + 2] == -1) {
            const int k = (int)st[0].ops_i[4 * i];
            const float *q = st[0].ops_f + 5 * i;
            nodes[k].v = PpView{k, q[0], q[1], q[2], 1.0};
        }
    nodes[CONST].v = PpView{CONST, 0.0, 0.0, 4294967296.0, 1.0};
    std::vector<PpAdd> adds;
    const PpView none{-1, 0.0, 0.0, 0.0, 0.0};
    // Record op `a` as the next node, created with view `v` (both get its id), with its level and split record; returns
    // the view.  Node ids are the order of this call.
    auto add_node = [&](PpAdd a, PpView v, const PpSplitOp &op, bool cadd = false, bool wrap = false) {
        a.node = v.node = (int)nodes.size();
        const int lvl = 1 + std::max(std::max(nodes[a.n0].lvl, nodes[a.n1].lvl), a.nc >= 0 ? nodes[a.nc].lvl : 0);
        adds.push_back(a);
        nodes.push_back(Node{v, lvl, cadd, wrap});
        if (split)
            split->ops.push_back(op);
        return v;
    };
    // replay: cur = the views entering the stage
    std::vector<PpView> cur(P.n_in);
    for (int k = 0; k < P.n_in; ++k) {
        const PpView &w = nodes[k].v;
        cur[k] = w.lo == w.hi ? PpView{CONST, w.lo, w.hi, w.step, 1.0} : w;
    }
    for (int64_t s = 0; s < n_stages; ++s) {
        const PpStageIn &S = st[s];
        std::vector<PpView> buf(S.n_ops);
        for (int64_t i = 0; i < S.n_ops; ++i) {
            const int64_t *o = S.ops_i + 4 * i;
            if (o[2] == -1) {
                buf[i] = scaled(cur[o[0]], std::ldexp(1.0, (int)S.inp_shifts[o[0]]));
                continue;
            }
            if (o[2] == 4) { // FixedVariable._const_add of data * step (CombLogic.__call__, types.py:267-269)
                const PpView V = buf[o[0]];
                const double bias = (double)o[3] * (double)S.ops_f[5 * i + 2];
                PpAdd a{};
                a.n0 = a.n1 = V.node, a.nc = -1;
                a.flag = PP_ONE_OPERAND;
                PpView R{-1, V.lo + bias, V.hi + bias, std::min(V.step, std::ldexp(1.0, -pp_const_f(bias))), V.f};
                if (V.lo == V.hi) { // a constant plus a constant: not supported, as an adder of a constant is not
                    a.flag = PP_CONST_CADD;
                    R.step = V.step;
                } else if (nodes[V.node].cadd) {
                    bad("stage " + std::to_string(s) + " op " + std::to_string(i) + ": an opcode 4 constant addition of a constant addition (the tracer folds "
                        "the two into one op on the earlier operand; not covered)");
                }
                const double d = bias / V.f; // the node's _data, and the tracer's cost ceil(log2(|d| + 2^-f)) + f
                const int fd = pp_const_f(d);
                a.q0[0] = (float)(std::ceil(std::log2(std::fabs(d) + std::ldexp(1.0, -fd))) + fd);
                // data: int(_data / unscaled step), the same through every view of the node
                buf[i] = add_node(a, R, PpSplitOp{V, none, none, 4, (int)std::llround(d / (R.step / std::fabs(V.f)))}, true);
                continue;
            }
            if (o[2] == 6 || o[2] == -6) { // CombLogic.__call__: k.msb_mux(v0, +-v1 * 2^shift, op.qint) (types.py:272-281)
                const PpView K = buf[o[3] & 0xffffffffll];
                PpView A = buf[o[0]], B = o[2] < 0 ? negated(buf[o[1]]) : buf[o[1]];
                B = scaled(B, std::ldexp(1.0, (int32_t)(uint32_t)((uint64_t)o[3] >> 32)));
                const std::string at = "stage " + std::to_string(s) + " op " + std::to_string(i) + ": an opcode +-6 MSB mux ";
                if (K.lo == K.hi || A.lo == A.hi || B.lo == B.hi)
                    bad(at + "with a constant operand (not covered)");
                if (!(K.f > 0)) // (trace/tracer.py:119 asserts it of every traced mux)
                    bad(at + "whose condition has a negative factor (the tracer asserts a positive one)");
                if (nodes[K.node].wrap)
                    bad(at + "whose condition is a quantize (the tracer may mux on its operand instead; not covered)");
                // FixedVariable.msb_mux (trace/fixed_variable.py:788-859) with the explicit qint: a negative factor of a
                // mirrors the qint and muxes -a, -b, seen negated
                const float *q = S.ops_f + 5 * i;
                double qlo = q[0], qhi = q[1];
                const bool neg = A.f < 0;
                if (neg) {
                    const double t0 = 0.0 - qhi;
                    qhi = 0.0 - qlo, qlo = t0;
                    A = negated(A), B = negated(B);
                }
                const double step = std::min(A.step, B.step);
                if (!((double)q[2] <= step))
                    bad(at + "whose interval's step is larger than its operands' (the tracer asserts it is not)");
                const double lo = std::max((std::floor(qlo / step) + 0.0) * step, std::min(A.lo, B.lo));
                const double hi = std::min((std::floor(qhi / step) + 0.0) * step, std::max(A.hi, B.hi));
                PpAdd a{};
                a.n0 = A.node, a.n1 = B.node, a.nc = K.node;
                a.flag = PP_MUX;
                float dl = 0.f, cost = 0.f;
                cost_add(QInt{(float)A.lo, (float)A.hi, (float)A.step}, QInt{(float)B.lo, (float)B.hi, (float)B.step}, 0, false, P.adder_size, P.carry_size, dl, cost);
                a.q0[0] = cost / 2.f;
                a.q0[1] = dl;
                const PpView R = add_node(a, PpView{-1, lo, hi, step, A.f}, PpSplitOp{A, B, K, B.f > 0 ? 6 : -6, (int)std::log2(std::fabs(B.f / A.f))});
                buf[i] = neg ? negated(R) : R;
                continue;
            }
            if (o[2] == 8) { // FixedVariable.lookup of the operand (CombLogic.__call__): the table's interval, factor 1
                const PpView V = buf[o[0]];
                if (V.lo == V.hi)
                    bad("stage " + std::to_string(s) + " op " + std::to_string(i) + ": an opcode 8 lookup of a constant (the tracer makes a constant of it; not covered)");
                const float *q = S.ops_f + 5 * i;
                PpAdd a{};
                a.n0 = a.n1 = V.node, a.nc = -1;
                a.flag = PP_LOOKUP;
                // get_cost_and_latency: b_in the kif bits of the operand as the tracer sees it, b_out the result's
                const int b_in = pp_kif_prop_bits(V.lo, V.hi, V.step), b_out = pp_kif_prop_bits(q[0], q[1], q[2]);
                double cost = std::ldexp(1.0, std::max(b_in - 5, 0)) * std::ceil(b_out / 2.0);
                if (b_in < 5)
                    cost *= b_in / 5.0;
                a.q0[0] = (float)cost;
                a.q0[1] = (float)std::max(b_in - 6, 1);
                buf[i] = add_node(a, PpView{-1, q[0], q[1], q[2], 1.0}, PpSplitOp{V, none, none, 8, (int)o[3]});
                continue;
            }
            if (o[2] != 0 && o[2] != 1) { // relu (+-2) / quantize (+-3) of the operand (negated for the negative opcode)
                PpView V = o[2] < 0 ? negated(buf[o[0]]) : buf[o[0]];
                if (V.lo == V.hi) { // a constant: the tracer folds it (relu / quantize of 0 is 0)
                    if (V.lo != 0.0)
                        bad("stage " + std::to_string(s) + " op " + std::to_string(i) + ": an activation of the constant " + std::to_string(V.lo) +
                            " (only the constant 0 is covered)");
                    buf[i] = nodes[CONST].v;
                    continue;
                }
                const float *q = S.ops_f + 5 * i;
                int kk, ii, ff;
                pp_minimal_kif(q[0], q[1], q[2], kk, ii, ff);
                const bool relu = std::abs(o[2]) == 2;
                const PpAct r = relu ? pp_relu(V.lo, V.hi, V.step, ii, ff) : pp_quantize(V.lo, V.hi, V.step, kk, ii, ff);
                if (r.kind == 0) {
                    buf[i] = V;
                    continue;
                }
                if (r.kind == 1) {
                    if (r.lo != 0.0)
                        bad("stage " + std::to_string(s) + " op " + std::to_string(i) + ": the activation makes the constant " + std::to_string(r.lo) +
                            " (only the constant 0 is covered)");
                    buf[i] = nodes[CONST].v;
                    continue;
                }
                PpAdd a{};
                a.n0 = a.n1 = V.node, a.nc = -1;
                a.flag = PP_ONE_OPERAND;
                const int kb = pp_kif_prop_bits(r.lo, r.hi, r.step); // the tracer's cost: half a LUT per bit for relu, and for a negation
                a.q0[0] = (float)((V.f < 0 ? kb / 2.0 : 0.0) + (relu ? kb / 2.0 : 0.0));
                buf[i] = add_node(a, PpView{-1, r.lo, r.hi, r.step, std::fabs(V.f)}, PpSplitOp{V, none, none, (V.f < 0 ? -1 : 1) * (relu ? 2 : 3), 0}, false, !relu);
                continue;
            }
            PpView A = buf[o[0]], B = scaled(buf[o[1]], std::ldexp(1.0, (int)o[3]));
            if (o[2] == 1)
                B = negated(B);
            PpAdd a{};
            a.n0 = A.node, a.n1 = B.node, a.nc = -1;
            a.flag = (A.lo == A.hi || B.lo == B.hi) ? PP_CONST_OPERAND : PP_ADDER;
            PpView X = A, Y = B; // FixedVariable.__add__: the operand with a positive factor first; both negative: negate both
            bool neg = false;
            if (A.f < 0) {
                if (B.f > 0)
                    X = B, Y = A;
                else
                    X = negated(A), Y = negated(B), neg = true;
            }
            // the new node is X + Y (factor X.f), seen negated when both operands were; in this order, as the tracer's
            // Decimal arithmetic gives the signs of zero bounds (which reach the split's op intervals)
            const double clo = X.lo + Y.lo, chi = X.hi + Y.hi, step = std::min(A.step, B.step);
            const double lo = neg ? 0.0 - chi : clo, hi = neg ? 0.0 - clo : chi, f = neg ? -X.f : X.f;
            a.q0[0] = (float)X.lo, a.q0[1] = (float)X.hi, a.q0[2] = (float)X.step;
            a.q1[0] = (float)Y.lo, a.q1[1] = (float)Y.hi, a.q1[2] = (float)Y.step;
            if (a.flag == PP_ADDER && lo == hi)
                a.flag = PP_CONST_SUM;
            buf[i] = add_node(a, PpView{-1, lo, hi, step, f}, PpSplitOp{X, Y, none, Y.f < 0, (int)std::log2(std::fabs(Y.f / X.f))});
        }
        std::vector<PpView> next(S.n_out);
        for (int64_t k = 0; k < S.n_out; ++k) {
            const int64_t i = S.out_idxs[k];
            if (i < 0)
                next[k] = nodes[CONST].v;
            else
                next[k] = scaled(scaled(buf[i], std::ldexp(1.0, (int)S.out_shifts[k])), S.out_negs[k] ? -1.0 : 1.0);
        }
        cur.swap(next);
    }
    P.n_nodes = (int)nodes.size();
    P.n_out = (int)cur.size();
    if (split) {
        split->own_q.resize(3 * (size_t)P.n_nodes);
        for (int v = 0; v < P.n_nodes; ++v) {
            const PpView w = scaled(nodes[v].v, 1.0 / nodes[v].v.f); // FixedVariable.unscaled
            split->own_q[3 * v] = w.lo, split->own_q[3 * v + 1] = w.hi, split->own_q[3 * v + 2] = w.step;
        }
        split->out_v = cur;
        for (const PpView &v : cur) {
            split->out_shift.push_back((int64_t)std::log2(std::fabs(v.f)));
            split->out_neg.push_back(v.f < 0);
        }
    }
    // liveness (comb_trace's dead-statement elimination) and bits
    std::vector<char> live(P.n_nodes, 0);
    for (const PpView &v : cur) {
        P.out_node.push_back(v.node);
        live[v.node] = 1;
        P.out_bits += v.node == CONST ? 0 : pp_kif_bits(v.lo, v.hi, v.step);
    }
    for (size_t k = adds.size(); k-- > 0;)
        if (live[adds[k].node]) {
            live[adds[k].n0] = live[adds[k].n1] = 1;
            if (adds[k].nc >= 0)
                live[adds[k].nc] = 1;
        }
    P.node_bits.assign(P.n_nodes, -1);
    for (int v = 0; v < P.n_nodes; ++v) {
        if (!live[v])
            continue;
        if (v == CONST) {
            P.node_bits[v] = 0;
            continue;
        }
        PpView w = nodes[v].v;
        if (w.f < 0)
            w = scaled(w, -1.0); // the node's own interval (the op's qint in the traced graph)
        P.node_bits[v] = pp_kif_bits(w.lo, w.hi, w.step);
    }
    // adders by level (stable: replay order within a level); level l + 1 is adds[lvl_begin[l], lvl_begin[l + 1])
    int n_lv = 0;
    for (const PpAdd &a : adds)
        n_lv = std::max(n_lv, nodes[a.node].lvl);
    P.lvl_begin.assign(n_lv + 1, 0);
    for (const PpAdd &a : adds)
        ++P.lvl_begin[nodes[a.node].lvl];
    for (int l = 1; l <= n_lv; ++l)
        P.lvl_begin[l] += P.lvl_begin[l - 1];
    std::vector<int> pos(P.lvl_begin.begin(), P.lvl_begin.end() - 1);
    P.adds.resize(adds.size());
    for (const PpAdd &a : adds)
        P.adds[pos[nodes[a.node].lvl - 1]++] = a;
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
