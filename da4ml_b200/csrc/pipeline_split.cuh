// pipeline_split.cuh -- build the register stages of solver designs (the op tables of every stage) as the reference's
// deploy path does: re-trace under a latency cutoff, gather with comb_trace, split with to_pipeline (reference:
// trace/tracer.py gather_variables / _comb_trace / dead_statement_elimination; trace/pipeline.py to_pipeline and
// _get_new_idx; retime_pipeline keeps the split of its last successful round).
//
// A split task is a priced task (pipeline_price.cuh) at the (cutoff, input latencies) its split comes from.  The host
// adds, per design and only when splits are asked for, what pricing does not need: the *items* -- gather_variables'
// list before its sort (every input, then the adders reachable from the outputs, and one constant per all-zero output
// column, which pp_prepare folds into one node) -- with each item's gather position, its own interval and, for an adder,
// FixedVariable.__add__'s operand order and the op it becomes.  Two kernels, one CTA per task:
//   pipeline_split_kernel        replays the latencies through pp_replay (the pricing kernel's code), sorts the items by
//                                gather_variables' key lat * N + position (a CTA-wide LSD radix sort of the key's IEEE
//                                bits; stable, so ties go to the lower position), gives every item its producer stage
//                                and last consumer stage, finds the items dead_statement_elimination keeps, and counts
//                                the rows and outputs of every stage.  A stage with
//                                no row or (before the last) no output is to_pipeline's KeyError, reported per task.
//   pipeline_split_write_kernel  finds for every copy (a value carried across boundary j) the first event that needs it
//                                (events: (op, operand 0 / operand 1 / a mux's condition / the op itself), then the
//                                outputs, the order of to_pipeline's _get_new_idx calls), orders every
//                                stage's rows by the event that created them (a second radix sort over (stage, event)),
//                                and writes the op tables with operands remapped to the reading stage's rows.
// ps_split drives both, between them one small copy of the counts; the tables come back in one copy.
#pragma once
#include "pipeline_price.cuh"

#include <cstring>

namespace da {

enum PsStatus : int { PS_SPLIT = 0, PS_NOT_OK = 1 /* the task is not ok: no split */, PS_KEY_ERROR = 2 /* to_pipeline raises KeyError */, PS_INTERNAL = 3 };

// What an item that is not a network input is (PsItem::inp < 0)
enum PsKind : int {
    PS_ADDER = -1,
    PS_CONSTANT = -2,     // an all-zero output column
    PS_ONE_OPERAND = -3,  // relu / quantize (opcodes +-2 / +-3), a constant addition (4) or a lookup (8)
    PS_MUX = -4,          // an MSB mux (opcode +-6)
};

struct PsItem {
    double lo, hi, step;  // the op's interval (the node's own)
    long long data;       // see x, y, z, opc
    int node, gpos;       // node id (PpDesign) and position in gather_variables' list
    int inp;              // >= 0: network input k; else a PsKind
    int x, y, z, opc;     // adder: items of the operands in _from order, opcode, data the shift; one-operand op: the
                          // operand's item, y -1, opcode and data as PpSplitOp; MSB mux: the data operands a, b and the
                          // condition z (_from is (z, a, b)), opcode +-6, data the shift of b (the written op's data is
                          // shift << 32 | the condition's row); input: opcode -1, or 5 and the value in steps for an input
                          // with a point interval (a constant to the tracer).  z is -1 but for a mux.
    int live;             // reachable from the outputs
};

struct PsDesign {
    PpDesign pp;
    const PsItem *items;  // [n_items] in gather order
    const int *out_item;  // [n_out]
    int n_items;          // gather_variables' N: every input, kept or not, and every traced node
};

struct PsCount {
    int status, n_st, s_out, n_copies, n_kept, pad;
};

struct PsTask {
    PpTask pp;            // design, cutoff, latencies, lat workspace [n_nodes]
    int n_st, pad;        // the stage count pricing found for this (cutoff, latencies)
    PsCount *count;
    int *nrow, *nout;     // [n_st] rows / outputs of each stage
    float *cost;          // [n_nodes]
    unsigned long long *key, *key2;
    int *val, *val2, *rank, *stg, *last, *keep, *flag, *inpos, *coff, *cnt; // [n_items] ([n_items + 1] flag, coff; [16 * threads + 1] cnt)
    // write pass
    int *ev, *cown, *cpos, *ownpos, *cscan, *start;   // [copies] x3, [n_items], [rows + 1], [n_st + 1]
    unsigned long long *rkey, *rkey2;
    int *rval, *rval2;                                // [n_items + copies]
    int64_t *ops_i, *outs;                            // [rows][4], [copies + n_out]
    double *ops_f;                                    // [rows][5]
};

struct PsShared {
    unsigned long long fail, latmax, and_, or_;
    int kept, beyond, part[1025];
};

// exclusive scan of a[0, n) in place, a[n] = the total.  Every thread of the CTA calls it; it ends with a barrier.
__device__ __forceinline__ void ps_scan(int *a, int n, PsShared &sh) {
    const int tid = threadIdx.x, nt = blockDim.x, ch = (n + nt - 1) / nt;
    const int b = min(n, tid * ch), e = min(n, b + ch);
    int s = 0;
    for (int i = b; i < e; ++i)
        s += a[i];
    sh.part[tid] = s;
    __syncthreads();
    if (tid == 0) {
        int run = 0;
        for (int k = 0; k < nt; ++k) {
            const int v = sh.part[k];
            sh.part[k] = run;
            run += v;
        }
        sh.part[nt] = run;
        a[n] = run;
    }
    __syncthreads();
    s = sh.part[tid];
    for (int i = b; i < e; ++i) {
        const int v = a[i];
        a[i] = s;
        s += v;
    }
    __syncthreads();
}

// Stable LSD radix sort of (key, val)[0, n) by key, 4 bits a pass; passes whose digit is the same in every key are
// skipped.  The result is in (key, val) on return (the pointers are swapped with the second buffers as needed).  `cnt`:
// [16 * blockDim.x + 1].  Each thread takes one contiguous chunk, so a pass keeps the order of equal digits.
__device__ __forceinline__ void ps_sort(unsigned long long *&key, int *&val, unsigned long long *&key2, int *&val2, int n, int *cnt, PsShared &sh) {
    const int tid = threadIdx.x, nt = blockDim.x, ch = (n + nt - 1) / nt;
    const int b = min(n, tid * ch), e = min(n, b + ch);
    if (tid == 0)
        sh.and_ = ~0ull, sh.or_ = 0ull;
    __syncthreads();
    unsigned long long a = ~0ull, o = 0ull;
    for (int i = b; i < e; ++i)
        a &= key[i], o |= key[i];
    atomicAnd(&sh.and_, a);
    atomicOr(&sh.or_, o);
    __syncthreads();
    const unsigned long long diff = sh.and_ ^ sh.or_;
    for (int shift = 0; shift < 64; shift += 4) {
        if (((diff >> shift) & 15ull) == 0)
            continue;
        int c[16];
        for (int d = 0; d < 16; ++d)
            c[d] = 0;
        for (int i = b; i < e; ++i)
            ++c[(key[i] >> shift) & 15ull];
        for (int d = 0; d < 16; ++d)
            cnt[d * nt + tid] = c[d];
        __syncthreads();
        ps_scan(cnt, 16 * nt, sh);
        for (int d = 0; d < 16; ++d)
            c[d] = cnt[d * nt + tid];
        for (int i = b; i < e; ++i) {
            const int o2 = c[(key[i] >> shift) & 15ull]++;
            key2[o2] = key[i];
            val2[o2] = val[i];
        }
        __syncthreads();
        unsigned long long *tk = key;
        key = key2, key2 = tk;
        int *tv = val;
        val = val2, val2 = tv;
    }
}

__global__ void __launch_bounds__(256) pipeline_split_kernel(const PsDesign *designs, const PsTask *tasks) {
    DA_SHARED_VAR(PsShared, sh);
    const PsTask t = tasks[blockIdx.x];
    const PsDesign D = designs[t.pp.design];
    const PpDesign &d = D.pp;
    const double c = t.pp.cutoff;
    const int tid = threadIdx.x, nt = blockDim.x, M = D.n_items;
    if (tid == 0)
        sh.fail = ~0ull, sh.latmax = 0ull, sh.kept = 0, sh.beyond = 0;
    for (int v = tid; v < d.n_nodes; v += nt)
        t.pp.lat[v] = v < d.n_in && t.pp.in_lat ? t.pp.in_lat[v] : 0.0;
    __syncthreads();
    pp_replay<true>(d, t.pp, sh.fail, t.cost);
    if (sh.fail != ~0ull) {
        if (tid == 0)
            *t.count = PsCount{PS_NOT_OK, 0, -1, 0, 0, 0};
        return;
    }
    const double *lat = t.pp.lat;
    for (int i = tid; i < M; i += nt) {
        const PsItem &it = D.items[i];
        t.key[i] = pp_dbits(pp_add(pp_mul(lat[it.node], (double)M), (double)it.gpos)); // gather_variables' key
        t.val[i] = i;
        t.stg[i] = t.last[i] = pp_stage(lat[it.node], c);
        t.keep[i] = it.live;
    }
    for (int o = tid; o < d.n_out; o += nt)
        atomicMax(&sh.latmax, pp_dbits(lat[D.items[D.out_item[o]].node]));
    __syncthreads();
    unsigned long long *key = t.key, *key2 = t.key2;
    int *val = t.val, *val2 = t.val2;
    ps_sort(key, val, key2, val2, M, t.cnt, sh);
    for (int r = tid; r < M; r += nt) {
        t.rank[val[r]] = r;
        t.flag[r] = val[r] < d.n_in;
    }
    const int s_out = pp_stage(pp_bitsd(sh.latmax), c), n_st = s_out + 1;
    if (n_st != t.n_st) { // (pricing found another stage count: cannot happen, the replay is the same code)
        if (tid == 0)
            *t.count = PsCount{PS_INTERNAL, n_st, s_out, 0, 0, 0};
        return;
    }
    __syncthreads();
    // dead_statement_elimination walks the sorted list backwards from the outputs and keeps what a kept op reads through
    // id0 / id1.  An input op's id0 is its input number, so a kept input k also keeps whatever sits at position k of the
    // list, which is another input than k when input latencies reorder the list (an input nothing reads, kept as the
    // reference keeps it).  Everything else the walk keeps is live already.  Inputs in descending position:
    ps_scan(t.flag, M, sh);
    for (int r = tid; r < M; r += nt)
        if (val[r] < d.n_in)
            t.inpos[t.flag[r]] = r;
    __syncthreads();
    if (tid == 0)
        for (int q = d.n_in - 1; q >= 0; --q) {
            const int k = val[t.inpos[q]];
            if (t.keep[k] && D.items[k].opc != 5 && k < M && val[k] < d.n_in)
                t.keep[val[k]] = 1;
        }
    // last consumer stage of every item: the stage of each adder reading it, and the output stage
    for (int i = tid; i < M; i += nt) {
        const PsItem &it = D.items[i];
        if (it.inp == PS_ADDER || it.inp == PS_ONE_OPERAND || it.inp == PS_MUX)
            atomicMax(&t.last[it.x], t.stg[i]);
        if (it.inp == PS_ADDER || it.inp == PS_MUX)
            atomicMax(&t.last[it.y], t.stg[i]);
        if (it.inp == PS_MUX)
            atomicMax(&t.last[it.z], t.stg[i]);
    }
    for (int o = tid; o < d.n_out; o += nt)
        atomicMax(&t.last[D.out_item[o]], s_out);
    for (int s = tid; s < n_st; s += nt)
        t.nrow[s] = t.nout[s] = 0;
    __syncthreads();
    // an item produced in stage p and last read in stage q is copied into stages p + 1 .. q: one row there each, and one
    // output of the stage before
    for (int i = tid; i < M; i += nt)
        t.coff[i] = t.last[i] - t.stg[i];
    __syncthreads();
    ps_scan(t.coff, M, sh);
    // A kept item past the output stage (an input nothing reads, kept by the walk above, whose own latency is later than
    // every output's) gives to_pipeline a stage with ops and no outputs: its KeyError.  Nothing reads such an item, so
    // it has no copies; it is counted nowhere.
    for (int i = tid; i < M; i += nt) {
        if (!t.keep[i])
            continue;
        if (t.stg[i] < 0 || t.stg[i] > s_out) {
            sh.beyond = 1;
            continue;
        }
        atomicAdd(&sh.kept, 1);
        atomicAdd(&t.nrow[t.stg[i]], 1);
        for (int s = t.stg[i] + 1; s <= t.last[i]; ++s) {
            atomicAdd(&t.nrow[s], 1);
            atomicAdd(&t.nout[s - 1], 1);
        }
    }
    __syncthreads();
    if (tid == 0) {
        bool key_error = sh.beyond != 0;
        for (int s = 0; s < n_st; ++s)
            key_error |= t.nrow[s] == 0 || (s < s_out && t.nout[s] == 0);
        t.nout[s_out] = d.n_out;
        *t.count = PsCount{key_error ? PS_KEY_ERROR : PS_SPLIT, n_st, s_out, t.coff[M], sh.kept, 0};
    }
}

__global__ void __launch_bounds__(256) pipeline_split_write_kernel(const PsDesign *designs, const PsTask *tasks) {
    DA_SHARED_VAR(PsShared, sh);
    const PsTask t = tasks[blockIdx.x];
    const PsDesign D = designs[t.pp.design];
    const PsCount k0 = *t.count;
    const int tid = threadIdx.x, nt = blockDim.x, M = D.n_items, C = k0.n_copies, R = k0.n_kept + C, s_out = k0.s_out, n_out = D.pp.n_out;
    const long long E = 4ll * M + n_out; // events: 4 * (op position) + (0, 1: its operands; 2: a mux's condition; 3: the op), then 4M + output
    const double c = t.pp.cutoff;
    const int *stg = t.stg, *coff = t.coff, *rank = t.rank;
    for (int i = tid; i < M; i += nt)
        for (int k = coff[i]; k < coff[i + 1]; ++k)
            t.ev[k] = 0x7fffffff, t.cown[k] = i;
    __syncthreads();
    // copy k of item v carries it across boundary stg[v] + k - coff[v]; an event placing v in stage s needs the copies
    // across every boundary below s: record it at the last one, a suffix min then gives each copy its first event
    for (int i = tid; i < M; i += nt) {
        const PsItem &it = D.items[i];
        if (it.inp != PS_ADDER && it.inp != PS_ONE_OPERAND && it.inp != PS_MUX)
            continue;
        const int s = stg[i];
        if (s > stg[it.x])
            atomicMin(&t.ev[coff[it.x] + s - 1 - stg[it.x]], 4 * rank[i]);
        if (it.inp != PS_ONE_OPERAND && s > stg[it.y])
            atomicMin(&t.ev[coff[it.y] + s - 1 - stg[it.y]], 4 * rank[i] + 1);
        if (it.inp == PS_MUX && s > stg[it.z])
            atomicMin(&t.ev[coff[it.z] + s - 1 - stg[it.z]], 4 * rank[i] + 2);
    }
    for (int o = tid; o < n_out; o += nt) {
        const int v = D.out_item[o];
        if (s_out > stg[v])
            atomicMin(&t.ev[coff[v] + s_out - 1 - stg[v]], 4 * M + o);
    }
    __syncthreads();
    for (int i = tid; i < M; i += nt)
        for (int k = coff[i + 1] - 2; k >= coff[i]; --k)
            t.ev[k] = min(t.ev[k], t.ev[k + 1]);
    __syncthreads();
    // rows: the item's own (its stage, event 4p + 3) and its copies (stage j + 1, the copy's event); the R rows of the
    // split sort before the items that are not kept
    for (int i = tid; i < M; i += nt) {
        t.rkey[i] = t.keep[i] ? (unsigned long long)stg[i] * E + 4ull * rank[i] + 3 : (unsigned long long)k0.n_st * E;
        t.rval[i] = i;
    }
    for (int k = tid; k < C; k += nt) {
        const int i = t.cown[k];
        t.rkey[M + k] = (unsigned long long)(stg[i] + k - coff[i] + 1) * E + (unsigned long long)t.ev[k];
        t.rval[M + k] = M + k;
    }
    __syncthreads();
    unsigned long long *rkey = t.rkey, *rkey2 = t.rkey2;
    int *rval = t.rval, *rval2 = t.rval2;
    ps_sort(rkey, rval, rkey2, rval2, M + C, t.cnt, sh);
    for (int r = tid; r < R; r += nt) {
        const long long s = (long long)(rkey[r] / E); // (< n_st: a task with a kept item past the output stage is not written)
        if (s < k0.n_st && (r == 0 || (long long)(rkey[r - 1] / E) != s))
            t.start[s] = r;
        t.cscan[r] = rval[r] >= M;
    }
    if (tid == 0)
        t.start[k0.n_st] = R;
    __syncthreads();
    ps_scan(t.cscan, R, sh); // copy rows before each row
    for (int r = tid; r < R; r += nt) {
        const int s = (int)(rkey[r] / E), v = rval[r], pos = r - t.start[s];
        if (v < M)
            t.ownpos[v] = pos;
        else
            t.cpos[v - M] = pos;
    }
    __syncthreads();
    auto where = [&](int v, int s) { return s == stg[v] ? t.ownpos[v] : t.cpos[coff[v] + s - 1 - stg[v]]; }; // row of item v in stage s
    for (int r = tid; r < R; r += nt) {
        const int s = (int)(rkey[r] / E), v = rval[r];
        int64_t *oi = t.ops_i + 4 * (size_t)r;
        double *of = t.ops_f + 5 * (size_t)r;
        if (v < M) {
            const PsItem &it = D.items[v];
            double cost = 0.0;
            if (it.inp >= 0 && it.opc == 5) // an input with a point interval: a constant
                oi[0] = -1, oi[1] = -1, oi[2] = 5, oi[3] = it.data;
            else if (it.inp >= 0)
                oi[0] = it.inp, oi[1] = -1, oi[2] = -1, oi[3] = 0;
            else if (it.inp == PS_CONSTANT)
                oi[0] = -1, oi[1] = -1, oi[2] = 5, oi[3] = 0;
            else {
                oi[0] = where(it.x, s), oi[1] = it.inp != PS_ONE_OPERAND ? where(it.y, s) : -1, oi[2] = it.opc, oi[3] = it.data;
                if (it.inp == PS_MUX) // to_pipeline's shift << 32 | the condition's row, the shift as its low 32 bits
                    oi[3] = (int64_t)(((unsigned long long)(unsigned)it.data << 32) | (unsigned long long)where(it.z, s));
                cost = (double)t.cost[it.node];
            }
            of[0] = it.lo, of[1] = it.hi, of[2] = it.step, of[3] = t.pp.lat[it.node], of[4] = cost;
        }
        else { // a copy into stage s: reads output `crank` of stage s - 1, which is the item's row there
            const int i = t.cown[v - M], crank = t.cscan[r] - t.cscan[t.start[s]];
            const PsItem &it = D.items[i];
            oi[0] = crank, oi[1] = -1, oi[2] = -1, oi[3] = 0;
            of[0] = it.lo, of[1] = it.hi, of[2] = it.step, of[3] = pp_mul(c, (double)s), of[4] = 0.0;
            // output `crank` of stage s - 1, whose outputs follow those of the stages before it (the copies into
            // stages 1 .. s - 1): the copy rows before this one, cscan[r]
            t.outs[t.cscan[r]] = where(i, s - 1);
        }
    }
    // the last stage's outputs: the design's
    for (int o = tid; o < n_out; o += nt)
        t.outs[C + o] = where(D.out_item[o], s_out);
}

// ---- host side ------------------------------------------------------------------------------------------------------

struct PsPrep {
    std::vector<PsItem> items;
    std::vector<int> out_item;
    std::vector<int64_t> out_shift, out_neg;
};

// gather_variables on the prepared design: every input at its position, then a depth-first post-order from the outputs
// in output order, operands in _from order (an MSB mux's condition first); the items are the gathered values
// dead_statement_elimination keeps, which treats a mux's condition as a third operand.
inline PsPrep ps_prepare(const PpPrepared &P, const PpSplitInfo &S) {
    PsPrep Q;
    const int CONST = P.n_in;
    std::vector<int> item_of(P.n_nodes, -1);
    // an op's interval is FixedVariable.unscaled of the view gather_variables met the node through first (its bounds'
    // signs of zero depend on that view's factor); own[node] is set when the walk enters the node
    std::vector<double> own(S.own_q);
    auto enter = [&](int node, const PpView &v) { // `self * (1 / factor)` in Decimal
        const double o = 1.0 / v.f, a = v.lo * o, b = v.hi * o;
        own[3 * (size_t)node] = std::min(a, b), own[3 * (size_t)node + 1] = std::max(a, b), own[3 * (size_t)node + 2] = std::fabs(v.step * o);
    };
    auto add_item = [&](int node, int gpos) {
        PsItem it{};
        it.node = node, it.gpos = gpos;
        it.lo = own[3 * (size_t)node], it.hi = own[3 * (size_t)node + 1], it.step = own[3 * (size_t)node + 2];
        it.inp = node < P.n_in ? node : PS_CONSTANT;
        it.x = it.y = it.z = -1;
        it.opc = -1;
        it.live = node < P.n_in ? P.node_bits[node] >= 0 : 1;
        if (it.inp >= 0 && it.lo == it.hi) { // (0, 0, 2^32) for 0, else the step _const_f gives the value
            it.step = std::ldexp(1.0, -pp_const_f(it.lo));
            it.opc = 5, it.data = (int)(it.lo / it.step);
        }
        if (node > CONST) {
            const PpSplitOp &op = S.ops[node - CONST - 1];
            it.inp = op.z.node >= 0 ? PS_MUX : op.y.node >= 0 ? PS_ADDER : PS_ONE_OPERAND;
            it.x = item_of[op.x.node];
            it.y = op.y.node < 0 ? -1 : item_of[op.y.node];
            it.z = op.z.node < 0 ? -1 : item_of[op.z.node];
            it.opc = op.opc, it.data = op.data;
        }
        Q.items.push_back(it);
        return (int)Q.items.size() - 1;
    };
    for (int k = 0; k < P.n_in; ++k) // every input, kept or not: the positions count them
        item_of[k] = add_item(k, k);
    int pos = P.n_in;
    std::vector<char> seen(P.n_nodes, 0);
    for (int k = 0; k < P.n_in; ++k)
        seen[k] = 1;
    struct Entry {
        int node;
        bool done;
        const PpView *view;
    };
    std::vector<Entry> stack;
    std::vector<char> entered(P.n_nodes, 0);
    for (int o = 0; o < P.n_out; ++o) {
        const int root = P.out_node[o];
        if (root == CONST) { // a fresh constant for every all-zero column
            Q.out_item.push_back(add_item(CONST, pos++));
            continue;
        }
        stack.assign(1, {root, false, &S.out_v[o]});
        while (!stack.empty()) {
            const Entry e = stack.back();
            const int v = e.node;
            stack.pop_back();
            if (e.done) {
                if (!seen[v]) {
                    seen[v] = 1;
                    item_of[v] = add_item(v, pos++);
                }
                continue;
            }
            if (seen[v])
                continue;
            if (!entered[v]) {
                entered[v] = 1;
                enter(v, *e.view);
            }
            stack.push_back({v, true, nullptr});
            if (v > CONST) {
                const PpSplitOp &op = S.ops[v - CONST - 1];
                if (op.y.node >= 0)
                    stack.push_back({op.y.node, false, &op.y});
                stack.push_back({op.x.node, false, &op.x});
                if (op.z.node >= 0) // an MSB mux's _from is (condition, a, b)
                    stack.push_back({op.z.node, false, &op.z});
            }
        }
        Q.out_item.push_back(item_of[root]);
    }
    Q.out_shift = S.out_shift;
    Q.out_neg.assign(S.out_neg.begin(), S.out_neg.end());
    return Q;
}

// One task's split as it comes back: per stage (n_in, n_out, n_ops), the stages' out_idxs and op tables concatenated.
struct PsSplit {
    int status = PS_NOT_OK, n_st = 0;
    int64_t n_rows = 0, n_outs = 0;
    std::vector<int64_t> meta;     // [n_st][3]
    size_t o_ops_i = 0, o_ops_f = 0, o_outs = 0; // byte offsets into PsResult::tables
};

struct PsResult {
    std::vector<PsSplit> tasks;                           // [n_designs * n_cutoffs]
    std::vector<char> tables;
    std::vector<std::vector<int64_t>> out_shift, out_neg; // per design: the last stage's (comb.out_shifts / out_negs)
    int64_t n_cutoffs = 1, launches = 0;
};

// {status (PsStatus), n_stages, n_rows, n_outs} of task t
inline void ps_info(const PsResult &R, int64_t t, int64_t out[4]) {
    const PsSplit &S = R.tasks[t];
    out[0] = S.status, out[1] = S.n_st, out[2] = S.n_rows, out[3] = S.n_outs;
}

// Task t's split, stages concatenated: meta [n_stages][3] (n_in, n_out, n_ops), out_idxs / out_shifts / out_negs
// [n_outs], ops_i [n_rows][4], ops_f [n_rows][5].
inline void ps_copy(const PsResult &R, int64_t t, int64_t *meta, int64_t *out_idxs, int64_t *out_shifts, int64_t *out_negs, int64_t *ops_i, double *ops_f) {
    const PsSplit &S = R.tasks[t];
    const int d = (int)(t / R.n_cutoffs);
    std::copy(S.meta.begin(), S.meta.end(), meta);
    std::memcpy(out_idxs, R.tables.data() + S.o_outs, 8 * (size_t)S.n_outs);
    std::memcpy(ops_i, R.tables.data() + S.o_ops_i, 8 * 4 * (size_t)S.n_rows);
    std::memcpy(ops_f, R.tables.data() + S.o_ops_f, 8 * 5 * (size_t)S.n_rows);
    const size_t n_last = R.out_shift[d].size(), n0 = (size_t)S.n_outs - n_last;
    std::fill(out_shifts, out_shifts + n0, 0);
    std::fill(out_negs, out_negs + n0, 0);
    std::copy(R.out_shift[d].begin(), R.out_shift[d].end(), out_shifts + n0);
    std::copy(R.out_neg[d].begin(), R.out_neg[d].end(), out_negs + n0);
}

// `Dev`: buffer(which, bytes) -> device base of buffer `which` (0: designs and count-pass workspaces, 1: write-pass
// workspaces, 2: tables), valid until the next call with the same `which`; up(dst, src, bytes) / down(dst, src, bytes)
// (down synchronises); count(designs, tasks, n) / write(designs, tasks, n): one launch of each kernel; `threads`.
// `dev_desc[d]`: the priced design's device view.  `lat` / `dev_lat`: the input latencies on the host / device (or null),
// design d's at `lat_off[d]`.
template <class Dev>
inline PsResult ps_split(const std::vector<PpPrepared> &prep, const std::vector<PsPrep> &sp, const std::vector<PpDesign> &dev_desc, const std::vector<PpAnswer> &ans,
                         const double *cutoffs, int64_t n_cutoffs, bool retiming, const double *lat, const double *dev_lat, const std::vector<int64_t> &lat_off, Dev &dev) {
    struct Job {
        int64_t task;
        int design, n_st;
        double cutoff;
        bool zero, write;
    };
    const int64_t n_tasks = (int64_t)ans.size();
    PsResult out;
    out.tasks.resize(n_tasks);
    out.n_cutoffs = n_cutoffs;
    for (const PsPrep &q : sp)
        out.out_shift.push_back(q.out_shift), out.out_neg.push_back(q.out_neg);
    std::vector<Job> jobs;
    for (int64_t t = 0; t < n_tasks; ++t) {
        const int d = (int)(t / n_cutoffs);
        const double c = cutoffs[t % n_cutoffs];
        if (ans[t].status != PP_OK)
            continue;
        jobs.push_back(Job{t, d, ans[t].stages, ans[t].retimed ? ans[t].cutoff : c, ans[t].retimed, true});
        bool late = false; // an input past the first stage: the first split (the one to_pipeline makes before retiming) may fail
        for (int k = 0; lat && k < prep[d].n_in; ++k)
            late |= pp_stage(lat[lat_off[d] + k], c) >= 1;
        if (retiming && ans[t].retimed && late)
            jobs.push_back(Job{t, d, ans[t].first_stages, c, false, false});
    }
    if (jobs.empty())
        return out;
    const int nt = dev.threads;
    struct Carver { // bump allocator, 256 B aligned pieces
        size_t off = 0;
        size_t take(size_t bytes) {
            const size_t o = off;
            off += (bytes + 255) & ~size_t(255);
            return o;
        }
    };
    // count pass: designs, workspaces, counts (one block, copied back at once)
    std::vector<char> used(prep.size(), 0);
    for (const Job &j : jobs)
        used[j.design] = 1;
    Carver c0;
    std::vector<size_t> o_items(prep.size()), o_oitem(prep.size());
    for (size_t d = 0; d < prep.size(); ++d)
        if (used[d]) {
            o_items[d] = c0.take(sizeof(PsItem) * sp[d].items.size());
            o_oitem[d] = c0.take(sizeof(int) * sp[d].out_item.size());
        }
    const size_t o_desc = c0.take(sizeof(PsDesign) * prep.size());
    std::vector<size_t> o_ws(jobs.size()), o_cnt(jobs.size());
    size_t cnt_ints = 0;
    for (size_t k = 0; k < jobs.size(); ++k) {
        o_cnt[k] = cnt_ints;
        cnt_ints += 6 + 2 * (size_t)jobs[k].n_st;
    }
    const size_t o_counts = c0.take(sizeof(int) * cnt_ints);
    auto ws_bytes = [&](const Job &j) {
        const size_t M = sp[j.design].items.size(), N = prep[j.design].n_nodes;
        return 8 * N + 4 * N + 2 * 8 * M + 7 * 4 * M + 2 * 4 * (M + 1) + 4 * (16 * (size_t)nt + 1) + 64;
    };
    for (size_t k = 0; k < jobs.size(); ++k)
        o_ws[k] = c0.take(ws_bytes(jobs[k]));
    const size_t o_tasks = c0.take(sizeof(PsTask) * jobs.size());
    char *b0 = dev.buffer(0, c0.off);
    std::vector<PsDesign> desc(prep.size());
    for (size_t d = 0; d < prep.size(); ++d) {
        desc[d] = PsDesign{dev_desc[d], nullptr, nullptr, 0};
        if (!used[d])
            continue;
        dev.up(b0 + o_items[d], sp[d].items.data(), sizeof(PsItem) * sp[d].items.size());
        dev.up(b0 + o_oitem[d], sp[d].out_item.data(), sizeof(int) * sp[d].out_item.size());
        desc[d].items = (const PsItem *)(b0 + o_items[d]);
        desc[d].out_item = (const int *)(b0 + o_oitem[d]);
        desc[d].n_items = (int)sp[d].items.size();
    }
    dev.up(b0 + o_desc, desc.data(), sizeof(PsDesign) * desc.size());
    std::vector<PsTask> tasks(jobs.size());
    for (size_t k = 0; k < jobs.size(); ++k) {
        const Job &j = jobs[k];
        const size_t M = sp[j.design].items.size(), N = prep[j.design].n_nodes;
        PsTask &T = tasks[k];
        T = PsTask{};
        T.pp.design = j.design;
        T.pp.cutoff = j.cutoff;
        T.pp.in_lat = dev_lat && !j.zero ? dev_lat + lat_off[j.design] : nullptr;
        char *w = b0 + o_ws[k];
        T.pp.lat = (double *)w, w += 8 * N;
        T.key = (unsigned long long *)w, w += 8 * M;
        T.key2 = (unsigned long long *)w, w += 8 * M;
        T.cost = (float *)w, w += 4 * N;
        int *iw = (int *)w;
        T.val = iw, iw += M;
        T.val2 = iw, iw += M;
        T.rank = iw, iw += M;
        T.stg = iw, iw += M;
        T.last = iw, iw += M;
        T.keep = iw, iw += M;
        T.inpos = iw, iw += M;
        T.flag = iw, iw += M + 1;
        T.coff = iw, iw += M + 1;
        T.cnt = iw;
        int *cw = (int *)(b0 + o_counts) + o_cnt[k];
        T.count = (PsCount *)cw;
        T.nrow = cw + 6;
        T.nout = cw + 6 + j.n_st;
        T.n_st = j.n_st;
    }
    dev.up(b0 + o_tasks, tasks.data(), sizeof(PsTask) * tasks.size());
    dev.count((const PsDesign *)(b0 + o_desc), (const PsTask *)(b0 + o_tasks), (int)jobs.size());
    ++out.launches;
    std::vector<int> counts(cnt_ints);
    dev.down(counts.data(), b0 + o_counts, sizeof(int) * cnt_ints);
    std::vector<char> failed(n_tasks, 0);
    for (size_t k = 0; k < jobs.size(); ++k) {
        const PsCount &q = *(const PsCount *)&counts[o_cnt[k]];
        if (q.status == PS_INTERNAL || q.status == PS_NOT_OK)
            throw std::runtime_error("pipeline_split: task " + std::to_string(jobs[k].task) + " does not replay as it was priced");
        if (q.status == PS_KEY_ERROR)
            failed[jobs[k].task] = 1;
    }
    // write pass: the jobs whose split is kept
    Carver c1, c2;
    std::vector<size_t> wk;
    std::vector<size_t> o_w1;
    for (size_t k = 0; k < jobs.size(); ++k) {
        const Job &j = jobs[k];
        PsSplit &S = out.tasks[j.task];
        if (!j.write)
            continue;
        if (failed[j.task]) {
            S.status = PS_KEY_ERROR;
            continue;
        }
        const PsCount &q = *(const PsCount *)&counts[o_cnt[k]];
        const size_t M = sp[j.design].items.size(), C = (size_t)q.n_copies, R = (size_t)q.n_kept + C;
        S.status = PS_SPLIT;
        S.n_st = q.n_st;
        S.n_rows = (int64_t)R;
        S.n_outs = (int64_t)(C + prep[j.design].n_out);
        S.meta.resize(3 * (size_t)q.n_st);
        int64_t n_in = prep[j.design].n_in;
        for (int s = 0; s < q.n_st; ++s) {
            S.meta[3 * s] = n_in;
            S.meta[3 * s + 1] = n_in = counts[o_cnt[k] + 6 + q.n_st + s];
            S.meta[3 * s + 2] = counts[o_cnt[k] + 6 + s];
        }
        S.o_ops_i = c2.off, c2.off += 8 * 4 * R;
        S.o_ops_f = c2.off, c2.off += 8 * 5 * R;
        S.o_outs = c2.off, c2.off += 8 * (size_t)S.n_outs;
        wk.push_back(k);
        o_w1.push_back(c1.take(4 * (3 * C + M + (R + 1) + (q.n_st + 1) + 2 * (M + C)) + 2 * 8 * (M + C) + 64));
    }
    if (wk.empty())
        return out;
    const size_t o_wtasks = c1.take(sizeof(PsTask) * wk.size());
    char *b1 = dev.buffer(1, c1.off), *b2 = dev.buffer(2, c2.off);
    std::vector<PsTask> wtasks;
    for (size_t q = 0; q < wk.size(); ++q) {
        const Job &j = jobs[wk[q]];
        const PsSplit &S = out.tasks[j.task];
        const PsCount &cq = *(const PsCount *)&counts[o_cnt[wk[q]]];
        const size_t M = sp[j.design].items.size(), R = (size_t)S.n_rows, C = (size_t)cq.n_copies;
        PsTask T = tasks[wk[q]];
        char *w = b1 + o_w1[q];
        T.rkey = (unsigned long long *)w, w += 8 * (M + C);
        T.rkey2 = (unsigned long long *)w, w += 8 * (M + C);
        int *iw = (int *)w;
        T.rval = iw, iw += M + C;
        T.rval2 = iw, iw += M + C;
        T.ev = iw, iw += C;
        T.cown = iw, iw += C;
        T.cpos = iw, iw += C;
        T.ownpos = iw, iw += M;
        T.cscan = iw, iw += R + 1;
        T.start = iw;
        T.ops_i = (int64_t *)(b2 + S.o_ops_i);
        T.ops_f = (double *)(b2 + S.o_ops_f);
        T.outs = (int64_t *)(b2 + S.o_outs);
        wtasks.push_back(T);
    }
    dev.up(b1 + o_wtasks, wtasks.data(), sizeof(PsTask) * wtasks.size());
    dev.write((const PsDesign *)(b0 + o_desc), (const PsTask *)(b1 + o_wtasks), (int)wtasks.size());
    ++out.launches;
    out.tables.resize(c2.off);
    dev.down(out.tables.data(), b2, c2.off);
    return out;
}

} // namespace da
