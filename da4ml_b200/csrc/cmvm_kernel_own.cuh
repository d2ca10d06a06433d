// cmvm_kernel_own.cuh -- the persistent solve kernel (owner-partitioned formulation, solve_owned.cuh): per greedy step ONE
// group exchange (the argmax), no cross-CTA counters and no L2 atomics.  The per-CTA context lives in shared memory
// (nothing of it is passed around by value).
#pragma once
#include "cmvm_kernels.cuh"
#include "solve_owned.cuh"
#ifdef DA_RECOUNT_PROF
#include <cstdio>
#endif

namespace da {

// shared-memory plan of one CTA of the owner-partitioned kernel (host and device agree through this function)
struct OwnPlan {
    OwnLayout lay;
    size_t bytes;
};
__host__ __device__ inline OwnPlan own_plan(int nchunk_cap, int n_out_max, int e_cap_max, int lcap, int hlog, int narrow) {
    OwnPlan P;
    size_t o = (page_cache_bytes(nchunk_cap) + 15) & ~size_t(15); // the page caches (carved in solve_own_kernel_body)
    auto take = [&](size_t bytes) {
        const size_t at = o;
        o += (bytes + 15) & ~size_t(15);
        return (uint32_t)at;
    };
    const int words = (n_out_max + 31) / 32;
    for (int r = 0; r < 3; ++r)
        P.lay.D[r] = take(sizeof(uint2) * (size_t)n_out_max);
    for (int r = 0; r < 3; ++r)
        P.lay.B[r] = take(sizeof(uint32_t) * (size_t)words);
    P.lay.pre = take(sizeof(uint32_t) * (size_t)words);
    P.lay.ver = take(sizeof(uint32_t) * (size_t)((e_cap_max + 31) / 32));
    P.lay.col_len = take(sizeof(int) * (size_t)n_out_max);
    P.lay.tcol = take(sizeof(uint16_t) * (size_t)n_out_max);
    P.lay.tpre = take(sizeof(int) * ((size_t)n_out_max + 1));
    P.lay.hkey = take(sizeof(uint32_t) << hlog);
    P.lay.hval = take(sizeof(uint32_t) << hlog);
    P.lay.hins = take(sizeof(uint16_t) << hlog);
    P.lay.lists = take((narrow ? 6 : 12) * (size_t)n_out_max * (size_t)lcap); // (lcap is even: the 32-bit plane arrays stay aligned)
    P.lay.narrow = narrow;
    P.lay.lcap = lcap;
    P.lay.hlog = hlog;
    P.lay.words = words;
    P.bytes = o;
    return P;
}

__device__ void solve_problem_own(const ProblemDesc &p, const Ctx &cx, const OwnCtx &ox) {
    const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, wid = tid >> 5, nw = nt >> 5;
    const int n_in = p.n_in, n_out = p.n_out, nbits = p.nbits, G = cx.cfg.G;
    const uint32_t thresh = method_threshold(p.method);
    BlockCtx &b = *cx.b;
    OwnBlock &ob = *ox.ob;

    if (tid == 0) {
        b.seg_len = 0;
        b.tb_mask = p.tb_mask;
        {
            // hot logs for the first expressions this CTA owns: its inputs and the earliest new expressions, the dense
            // rows that are rewritten again and again (not when the pool is too small to give each a few pages)
            const int n_own = (p.e_cap - cx.rank + G - 1) / G, H = min(n_own, DA_HOT_MAX);
            b.pages = min(cx.ws.fseg_cap >> cx.cfg.chunk_log, cx.cfg.nchunk_cap - 2);
            b.hot_top = b.pages;
            b.cap0 = b.pages << cx.cfg.chunk_log;
            b.n_used = 0;
            b.n_free = 0;
            b.hot_n = H > 0 && b.pages >= 8 * H ? H : 0;
            b.hot_room = 6 * (2 * nbits - 1); // 3 rewritten rows x shifts x signs
            for (int k = 0; k < DA_HOT_MAX; ++k)
                b.hot_len[k] = b.hot_snap[k] = b.hot_np[k] = 0;
        }
        b.n_new = 0;
        b.live_old = 0;
        b.n_dirty = 0;
        b.status = ST_OK;
        b.list_max = 0;
        b.r_count = 0ull;
        b.rescanned = 0ull;
        b.r_step = 0;
        b.rescan_step = 0;
        b.chosen = Best{0u, 0u, 0u};
        for (int k = 0; k < 8; ++k) {
            b.phase[k] = 0;
            b.peak[k] = 0;
            b.nslow[k] = 0;
        }
        b.phase[8] = 0;
        b.poll_iters = 0;
        ob.pool_used = 0;
        ob.helped = 0;
        ob.helped_ovf = 0;
        ob.pass_bits = 0;
        ob.n_ins = 0;
        ob.overflow = 0;
#ifdef DA_RECOUNT_PROF
        for (int k = 0; k < 4; ++k)
            ob.xphase[k] = 0;
#endif
    }
    for (int c = tid; c < cx.cfg.nchunk_cap; c += nt) {
        cx.cb_score[c] = 0u;
        cx.cb_khi[c] = 0u;
        cx.cb_klo[c] = 0u;
        cx.cb_dirty[c] = 0;
    }
    {
        DA_DYN_SHARED(da_smem);
        uint32_t *hkey = DA_SM(uint32_t, ox.lay.hkey), *hval = DA_SM(uint32_t, ox.lay.hval);
        for (int k = tid; k < (1 << ox.lay.hlog); k += nt) {
            hkey[k] = 0u;
            hval[k] = 0u;
        }
    }
    for (int i = cx.rank * nt + tid; i < p.e_cap; i += G * nt)
        cx.ws.mod_step[i] = 0u;
    group_sync(cx); // every CTA's share of the stamps is zero before anybody judges an entry by them
    own_init(p, cx, ox);
    // ---- input ops (state_opr.cc:146-149)
    for (int i = cx.rank * nt + tid; i < n_in; i += G * nt) {
        p.op_misc[i] = make_int4(i, -1, -1, 0);
        p.op_q[i] = make_float4(p.qint[3 * i], p.qint[3 * i + 1], p.qint[3 * i + 2], p.lat[i]);
        p.op_cost[i] = 0.0f;
    }

    Best best{0u, 0u, 0u};
    unsigned long long r0 = 0;
    if (p.method != M_DUMMY)
        r0 = initial_histogram(p, cx, thresh, best);
    if (r0)
        atomicAdd(&b.r_count, r0);
    __syncthreads();
    if (tid == 0) {
        atomicAdd((unsigned long long *)&p.result_meta[META_R0], b.r_count);
        b.r_count = 0ull; // from here on: the digit pairs of the greedy steps
        b.seg_len = min(b.seg_len, b.cap0);
        b.n_new = 0;
    }
    __syncthreads();
    if (wid == 0)
        hot_grow(cx); // the hot logs' first pages
    __syncthreads();
    // Two teams of warps work side by side in a greedy step: the first warps substitute, update and recount (team C,
    // barrier 1), the last quarter brings the argmax caches up to date for the rewritten expressions (team R, barrier 2)
    // -- which chunks a substitution invalidates varies wildly from CTA to CTA and step to step, and the group waits for
    // its slowest CTA.  (A CTA of a single warp does both one after the other.)  The last warp (of team R) publishes and
    // collects the exchanges; in a step its lane 0 executes the exchange's release fence while team C still counts:
    // team C signals barrier 3 once the writes the next step reads (own_update) are done.  Team R then counts pairs of
    // the recount's first pass next to team C (barriers 5 and 6, own_recount_help), and the teams join.
    const int rw = nw >= 4 ? nw / 4 : (nw >= 2 ? 1 : 0);
    const bool split = rw > 0;
    const int nt_c = nt - 32 * rw;
    const bool in_c = tid < nt_c;
    const Team tm_c = split ? Team{tid, nt_c, 1} : team_all(), tm_r = Team{tid - nt_c, 32 * rw, 2};
    const int pw = nw - 1, pub = nt - 32; // the exchange's warp and publishing thread

    int seg_cur = b.seg_len; // entries of this CTA's segment (every thread keeps a copy: team R must not read the live counter)
    refresh_chunks(cx, team_all(), seg_cur, 0u, 0u, false, true, thresh);
    publish_best(cx, Best{0u, 0u, 0u}, pw, false); // the exchange also orders the cells / input ops written above
    if (tid == pub) { // (it has published; nobody touches these before the barrier inside the collect)
        b.live_old = 0;
        b.n_new = 0;
    }
    int f_live = collect_best(cx, pw);
    const int f0 = f_live;
    int f_max = f_live;

    // ---- greedy loop (cmvm_core.cc:36-70)
    int t = 0;
    unsigned long long sum_f = 0;
    int status = b.scratch_i[1];
    if (tid == 0)
        b.t_start = clock64();
    while (status == ST_OK) {
        const Best ch = b.chosen;
        if (ch.score == 0u || p.method == M_DUMMY)
            break;
        if (n_in + t >= p.e_cap) {
            status = ST_EXPR_OVERFLOW;
            break;
        }
        const uint64_t key = ((uint64_t)ch.khi << 32) | ch.klo; // (collect_best has undone the tie-break mask)
        const uint32_t c0 = key_id0(key), c1 = key_id1(key);
        const int shift = key_shift(key), sub = key_sub(key);
        const uint32_t newid = (uint32_t)(n_in + t);
        const uint32_t stamp = (uint32_t)(t + 1);
        sum_f += (unsigned long long)f_live;
        f_max = max(f_max, f_live);
        if (tid == nt_c - 1) {
            // pair_to_op (state_opr.cc:211-225): every CTA needs the new record for the entries it emits in this step;
            // CTA 0 also publishes it (with the rewrite stamps) for the later steps
            QInt q0, q1;
            float l0, l1;
            load_op(p, c0, q0, l0);
            load_op(p, c1, q1, l1);
            float dlat, cost;
            cost_add(q0, q1, shift, sub != 0, p.adder_size, p.carry_size, dlat, cost);
            const QInt q = qint_add(q0, q1, shift, false, sub != 0);
            const float lat = fadd(fmaxf_std(l0, l1), dlat);
            int r = 0;
            ob.mid[r] = c0, ob.mq[r] = q0, ob.ml[r] = l0, ++r;
            if (c1 != c0)
                ob.mid[r] = c1, ob.mq[r] = q1, ob.ml[r] = l1, ++r;
            ob.mid[r] = newid, ob.mq[r] = q, ob.ml[r] = lat, ++r;
            ob.n_mods = r;
            if (cx.rank == 0) {
                p.op_misc[newid] = make_int4((int)c0, (int)c1, sub, shift);
                p.op_q[newid] = make_float4(q.min, q.max, q.step, lat);
                p.op_cost[newid] = cost;
                st_racy(&cx.ws.mod_step[c0], stamp);
                st_racy(&cx.ws.mod_step[c1], stamp);
                st_racy(&cx.ws.mod_step[newid], stamp);
                if (p.trace && t < p.trace_cap) {
                    int *tr = p.trace + 5 * (size_t)t;
                    tr[0] = (int)c0;
                    tr[1] = (int)c1;
                    tr[2] = shift;
                    tr[3] = sub;
                    tr[4] = f_live;
                }
            }
        }
        if (tid == 0)
            b.t_last = clock64();
        const bool compacting = b.scratch_i[3] != 0; // agreed by the whole group in the last exchange
        if (compacting) {
            compact_segment(cx, c0, c1, true, thresh, cx.rank == 0 ? &p.result_meta[META_COMPACTIONS] : nullptr);
            seg_cur = b.seg_len;
            __syncthreads(); // (every thread has its copy before team C appends)
        }
        const int seg0 = seg_cur; // what the argmax caches have to cover; this step's entries are appended behind it
        {
            // a hot expression of this CTA is rewritten: every entry of its log dies with it (uniform over the CTA)
            const bool k0 = (int)(c0 % (uint32_t)G) == cx.rank && (int)(c0 / (uint32_t)G) < b.hot_n;
            const bool k1 = c1 != c0 && (int)(c1 % (uint32_t)G) == cx.rank && (int)(c1 / (uint32_t)G) < b.hot_n;
            if (k0 || k1) {
                const int ks[2] = {(int)(c0 / (uint32_t)G), (int)(c1 / (uint32_t)G)};
                hot_free(cx, ks, (k0 ? 1u : 0u) | (k1 ? 2u : 0u));
                __syncthreads();
            }
        }
        best = Best{0u, 0u, 0u};
        if (in_c) {
            // A. substitution in the columns of c0 / c1 (redundantly on every CTA), B. the owners update their cells and lists,
            // C. the recount appends this step's entries
            own_substitute(p, cx, ox, tm_c, c0, c1, shift, sub);
            DA_LAP(0)
            own_update(p, cx, ox, tm_c, c0, c1, newid);
            if (split)
                named_arrive(3, nt_c + 32); // the writes the exchange carries are done (see below)
            DA_LAP(3)
            if (!split && !compacting)
                refresh_chunks(cx, tm_c, seg0, c0, c1, true, cx.cfg.accounting != 0, thresh);
            own_recount(p, cx, ox, tm_c, newid, stamp, thresh, best, split);
            DA_LAP(1)
        }
        else {
            // the argmax caches: entries touching c0 / c1 die
            const long long r0c = clock64();
            if (!compacting)
                refresh_chunks(cx, tm_r, seg0, c0, c1, true, cx.cfg.accounting != 0, thresh);
            if (tid >= pub) {
                // the exchange's release, off the step's critical path: once team C has arrived at barrier 3, the
                // publishing thread's fence orders its writes (and CTA 0's op record, written by team C's last thread
                // before) before the slot stores of publish_best.  The entries the recount appends meanwhile are private
                // to the CTA and need no release.
                if (tid == pub)
                    b.phase[2] += clock64() - r0c; // (phase 2 = the refresh and the fence, not the wait for team C)
                team_sync(Team{tid - pub, nt_c + 32, 3});
                if (tid == pub) {
                    const long long f0 = clock64();
                    fence_acq_rel_gpu();
                    b.phase[2] += clock64() - f0;
                }
            }
            own_recount_help(p, cx, ox, pub);
        }
        __syncthreads();
        DA_LAP(4)
        // The thread bests already hold every entry appended in this step: the chunk caches of publish_best need not
        // cover them yet.
        seg_cur = min(b.seg_len, b.cap0); // (before publish_best's barrier, behind which warp 0 hands out pages)
        publish_best(cx, best, pw, split);
        own_clear_rows(p, ox, team_all()); // (the rows were last read before the join)
        {
            // While the exchange is in flight: the maxima of the entries each log received in this step (every warp but
            // the exchange's takes some logs; only a log whose new entries lie in one page that is not dirty anyway needs
            // it), then warp 0 folds them into the cached maxima of their pages and gives the hot logs their room for the
            // next step (nothing is appended before the next step's team C starts, two exchanges' barriers away).
            const int nm = nw > 1 ? nw - 1 : 1, cl = cx.cfg.chunk_log; // (the exchange's warp is the last one)
            if (wid < nm) {
                for (int r = wid; r <= b.hot_n; r += nm) {
                    const int l0 = r == 0 ? seg0 : b.hot_snap[r - 1];
                    const int l1 = r == 0 ? min(b.seg_len, b.cap0) : min(b.hot_len[r - 1], b.hot_np[r - 1] << cl);
                    if (l1 > l0 && (l0 >> cl) == ((l1 - 1) >> cl) && !cx.cb_dirty[log_pos(cx, r, l0) >> cl]) // (uniform over the warp)
                        merge_appended_scan(cx, r, l0, l1, thresh);
                }
                if (nm > 1)
                    team_sync(Team{tid, 32 * nm, 4});
                else
                    __syncwarp();
            }
            if (wid == 0) {
                const int seg1 = min(b.seg_len, b.cap0);
                for (int r = lane; r <= b.hot_n; r += 32) {
                    if (r == 0)
                        merge_appended_apply(cx, 0, seg0, seg1);
                    else {
                        const int k = r - 1, l1 = min(b.hot_len[k], b.hot_np[k] << cl);
                        merge_appended_apply(cx, r, b.hot_snap[k], l1);
                        b.hot_len[k] = l1; // the log's fill becomes the next step's snapshot
                        b.hot_snap[k] = l1;
                    }
                }
                __syncwarp();
                hot_grow(cx);
            }
        }
        if (tid == pub) { // (it has published; nobody touches these before the barrier inside the collect)
            b.live_old = 0;
            b.n_new = 0;
            b.r_count += (unsigned long long)b.r_step;
            b.r_step = 0;
            b.rescanned += (unsigned long long)b.rescan_step;
            b.rescan_step = 0;
        }
        DA_LAP(5)
        f_live = collect_best(cx, pw);
        DA_LAP(7)
        ++t;
        if (cx.rank == 0 && tid == 0 && t >= 250 && t % 250 == 0 && ((t / 250) & (t / 250 - 1)) == 0 && t / 250 <= 64) {
            long long *ms = &p.result_meta[META_MILESTONES + 10 * (31 - __clz(t / 250))]; // (diagnostic: where the time of a stage goes)
            for (int k = 0; k < 9; ++k)
                ms[k] = b.phase[k];
            ms[9] = clock64() - b.t_start;
#ifdef DA_RECOUNT_PROF
            printf("  recount parts after %d steps (cumulative ms at 1.9 GHz): setup %.2f counting %.2f harvest %.2f\n", t, ob.xphase[0] / 1.9e6, ob.xphase[1] / 1.9e6, ob.xphase[2] / 1.9e6);
#endif
        }
        if (b.scratch_i[1] != ST_OK) {
            status = b.scratch_i[1];
            break;
        }
    }

    // ---- to_solution: column lists from the owner lists, then one warp per column
    own_scatter_columns(p, cx, ox);
    finish_columns(p, cx, t);
    // ---- bookkeeping
    __syncthreads();
    if (tid == 0) {
        b.r_count += (unsigned long long)b.r_step;
        b.rescanned += (unsigned long long)b.rescan_step;
        atomicAdd((unsigned long long *)&p.result_meta[META_SUM_R], b.r_count);
        atomicAdd((unsigned long long *)&p.result_meta[META_RESCANNED], b.rescanned);
        atomicAdd((unsigned long long *)&p.result_meta[META_HELPED], (unsigned long long)ob.helped);
        atomicAdd((unsigned long long *)&p.result_meta[META_HELPED_OVF], (unsigned long long)ob.helped_ovf);
        atomicMax((long long *)&p.result_meta[META_LIST_MAX], (long long)b.list_max);
        for (int k = 0; k < 8; ++k)
            atomicMax((long long *)&p.result_meta[META_PHASEMAX + k], b.phase[k]); // the slowest CTA's total per phase
        if (b.status != ST_OK)
            atomicMax((int *)&p.result_meta[META_STATUS], b.status);
    }
    if (cx.rank == 0 && tid == 0) {
        long long tree = 0, dfin = 0;
        for (int o = 0; o < n_out; ++o) {
            const int k = __ldcg(&cx.ws.col_k[o]);
            tree += k > 1 ? k - 1 : 0;
            dfin += k;
        }
        const long long n_ops = (long long)n_in + t + tree;
        p.result_meta[META_N_OPS] = n_ops;
        p.result_meta[META_T] = t;
        p.result_meta[META_SUM_F] = (long long)sum_f;
        p.result_meta[META_F0] = f0;
        p.result_meta[META_D_FINAL] = dfin;
        p.result_meta[META_F_MAX] = f_max;
        for (int k = 0; k < 8; ++k)
            p.result_meta[META_PHASE0 + k] = b.phase[k];
        p.result_meta[15] = b.poll_iters;
        if (status != ST_OK)
            atomicMax((int *)&p.result_meta[META_STATUS], status);
        if (n_ops > p.ops_cap)
            atomicMax((int *)&p.result_meta[META_STATUS], (int)ST_OPS_OVERFLOW);
    }
    group_sync(cx); // the workspace may be reused by the next problem of this group
    (void)lane;
    (void)wid;
    (void)nw;
    (void)nbits;
}

// grid = n_groups * G CTAs; group i solves problems i, i + n_groups, ...
__device__ __forceinline__ void solve_own_kernel_body(const ProblemDesc *probs, int n_probs, const GroupWs *wss, const OwnWs *ows, const LaunchCfg &cfg, int n_out_max, int e_cap_max, int lcap, int hlog, int narrow) {
    DA_DYN_SHARED(smem);
    DA_SHARED_VAR(BlockCtx, bctx);
    DA_SHARED_VAR(OwnBlock, oblk);
    DA_SHARED_VAR(Ctx, cxs);
    DA_SHARED_VAR(OwnCtx, oxs);
    if (threadIdx.x == 0) {
        Ctx &cx = cxs;
        cx.cfg = cfg;
        cx.rank = blockIdx.x % cfg.G;
        const int group = blockIdx.x / cfg.G;
        cx.ws = wss[group];
        cx.seg = cx.ws.fseg + (size_t)cx.rank * cx.ws.fseg_cap;
        cx.b = &bctx;
        unsigned char *sp = smem; // (page_cache_bytes)
        const int n = cfg.nchunk_cap;
        cx.cb_score = (uint32_t *)sp;
        sp += sizeof(uint32_t) * n;
        cx.cb_khi = (uint32_t *)sp;
        sp += sizeof(uint32_t) * n;
        cx.cb_klo = (uint32_t *)sp;
        sp += sizeof(uint32_t) * n;
        uint16_t *h = (uint16_t *)sp;
        cx.dirty_list = h, h += n;
        cx.pg_owner = h, h += n;
        cx.pg_used = h, h += n;
        cx.pg_slot = h, h += n;
        cx.pg_free = h, h += n;
        cx.hot_pg = h, h += DA_HOT_MAX * DA_HOT_PAGES;
        cx.cb_dirty = (unsigned char *)h;
        OwnCtx &ox = oxs;
        ox.ws = ows[group];
        ox.lay = own_plan(cfg.nchunk_cap, n_out_max, e_cap_max, lcap, hlog, narrow).lay;
        ox.ob = &oblk;
        ox.ovf = ox.ws.ovf + (size_t)cx.rank * (size_t)n_out_max * 3 * (size_t)ox.ws.ovf_cap;
        bctx.bar_target = 0u; // the host zeroes the arrive counter and the exchange slots before every launch
        bctx.epoch = 0u;
    }
    __syncthreads();
    // The problem's descriptor is read all through a greedy step, and every acquire of the exchange or of the group
    // barrier invalidates L1: from global memory each field would be an L2 round trip again (an op-record lookup chases
    // two of them before its own load).  So the CTA works from a copy in shared memory.
    DA_SHARED_VAR(ProblemDesc, pds);
    const int group = blockIdx.x / cfg.G, n_groups = gridDim.x / cfg.G;
    for (int pi = group; pi < n_probs; pi += n_groups) {
        if (threadIdx.x == 0)
            pds = probs[pi]; // (the previous problem ended with a group barrier: nobody reads the old copy any more)
        __syncthreads();
        solve_problem_own(pds, cxs, oxs);
    }
}
__global__ void __launch_bounds__(512, 1) cmvm_solve_kernel(const ProblemDesc *probs, int n_probs, const GroupWs *wss, const OwnWs *ows, LaunchCfg cfg, int n_out_max, int e_cap_max, int lcap, int hlog, int narrow) {
    solve_own_kernel_body(probs, n_probs, wss, ows, cfg, n_out_max, e_cap_max, lcap, hlog, narrow);
}

} // namespace da
