// solve_histogram.cuh -- the lazy pair histogram: liveness by rewrite stamps, chunk-cached argmax, in-place compaction,
// and the two group exchanges of a greedy step (FreqMap types.hh:39-100, selectors indexers.cc:6-90).
#pragma once
#include "solve_common.cuh"

namespace da {

// ---- lazy histogram -------------------------------------------------------------------------------
// (`m0` = key_id0 of the tie-break mask: the entry's key is stored masked)
__device__ __forceinline__ bool entry_live(const FEnt &e, const uint32_t *mod, uint32_t c0, uint32_t c1, bool purge, uint32_t m0) {
    if (e.y == DA_DEAD)
        return false;
    const uint64_t key = ((uint64_t)e.w << 32) | e.z;
    const uint32_t a = key_id0(key) ^ m0, c = key_id1(key);
    if (purge && (a == c0 || a == c1 || c == c0 || c == c1))
        return false;
    const uint32_t ma = __ldcg(&mod[a]), mc = __ldcg(&mod[c]);
    return e.y >= ma && e.y >= mc;
}

// One warp re-reads entries [lo, hi) of this CTA's segment: buries the entries found dead, returns the number of live
// ones and (in `out`) their maximum, both warp-uniform.  Loads are issued in batches (8 entries per lane, then their
// 16 stamp lookups) so the round trips overlap.
__device__ __forceinline__ int rescan_range(const Ctx &cx, int lo, int hi, uint32_t c0, uint32_t c1, bool purge, uint32_t thresh, Best &out) {
    const int lane = threadIdx.x & 31;
    const uint32_t *mod = cx.ws.mod_step;
    const uint32_t m0 = key_id0(cx.b->tb_mask);
    Best best{0u, 0u, 0u};
    int live = 0;
    constexpr int U = 8;
    for (int i0 = lo + lane; i0 < hi; i0 += 32 * U) {
        FEnt e[U];
        uint32_t ma[U], mc[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const int i = i0 + 32 * u;
            e[u] = make_uint4(0u, DA_DEAD, 0u, 0u);
            if (i < hi)
                e[u] = __ldcg(&cx.seg[i]);
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            ma[u] = mc[u] = 0u;
            if (e[u].y != DA_DEAD) {
                const uint64_t key = ((uint64_t)e[u].w << 32) | e[u].z;
                ma[u] = __ldcg(&mod[key_id0(key) ^ m0]);
                mc[u] = __ldcg(&mod[key_id1(key)]);
            }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            if (e[u].y == DA_DEAD)
                continue;
            const uint64_t key = ((uint64_t)e[u].w << 32) | e[u].z;
            const uint32_t a = key_id0(key) ^ m0, c = key_id1(key);
            const bool ok = !(purge && (a == c0 || a == c1 || c == c0 || c == c1)) && e[u].y >= ma[u] && e[u].y >= mc[u];
            if (ok) {
                ++live;
                if (e[u].x >= thresh) {
                    Best cand{e[u].x, e[u].w, e[u].z};
                    if (best_gt(cand, best))
                        best = cand;
                }
            }
            else
                cx.seg[i0 + 32 * u].y = DA_DEAD;
        }
    }
    out = warp_best(best);
#pragma unroll
    for (int off = 16; off > 0; off >>= 1)
        live += __shfl_xor_sync(0xffffffffu, live, off);
    return live;
}

// Bring every page cache up to date for the substitution (c0, c1): pages whose cached winner touches c0/c1, pages
// that received appends, or all pages in use (accounting / after compaction).  Block-wide.  A page is re-read by one
// warp, or -- when few large pages are dirty -- by several warps that each take a 256-entry-aligned part of it.
#ifndef DA_SPLIT_RESCAN
#define DA_SPLIT_RESCAN 1
#endif
// `tm`: the warps doing it; `seg_len`: the entries to cover (what other warps append meanwhile lies beyond).
__device__ void refresh_chunks(const Ctx &cx, const Team &tm, int seg_len, uint32_t c0, uint32_t c1, bool purge, bool all, uint32_t thresh) {
    const int tid = tm.tid, nt = tm.nt, lane = tid & 31, wid = tid >> 5, nw = nt >> 5;
    BlockCtx &b = *cx.b;
    const int ch_log = cx.cfg.chunk_log, ch = 1 << ch_log;
    const int nc = common_pages(cx, seg_len), npages = pages_in_use(cx, nc);
    for (int i = tid; i < npages; i += nt) {
        const int c = page_at(cx, i, nc);
        int lo_c, hi_c;
        page_span(cx, c, seg_len, lo_c, hi_c);
        if (hi_c <= lo_c)
            continue; // (nothing there: its cache is empty)
        bool d = all || cx.cb_dirty[c];
        if (!d && purge && cx.cb_score[c] != 0u) {
            const uint64_t key = ((uint64_t)cx.cb_khi[c] << 32) | cx.cb_klo[c];
            const uint32_t a = key_id0(key ^ b.tb_mask), e = key_id1(key);
            d = (a == c0 || a == c1 || e == c0 || e == c1);
        }
        if (d)
            cx.dirty_list[smem_add(&b.n_dirty, 1)] = c;
    }
    team_sync(tm);
    const int nd = b.n_dirty;
    int nparts = 1; // warps per dirty chunk (power of two, parts of at least 256 entries)
    if (DA_SPLIT_RESCAN && nd > 0)
        while (2 * nparts * nd <= nw && (ch >> 8) >= 2 * nparts)
            nparts *= 2;
    int live = 0;
    if (nparts > 1) { // (uniform over the CTA)
        if (wid < nd * nparts) {
            const int i = wid / nparts, part = wid - i * nparts;
            int base, end;
            page_span(cx, cx.dirty_list[i], seg_len, base, end);
            const int plen = ch / nparts;
            const int lo = base + part * plen;
            Best pb;
            const int pl = rescan_range(cx, lo, min(lo + plen, end), c0, c1, purge, thresh, pb);
            live += pl;
            if (lane == 0)
                b.warp_best[wid] = pb;
        }
        team_sync(tm);
        if (tid < nd) {
            Best v = b.warp_best[tid * nparts];
            for (int q = 1; q < nparts; ++q)
                if (best_gt(b.warp_best[tid * nparts + q], v))
                    v = b.warp_best[tid * nparts + q];
            const int chunk = cx.dirty_list[tid];
            cx.cb_score[chunk] = v.score;
            cx.cb_khi[chunk] = v.khi;
            cx.cb_klo[chunk] = v.klo;
            cx.cb_dirty[chunk] = 0;
        }
        if (tid == 0)
            atomicAdd(&b.rescan_step, nd << ch_log);
    }
    else {
        for (int i = wid; i < nd; i += nw) {
            const int chunk = cx.dirty_list[i];
            int base, end;
            page_span(cx, chunk, seg_len, base, end);
            Best v;
            live += rescan_range(cx, base, end, c0, c1, purge, thresh, v);
            if (lane == 0) {
                cx.cb_score[chunk] = v.score;
                cx.cb_khi[chunk] = v.khi;
                cx.cb_klo[chunk] = v.klo;
                cx.cb_dirty[chunk] = 0;
            }
        }
        if (lane == 0 && nd > wid) {
            const int mine = (nd - wid + nw - 1) / nw;
            atomicAdd(&b.rescan_step, mine << ch_log);
        }
    }
    if (lane == 0 && all && live)
        atomicAdd(&b.live_old, live);
    team_sync(tm);
    if (tid == 0)
        b.n_dirty = 0;
}

// Entries [l0, l1) of log r (0: the common log, k + 1: hot log k) were appended in this step: their maximum is folded
// into the cached maximum of their page instead of re-reading the whole page next step (they are live by construction).
// Part 1 (one warp, any time after the entries were written): the maximum -> pend[r]; part 2 (one thread, when nobody
// else touches the caches): pend[r] -> the page's cache.  Entries that straddle a page boundary, or land in a page that
// is dirty anyway, leave their pages dirty instead.
__device__ __forceinline__ void merge_appended_scan(const Ctx &cx, int r, int l0, int l1, uint32_t thresh) {
    const int lane = threadIdx.x & 31;
    Best best{0u, 0u, 0u};
    for (int v = l0 + lane; v < l1; v += 32) {
        const FEnt e = cx.seg[log_pos(cx, r, v)];
        if (e.x >= thresh) {
            const Best cand{e.x, e.w, e.z};
            if (best_gt(cand, best))
                best = cand;
        }
    }
    best = warp_best(best);
    if (lane == 0)
        cx.b->pend[r] = best;
}
__device__ __forceinline__ void merge_appended_apply(const Ctx &cx, int r, int l0, int l1) {
    if (l1 <= l0)
        return;
    const int cl = cx.cfg.chunk_log, ca = log_pos(cx, r, l0) >> cl;
    if ((l0 >> cl) != ((l1 - 1) >> cl) || cx.cb_dirty[ca]) {
        for (int v = l0 >> cl; v <= (l1 - 1) >> cl; ++v)
            cx.cb_dirty[log_pos(cx, r, v << cl) >> cl] = 1;
        return;
    }
    const Best best = cx.b->pend[r], cur{cx.cb_score[ca], cx.cb_khi[ca], cx.cb_klo[ca]};
    if (best_gt(best, cur)) {
        cx.cb_score[ca] = best.score;
        cx.cb_khi[ca] = best.khi;
        cx.cb_klo[ca] = best.klo;
    }
}

// Warp 0, between steps: give every hot log the room one step can fill (hot_room entries beyond its fill) -- pages from
// the free stack first, then from the top of the pool while the common log keeps at least twice its fill below.  A log
// that gets no page spills into the common log until it does.
__device__ void hot_grow(const Ctx &cx) {
    BlockCtx &b = *cx.b;
    const int lane = threadIdx.x & 31, cl = cx.cfg.chunk_log;
    const int lim = (2 * b.seg_len + (1 << cl) - 1) >> cl;
    for (int k0 = 0; k0 < b.hot_n; k0 += 32) {
        const int k = k0 + lane;
        int np = 0, need = 0;
        if (k < b.hot_n) {
            np = b.hot_np[k];
            while (np + need < DA_HOT_PAGES && ((np + need) << cl) < b.hot_len[k] + b.hot_room)
                ++need;
        }
        int incl = need;
#pragma unroll
        for (int off = 1; off < 32; off <<= 1) {
            const int u = __shfl_up_sync(0xffffffffu, incl, off);
            if (lane >= off)
                incl += u;
        }
        const int total = __shfl_sync(0xffffffffu, incl, 31);
        if (total == 0) // (warp-uniform)
            continue;
        const int n_free = b.n_free, top = b.hot_top, n_used = b.n_used;
        const int from_stack = min(total, n_free), from_top = min(total - from_stack, max(0, top - lim));
        for (int g = incl - need; g < incl && g < from_stack + from_top; ++g) {
            const int pg = g < from_stack ? cx.pg_free[n_free - 1 - g] : top - 1 - (g - from_stack);
            cx.pg_owner[pg] = (uint16_t)((k << 8) | np);
            cx.hot_pg[k * DA_HOT_PAGES + np] = (uint16_t)pg;
            cx.pg_used[n_used + g] = (uint16_t)pg;
            cx.pg_slot[pg] = (uint16_t)(n_used + g);
            ++np;
        }
        if (need)
            b.hot_np[k] = np;
        __syncwarp();
        if (lane == 0) {
            b.n_free = n_free - from_stack;
            b.hot_top = top - from_top;
            b.n_used = n_used + from_stack + from_top;
            b.cap0 = b.hot_top << cl;
        }
        __syncwarp();
    }
}

// Block-wide, at the start of a step (uniform over the CTA): the hot logs of `mask` (bit w: log k[w]) were rewritten --
// every entry of theirs is dead.  Each keeps its first page, emptied, and returns the others to the free stack.
__device__ void hot_free(const Ctx &cx, const int k[2], unsigned mask) {
    BlockCtx &b = *cx.b;
    const int tid = threadIdx.x, nt = blockDim.x;
    for (int w = 0; w < 2; ++w) {
        if (!((mask >> w) & 1u))
            continue;
        const int np = b.hot_np[k[w]];
        for (int j = tid; j < np; j += nt) {
            const int pg = cx.hot_pg[k[w] * DA_HOT_PAGES + j];
            cx.cb_score[pg] = 0u;
            cx.cb_khi[pg] = 0u;
            cx.cb_klo[pg] = 0u;
            cx.cb_dirty[pg] = 0;
        }
    }
    __syncthreads();
    if (tid == 0)
        for (int w = 0; w < 2; ++w) {
            if (!((mask >> w) & 1u))
                continue;
            const int np = b.hot_np[k[w]];
            for (int j = 1; j < np; ++j) {
                const int pg = cx.hot_pg[k[w] * DA_HOT_PAGES + j];
                cx.pg_free[b.n_free++] = (uint16_t)pg;
                const int s = cx.pg_slot[pg], m = cx.pg_used[--b.n_used]; // (swap-remove from the list in use)
                cx.pg_used[s] = (uint16_t)m;
                cx.pg_slot[m] = (uint16_t)s;
            }
            b.hot_np[k[w]] = min(np, 1);
            b.hot_len[k[w]] = b.hot_snap[k[w]] = 0;
        }
}

// In-place compaction of this CTA's common log (drops dead entries; order is irrelevant), then every page cache is
// rebuilt.  Tiles of 8 x blockDim entries: all reads of a tile complete before its survivors are written to
// positions that never pass the tile's end.
__device__ __noinline__ void compact_segment(const Ctx &cx, uint32_t c0, uint32_t c1, bool purge, uint32_t thresh, long long *compactions) {
    const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31;
    BlockCtx &b = *cx.b;
    const int len = b.seg_len;
    const uint32_t m0 = key_id0(b.tb_mask);
    constexpr int K = 8;
    if (tid == 0)
        b.cmp_out = 0;
    __syncthreads();
    for (int base = 0; base < len; base += K * nt) {
        FEnt e[K];
        bool live[K];
#pragma unroll
        for (int k = 0; k < K; ++k) {
            const int i = base + k * nt + tid;
            live[k] = false;
            if (i < len) {
                e[k] = __ldcg(&cx.seg[i]);
                live[k] = entry_live(e[k], cx.ws.mod_step, c0, c1, purge, m0);
            }
        }
        __syncthreads(); // every read of this tile is complete
#pragma unroll
        for (int k = 0; k < K; ++k) {
            const unsigned bal = __ballot_sync(0xffffffffu, live[k]);
            int wbase = 0;
            if (lane == 0 && bal)
                wbase = atomicAdd(&b.cmp_out, __popc(bal));
            wbase = __shfl_sync(0xffffffffu, wbase, 0);
            if (live[k])
                cx.seg[wbase + __popc(bal & ((1u << lane) - 1u))] = e[k];
        }
    }
    __syncthreads();
    if (tid == 0) {
        b.seg_len = b.cmp_out;
        b.live_old = 0;
        if (compactions)
            atomicAdd((unsigned long long *)compactions, 1ull);
    }
    // every cached maximum of the common log referred to the old positions: forget them all (the pages in use are
    // rebuilt below; the hot logs did not move)
    for (int c = tid; c < common_pages(cx, len); c += nt) {
        cx.cb_score[c] = 0u;
        cx.cb_khi[c] = 0u;
        cx.cb_klo[c] = 0u;
        cx.cb_dirty[c] = 0;
    }
    __syncthreads();
    refresh_chunks(cx, team_all(), b.seg_len, c0, c1, false, true, thresh);
    if (tid == 0 && !cx.cfg.accounting)
        b.live_old = 0;
    __syncthreads();
}

// Block-reduce (thread bests + page caches) and publish this CTA's candidate through the exchange: warp `pw` reduces, its
// lane 0 publishes (`fenced`: that thread has already executed the release fence, see xchg_publish).  The page caches
// are only read here, so the caller may update them as soon as this returns.
__device__ void publish_best(const Ctx &cx, Best best, int pw, bool fenced) {
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5, nw = blockDim.x >> 5;
    BlockCtx &b = *cx.b;
    const int nc = common_pages(cx, b.seg_len), npages = pages_in_use(cx, nc);
    // free pages run short: ask the whole group to compact together (read before the barrier, behind which warp 0 hands
    // out the next pages)
    const bool want = b.seg_len > b.cap0 - (b.cap0 >> 2);
    for (int i = tid; i < npages; i += blockDim.x) {
        const int c = page_at(cx, i, nc);
        Best cand{cx.cb_score[c], cx.cb_khi[c], cx.cb_klo[c]};
        if (best_gt(cand, best))
            best = cand;
    }
    best = warp_best(best);
    if (lane == 0)
        b.warp_best[wid] = best;
    __syncthreads();
    if (wid == pw) {
        Best v = lane < nw ? b.warp_best[lane] : Best{0u, 0u, 0u};
        v = warp_best(v);
        if (lane == 0) {
            const int live = cx.cfg.accounting ? b.live_old + b.n_new : 0;
            xchg_publish(cx, v, b.status, want, live, fenced);
        }
    }
}

// Gather every CTA's candidate -> chosen pair (identical on every CTA); returns |F| (accounting mode).  Warp `pw` (the
// publishing warp) polls all G slots at once -- lane i reads slot i, i + 32, ... until every word carries this
// exchange's tag --, reduces them in registers and hands the result to the CTA with one barrier.
__device__ int collect_best(const Ctx &cx, int pw) {
    const int tid = threadIdx.x, lane = tid & 31, G = cx.cfg.G;
    BlockCtx &b = *cx.b;
    if ((tid >> 5) == pw) {
        __syncwarp(); // the epoch (and in a group of one CTA the payload) were written by lane 0
        const unsigned epoch = b.epoch;
        const unsigned long long tag = xchg_tag(epoch);
        const bool acc = cx.cfg.accounting != 0;
        const unsigned long long *s = cx.ws.xchg + (size_t)(epoch & 1u) * 4 * G;
        const long long t0 = clock64();
        int iters = 0;
        Best v{0u, 0u, 0u};
        int live = 0, st = 0;
        for (int i = lane; i < G; i += 32) {
            unsigned long long w0, w1, w2;
            if (G > 1) {
                while (true) { // (w0 last: its acquire load is the one that synchronizes with the writer)
                    w1 = ld_relaxed_u64(s + G + i);
                    w2 = acc ? ld_relaxed_u64(s + 2 * G + i) : tag;
                    w0 = ld_acquire_u64(s + i);
                    if (xchg_current(w0, tag) && xchg_current(w1, tag) && xchg_current(w2, tag))
                        break;
                    ++iters;
                }
            }
            else
                w0 = b.xw[0], w1 = b.xw[1], w2 = b.xw[2];
            if ((w0 >> 50) & 1ULL)
                st |= 0x100; // somebody's segment is filling up
            const unsigned long long key = ((w0 & 0x3fffULL) << 50) | (w1 & DA_XCHG_LO);
            const Best c{(uint32_t)(w0 >> 14), (uint32_t)(key >> 32), (uint32_t)key};
            if (best_gt(c, v))
                v = c;
            if (acc)
                live += (int)(w2 & 0x0fffffffULL);
            st = max(st & 0xff, (int)((w0 >> 46) & 0xf)) | (st & 0x100);
        }
        __syncwarp();
        if (lane == 0) {
            b.phase[6] += clock64() - t0; // polling (lane 0's slots, then waiting for the rest of the warp)
            b.poll_iters += iters;
        }
        v = warp_best(v);
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            live += __shfl_xor_sync(0xffffffffu, live, off);
            const int o = __shfl_xor_sync(0xffffffffu, st, off);
            st = max(st & 0xff, o & 0xff) | ((st | o) & 0x100);
        }
        if (lane == 0) {
            b.chosen = Best{v.score, v.khi ^ (uint32_t)(b.tb_mask >> 32), v.klo ^ (uint32_t)b.tb_mask}; // (the key as pack_key formed it)
            b.scratch_i[0] = live;
            b.scratch_i[1] = st & 0xff;
            b.scratch_i[3] = (st >> 8) & 1;
        }
    }
    __syncthreads();
    return b.scratch_i[0];
}

// Initial pair histogram (state_opr.cc:115-144, types.hh:73-100): warp per (a <= c) pair block, lanes over relative
// shifts, sign planes streamed over the output columns.  Appends the entries with count >= 2 to this CTA's segment and
// returns this thread's digit pairs.
__device__ unsigned long long initial_histogram(const ProblemDesc &p, const Ctx &cx, uint32_t thresh, Best &best) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
    const int n_in = p.n_in, n_out = p.n_out, nbits = p.nbits, G = cx.cfg.G;
    unsigned long long r0 = 0;
    {
        // ---- initial pair histogram (state_opr.cc:115-144, types.hh:73-100): warp per (a<=c) pair block,
        //      lanes over relative shifts, sign planes streamed over the output columns
        const long long n_pairs = (long long)n_in * (n_in + 1) / 2;
        const int n_sh = 2 * nbits - 1;
        for (long long pi = (long long)cx.rank * nw + wid; pi < n_pairs; pi += (long long)G * nw) {
            long long a = (long long)(((2.0 * n_in + 1.0) - sqrt((2.0 * n_in + 1.0) * (2.0 * n_in + 1.0) - 8.0 * (double)pi)) * 0.5);
            while (a > 0 && a * (2LL * n_in - a + 1) / 2 > pi)
                --a;
            while ((a + 1) * (2LL * n_in - (a + 1) + 1) / 2 <= pi)
                ++a;
            const long long c = a + (pi - a * (2LL * n_in - a + 1) / 2);
            const uint2 *ra = p.masks0 + (size_t)a * n_out;
            const uint2 *rc = p.masks0 + (size_t)c * n_out;
            QInt qa, qc;
            float la, lc;
            load_op(p, (uint32_t)a, qa, la);
            load_op(p, (uint32_t)c, qc, lc);
            for (int s0 = 0; s0 < n_sh; s0 += 32) {
                const int si = s0 + lane;
                const int s = si - (nbits - 1);
                const bool active = si < n_sh && !(a == c && s >= 0);
                uint32_t same = 0, diff = 0;
                if (active) {
                    if (s >= 0) {
                        for (int o = 0; o < n_out; ++o) {
                            const uint2 x = ra[o], y = rc[o];
                            same += __popc(x.x & (y.x >> s)) + __popc(x.y & (y.y >> s));
                            diff += __popc(x.x & (y.y >> s)) + __popc(x.y & (y.x >> s));
                        }
                    }
                    else {
                        const int d = -s;
                        for (int o = 0; o < n_out; ++o) {
                            const uint2 x = ra[o], y = rc[o];
                            same += __popc((x.x >> d) & y.x) + __popc((x.y >> d) & y.y);
                            diff += __popc((x.x >> d) & y.y) + __popc((x.y >> d) & y.x);
                        }
                    }
                    r0 += same + diff;
                    if (same >= 2)
                        emit_entry(p, cx, (uint32_t)a, (uint32_t)c, s, 0, same, qa, la, qc, lc, 0u, thresh, best);
                    if (diff >= 2)
                        emit_entry(p, cx, (uint32_t)a, (uint32_t)c, s, 1, diff, qa, la, qc, lc, 0u, thresh, best);
                }
            }
        }
    }
    return r0;
}

} // namespace da
