// solve_common.cuh -- shared pieces of the persistent solve kernel: argmax candidate type, per-CTA context,
// column-list references, the group barrier / all-gather exchange, op-record access, histogram append.
#pragma once
#include "cmvm_num.cuh"
#include "cmvm_types.cuh"

namespace da {

// ------------------------------------------------------------------------------------------------
// small device helpers

__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned *p) {
#ifdef DA_CPU_SIM
    simt::poll_yield(); // a poll: let the other simulated threads run
    return __atomic_load_n(p, __ATOMIC_ACQUIRE);
#else
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
#endif
}

// atomic add on a counter of the CTA's shared-memory context.  The context is reached through a generic pointer, for
// which atomicAdd compiles to a generic-address ATOM; the explicit state space gives the native shared-memory atomic.
#ifndef DA_SMEM_ATOM
#define DA_SMEM_ATOM 1
#endif
__device__ __forceinline__ int smem_add(int *p, int v) {
#if DA_SMEM_ATOM && !defined(DA_CPU_SIM)
    int old;
    asm volatile("atom.shared.add.s32 %0, [%1], %2;" : "=r"(old) : "r"((unsigned)__cvta_generic_to_shared(p)), "r"(v) : "memory");
    return old;
#else
    return atomicAdd(p, v);
#endif
}

// A store that races with other threads BY DESIGN: either every racer writes the same value (dirty flags) or the readers
// accept the old and the new value alike (rewrite stamps of c0 / c1 while other CTAs purge them explicitly).  A plain
// store on the GPU; an atomic one under the CPU simulation so that its race checker reports only unintended races.
template <class T> __device__ __forceinline__ void st_racy(T *p, T v) {
#ifdef DA_CPU_SIM
    __atomic_store_n(p, v, __ATOMIC_RELAXED);
#else
    *p = v;
#endif
}

// the matching load: a value other threads may be changing right now (a fresh read every time it is executed)
template <class T> __device__ __forceinline__ T ld_racy(const T *p) {
#ifdef DA_CPU_SIM
    return __atomic_load_n(p, __ATOMIC_RELAXED);
#else
    return *(const volatile T *)p;
#endif
}

// A team of warps of the CTA that works through a phase together: the whole CTA (bar 0 = __syncthreads) or a part of it
// with its own hardware barrier (bar.sync id, threads), so that two independent phases can run side by side.
struct Team {
    int tid, nt; // this thread's index in the team, threads of the team (a multiple of 32)
    int bar;     // 0: the whole CTA
};
__device__ __forceinline__ Team team_all() { return Team{(int)threadIdx.x, (int)blockDim.x, 0}; }
__device__ __forceinline__ void team_sync(const Team &t) {
    if (t.bar == 0)
        __syncthreads();
    else {
#ifdef DA_CPU_SIM
        da_sim_named_barrier(t.bar, t.nt);
#else
        asm volatile("bar.sync %0, %1;" ::"r"(t.bar), "r"(t.nt) : "memory");
#endif
    }
}
// Producer side of named barrier `bar` for n threads: signals this thread's earlier memory accesses to the threads that
// wait on it with bar.sync, without waiting itself.  (The CPU simulation waits: it models only complete barriers.)
__device__ __forceinline__ void named_arrive(int bar, int n) {
#ifdef DA_CPU_SIM
    da_sim_named_barrier(bar, n);
#else
    asm volatile("bar.arrive %0, %1;" ::"r"(bar), "r"(n) : "memory");
#endif
}

struct Best {
    uint32_t score, khi, klo;
};
__device__ __forceinline__ bool best_gt(const Best &a, const Best &b) {
    if (a.score != b.score)
        return a.score > b.score;
    if (a.khi != b.khi)
        return a.khi > b.khi;
    return a.klo > b.klo;
}
__device__ __forceinline__ Best warp_best(Best b) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
        Best o;
        o.score = __shfl_xor_sync(0xffffffffu, b.score, off);
        o.khi = __shfl_xor_sync(0xffffffffu, b.khi, off);
        o.klo = __shfl_xor_sync(0xffffffffu, b.klo, off);
        if (best_gt(o, b))
            b = o;
    }
    return b;
}


// Block-level context kept in shared memory
struct BlockCtx {
    Best warp_best[32];
    int warp_sum[32];
    int warp_st[32];
    Best chosen;       // pair selected for the current step (score==0 -> none), key unmasked (see tb_mask below)
    // This CTA's histogram segment is a pool of `pages` pages of 2^chunk_log entries.  The common log fills it from page 0
    // upwards, [0, seg_len); the hot logs take single pages from its top downwards, [hot_top, pages), and give them back
    // to a free stack.  A hot log holds the entries whose passive partner is one of the first hot_n expressions this CTA
    // owns: such an expression is rewritten over and over, and every time ALL entries of its log die at once -- its pages
    // are freed instead of re-reading them.  A hot log that cannot get a page spills into the common log.
    int seg_len;       // entries (live + dead) in the common log, [0, cap0)
    int cap0;          // room of the common log: hot_top pages
    int pages, hot_top, n_used, n_free, hot_n;
    int hot_room;      // entries one step can append to one hot log at most: a hot log keeps that much room ahead
    int hot_len[DA_HOT_MAX];  // entries of each hot log (may run past its pages while a step appends: readers clamp)
    int hot_snap[DA_HOT_MAX]; // the same at the start of the step (what the argmax caches have to cover)
    int hot_np[DA_HOT_MAX];   // pages each hot log holds
    Best pend[DA_HOT_MAX + 1]; // maximum of the entries appended to each log in the current step (0: the common log)
    int n_new;         // entries appended in the current step
    int live_old;      // live entries counted by the last full rescan (accounting mode)
    int n_dirty;       // pages to re-read in the current step
    int status;        // sticky error
    int list_max;      // longest column list seen by this CTA
    unsigned long long r_count;   // digit pairs enumerated by this CTA (all steps)
    unsigned long long rescanned; // histogram entries re-read by this CTA (all steps)
    unsigned bar_target;
    unsigned epoch;    // exchanges done by this group so far (tags the all-gather slots)
    int scratch_i[4];
    long long phase[9]; // the step's phases (DA_LAP), then team R's counting in the recount (own_recount_help)
    long long t_last;
    long long t_start; // start of the greedy loop (thread 0; the milestones of the phase timers)
    long long poll_iters;
    long long peak[8];
    long long nslow[8];
    int cmp_out;
    int r_step;        // digit pairs enumerated in the current step
    int rescan_step;   // histogram entries re-read in the current step
    unsigned long long xw[3]; // a group of one CTA: the payload words of its exchange
    // The problem's tie-break mask (ProblemDesc::tb_mask).  Histogram entries, page caches, Bests and the exchange carry
    // pack_key ^ tb_mask, so that every comparison of (score, key) applies the seeded order as it stands; whoever reads
    // id0, sub or shift out of a key XORs the mask back first (id1 is never masked).
    unsigned long long tb_mask;
};

struct Ctx {
    LaunchCfg cfg;
    int rank;
    GroupWs ws;
    FEnt *seg; // this CTA's histogram segment (global)
    // shared memory
    BlockCtx *b;
    uint32_t *cb_score, *cb_khi, *cb_klo; // per-page cached maximum
    unsigned char *cb_dirty;
    uint16_t *dirty_list;
    uint16_t *pg_owner;           // hot page -> (hot log << 8) | its index in that log
    uint16_t *pg_used, *pg_slot;  // the hot pages in use [0, n_used), and each one's position in that list
    uint16_t *pg_free;            // free stack of hot pages [0, n_free)
    uint16_t *hot_pg;             // [DA_HOT_MAX][DA_HOT_PAGES] the pages of each hot log, in order
};

// Barrier across the G CTAs of a group: monotonic counter, release on arrive / acquire on poll, split in
// arrive / wait so independent work overlaps the wait.  Cross-CTA data is always read with ld.cg.
__device__ __forceinline__ void group_arrive(const Ctx &cx) {
    __syncthreads();
    if (cx.cfg.G > 1 && threadIdx.x == 0) {
#ifdef DA_CPU_SIM
        __atomic_fetch_add(cx.ws.barrier, 1u, __ATOMIC_RELEASE);
#else
        asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(cx.ws.barrier) : "memory");
#endif
        cx.b->bar_target += (unsigned)cx.cfg.G;
    }
}
__device__ __forceinline__ void group_wait(const Ctx &cx) {
    if (cx.cfg.G > 1 && threadIdx.x == 0) {
        const unsigned target = cx.b->bar_target;
        while ((int)(ld_acquire_u32(cx.ws.barrier) - target) < 0) {
        }
    }
    __syncthreads();
}
__device__ __forceinline__ void group_sync(const Ctx &cx) {
    group_arrive(cx);
    group_wait(cx);
}

// Tagged all-gather exchange: every CTA pushes its candidate into its own slot and reads all G slots; there is no
// arrive counter and no second round trip.  Every 64-bit word of a slot carries the exchange's tag in its top 13 bits,
// so a reader knows from the word alone that it is current:
//   w0 = tag | want (1) | status (4) | score (32) | key >> 50 (14)      w1 = tag | key & (2^50 - 1)
//   w2 = tag | live (28), accounting mode only
// Slots are double-buffered by exchange parity and laid out word-major ([parity][word][G]), so that one warp reads the
// words of all CTAs in a few coalesced lines.  A slot is overwritten two exchanges later, which no CTA can reach before
// every CTA has read it; the tag therefore only has to differ from that of the exchange two before (it runs through
// 1..8191 and never matches the zeroes the host writes before a launch).  The epoch runs on across the problems a group
// solves one after the other.
//
// Memory model.  Besides the payload, readers of the next step need the global writes of this step that precede the
// exchange: the cells and directory entries of own_update and CTA 0's op record and rewrite stamps.  The publishing
// thread executes fence.acq_rel.gpu after those writes (directly, or after a CTA barrier that orders them) and then
// stores the words with strong relaxed stores: fence + strong store in one thread is a release pattern.  The reader
// loads w0 with ld.acquire.gpu after the other words; observing w0's tag synchronizes with the writer, and the CTA
// barrier behind the collect passes that on to every thread of the reading CTA.  The reader's loads of exchange e are
// ordered before its own publish of e + 1 (CTA barrier, then the publisher's fence), which every writer of e + 2
// observes first: the parity slot is never overwritten while somebody still reads it.
#define DA_XCHG_LO ((1ULL << 50) - 1ULL)
__device__ __forceinline__ unsigned long long xchg_tag(unsigned epoch) { return (unsigned long long)(epoch % 8191u + 1u) << 51; }
__device__ __forceinline__ bool xchg_current(unsigned long long w, unsigned long long tag) { return (w & ~((1ULL << 51) - 1ULL)) == tag; }

__device__ __forceinline__ void fence_acq_rel_gpu() {
#ifdef DA_CPU_SIM
    __atomic_thread_fence(__ATOMIC_ACQ_REL); // (the race checker does not model fences: the slot stores are release stores)
#else
    asm volatile("fence.acq_rel.gpu;" ::: "memory");
#endif
}
__device__ __forceinline__ void st_relaxed_u64(unsigned long long *p, unsigned long long v) {
#ifdef DA_CPU_SIM
    __atomic_store_n(p, v, __ATOMIC_RELEASE);
#else
    asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
#endif
}
// polls of an exchange slot (a poll yields under the CPU simulation)
__device__ __forceinline__ unsigned long long ld_relaxed_u64(const unsigned long long *p) {
#ifdef DA_CPU_SIM
    simt::poll_yield();
    return __atomic_load_n(p, __ATOMIC_RELAXED);
#else
    unsigned long long v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
#endif
}
__device__ __forceinline__ unsigned long long ld_acquire_u64(const unsigned long long *p) {
#ifdef DA_CPU_SIM
    simt::poll_yield();
    return __atomic_load_n(p, __ATOMIC_ACQUIRE);
#else
    unsigned long long v;
    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
#endif
}

// One thread: this CTA's candidate -> its slot.  `fenced`: the thread has executed the release fence since the writes
// the exchange has to carry (else it fences here).
__device__ __forceinline__ void xchg_publish(const Ctx &cx, const Best &v, int status, bool want, int live, bool fenced) {
    BlockCtx &b = *cx.b;
    b.epoch += 1u;
    const unsigned long long tag = xchg_tag(b.epoch), key = ((unsigned long long)v.khi << 32) | v.klo;
    const unsigned long long w0 = tag | ((unsigned long long)want << 50) | ((unsigned long long)(status & 0xf) << 46) | ((unsigned long long)v.score << 14) | (key >> 50);
    const unsigned long long w1 = tag | (key & DA_XCHG_LO), w2 = tag | ((unsigned long long)live & 0x0fffffffULL);
    const int G = cx.cfg.G;
    if (G > 1) {
        if (!fenced)
            fence_acq_rel_gpu();
        unsigned long long *s = cx.ws.xchg + (size_t)(b.epoch & 1u) * 4 * G + cx.rank;
        st_relaxed_u64(s + G, w1);
        if (cx.cfg.accounting)
            st_relaxed_u64(s + 2 * G, w2);
        st_relaxed_u64(s, w0);
    }
    else {
        b.xw[0] = w0;
        b.xw[1] = w1;
        b.xw[2] = w2;
    }
}

__device__ __forceinline__ void load_op(const ProblemDesc &p, uint32_t id, QInt &q, float &lat) {
    if ((int)id < p.n_in) {
        q.min = p.qint[3 * id + 0];
        q.max = p.qint[3 * id + 1];
        q.step = p.qint[3 * id + 2];
        lat = p.lat[id];
    }
    else {
        float4 v = __ldcg(&p.op_q[id]);
        q.min = v.x;
        q.max = v.y;
        q.step = v.z;
        lat = v.w;
    }
}

#define DA_DEAD 0xffffffffu
#define DA_LAP(k)                                                              \
    if (threadIdx.x == 0) {                                                    \
        const long long _now = clock64();                                      \
        cx.b->phase[k] += _now - cx.b->t_last;                                 \
        cx.b->peak[k] = max(cx.b->peak[k], _now - cx.b->t_last);               \
        if (_now - cx.b->t_last > 20000)                                       \
            cx.b->nslow[k] += 1;                                               \
        cx.b->t_last = _now;                                                   \
    }

// Pages of the segment in use: the common log's pages [0, nc) (nc = common_pages(seg_len)), then the hot pages in use.
// `seg_len` = fill of the common log; the hot logs' fills come from their step-start snapshot.
__device__ __forceinline__ int common_pages(const Ctx &cx, int seg_len) { return (seg_len + (1 << cx.cfg.chunk_log) - 1) >> cx.cfg.chunk_log; }
__device__ __forceinline__ int pages_in_use(const Ctx &cx, int nc) { return nc + cx.b->n_used; }
__device__ __forceinline__ int page_at(const Ctx &cx, int i, int nc) { return i < nc ? i : (int)cx.pg_used[i - nc]; }
// the entries [lo, hi) of page pg
__device__ __forceinline__ void page_span(const Ctx &cx, int pg, int seg_len, int &lo, int &hi) {
    const BlockCtx &b = *cx.b;
    const int cl = cx.cfg.chunk_log;
    lo = pg << cl;
    if (pg < b.hot_top)
        hi = min(lo + (1 << cl), seg_len);
    else {
        const int o = cx.pg_owner[pg];
        hi = lo + min(1 << cl, b.hot_snap[o >> 8] - ((o & 255) << cl));
    }
    hi = max(hi, lo);
}
// position of entry v of log r (0: the common log, k + 1: hot log k) in the segment
__device__ __forceinline__ int log_pos(const Ctx &cx, int r, int v) {
    const int cl = cx.cfg.chunk_log;
    return r == 0 ? v : ((int)cx.hot_pg[(r - 1) * DA_HOT_PAGES + (v >> cl)] << cl) + (v & ((1 << cl) - 1));
}

// Append one histogram entry (created at step `stamp`) to this CTA's segment and fold it into the
// thread's running best.
__device__ __forceinline__ void
emit_entry(const ProblemDesc &p, const Ctx &cx, uint32_t lo, uint32_t hi, int shift, int sub, uint32_t count, QInt q0, float l0, QInt q1, float l1, uint32_t stamp, uint32_t thresh, Best &best, bool mark_dirty = true, int hot = -1) {
    uint32_t score;
    if (!pair_score(p.method, count, q0, l0, q1, l1, score))
        return; // NaN score: can never be selected
    const uint64_t key = pack_key(lo, hi, shift, sub) ^ cx.b->tb_mask;
    int pos = -1;
    if (hot >= 0) { // the passive partner's own log; when its pages are full the entry goes to the common log like any other
        const int q = smem_add(&cx.b->hot_len[hot], 1);
        if (q < (cx.b->hot_np[hot] << cx.cfg.chunk_log))
            pos = log_pos(cx, hot + 1, q);
    }
    if (pos < 0) {
        pos = smem_add(&cx.b->seg_len, 1);
        if (pos >= cx.b->cap0) {
            cx.b->status = ST_FSEG_OVERFLOW;
            return;
        }
    }
    if (cx.cfg.accounting)
        smem_add(&cx.b->n_new, 1); // only the exact live count of accounting mode needs it
    FEnt e;
    e.x = score;
    e.y = stamp;
    e.z = (uint32_t)key;
    e.w = (uint32_t)(key >> 32);
    cx.seg[pos] = e;
    if (mark_dirty) // (else the caller marks the chunks of everything it appended)
        st_racy(&cx.cb_dirty[pos >> cx.cfg.chunk_log], (unsigned char)1); // this page's cached maximum does not cover the new entry yet
    if (score >= thresh) {
        Best c{score, e.w, e.z};
        if (best_gt(c, best))
            best = c;
    }
}


} // namespace da
