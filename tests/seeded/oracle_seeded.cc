// oracle_seeded.cc -- TEST INFRASTRUCTURE ONLY: the CPU oracle (oracle/cmvm_oracle.cc, included unmodified) under the
// seeded tie-break of the greedy pair selection.  The seeded order is this project's extension, not the reference's:
// among histogram entries of equal selector score, the one whose pack_key ^ tb_mask(seed) is largest is taken, where
// pack_key = id1 << 36 | id0 << 8 | sub << 7 | shift + 64 (da4ml_b200/csrc/cmvm_num.cuh) and tb_mask(0) = 0, so seed 0
// is the reference's rule (">=" over the key-sorted histogram keeps the largest key).  Everything else -- substitution,
// recount, adder trees, decomposition, latency retries, the argmin over decompose_dc -- is the oracle's own code; only
// the control flow that calls the selection is restated here with the seed threaded through.
#include "../../oracle/cmvm_oracle.cc"

namespace orc {

static uint64_t tb_mask(uint64_t seed) {
    if (seed == 0)
        return 0;
    uint64_t x = seed + 0x9E3779B97F4A7C15ull; // splitmix64
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    x ^= x >> 31;
    return x & ((1ull << 36) - 1);
}
static uint64_t packed(const Key &k) { return ((uint64_t)k.id1 << 36) | ((uint64_t)k.id0 << 8) | ((uint64_t)(k.sub ? 1 : 0) << 7) | (uint64_t)(k.shift + 64); }

// The largest (score, packed key ^ mask) among entries whose score is at or above the starting `best`.
template <class T> struct Pick {
    T best;
    uint64_t mask;
    Key &out;
    bool found = false;
    void offer(const Key &k, T score) {
        if (score > best || (score == best && (!found || (packed(k) ^ mask) > (packed(out) ^ mask)))) {
            best = score;
            out = k;
            found = true;
        }
    }
};

// select_pair (indexers.cc:6-90) with the seeded order; the scores are the oracle's
static bool select_pair_seeded(const State &st, const std::string &m, uint64_t mask, Key &out) {
    if (m == "mc") {
        Pick<size_t> p{0, mask, out};
        for (auto &kv : st.freq)
            p.offer(kv.first, kv.second);
        return p.found;
    }
    if (m == "mc-dc" || m == "mc-pdc") {
        Pick<float> p{(m == "mc-dc") ? 0 : -std::numeric_limits<float>::infinity(), mask, out};
        float factor = 1e9;
        for (auto &kv : st.freq) {
            float l0 = st.ops[kv.first.id0].lat, l1 = st.ops[kv.first.id1].lat;
            p.offer(kv.first, kv.second - factor * std::abs(l0 - l1));
        }
        return p.found;
    }
    if (m == "wmc") {
        Pick<int64_t> p{0, mask, out};
        for (auto &kv : st.freq) {
            auto [ov, ac] = overlap_and_accum(st.ops[kv.first.id0].q, st.ops[kv.first.id1].q);
            (void)ac;
            p.offer(kv.first, int64_t(kv.second) * ov);
        }
        return p.found;
    }
    if (m == "wmc-dc" || m == "wmc-pdc") {
        Pick<float> p{(m == "wmc-dc") ? 0 : -std::numeric_limits<float>::infinity(), mask, out};
        for (auto &kv : st.freq) {
            auto [ov, ac] = overlap_and_accum(st.ops[kv.first.id0].q, st.ops[kv.first.id1].q);
            (void)ac;
            float l0 = st.ops[kv.first.id0].lat, l1 = st.ops[kv.first.id1].lat;
            p.offer(kv.first, kv.second * ov - 256 * std::abs(l0 - l1));
        }
        return p.found;
    }
    throw std::runtime_error("Unknown method: " + m);
}

// greedy / solve_single / solve_one / solve of cmvm_oracle.cc with the seed threaded through
static State greedy_seeded(const Mat &kernel, int n_in, int n_out, const std::string &method, const std::vector<QI> &q, const std::vector<float> &lat, int adder_size, int carry_size, Stage *cnt, uint64_t mask) {
    State st = create_state(kernel, n_in, n_out, q, lat, false, cnt);
    if (method != "mc" && method != "mc-dc" && method != "mc-pdc" && method != "wmc" && method != "wmc-dc" && method != "wmc-pdc" && method != "dummy") {
        if (!st.freq.empty())
            throw std::runtime_error("Unknown method: " + method);
        return st;
    }
    while (!st.freq.empty() && method != "dummy") {
        Key k;
        int64_t fsz = (int64_t)st.freq.size();
        if (!select_pair_seeded(st, method, mask, k))
            break;
        substitute(st, k, adder_size, carry_size);
        int64_t r = recount(st, k);
        if (cnt) {
            cnt->T += 1;
            cnt->sum_f += fsz;
            cnt->sum_r += r;
        }
    }
    return st;
}
static Stage solve_single_seeded(const Mat &k, int n_in, int n_out, const std::string &method, const std::vector<QI> &q, const std::vector<float> &lat, int adder_size, int carry_size, uint64_t mask) {
    Stage cnt;
    State st = greedy_seeded(k, n_in, n_out, method, q, lat, adder_size, carry_size, &cnt, mask);
    Stage out = finish(st, adder_size, carry_size);
    out.T = cnt.T, out.sum_f = cnt.sum_f, out.sum_r = cnt.sum_r, out.f0 = cnt.f0, out.r0 = cnt.r0, out.d0 = cnt.d0;
    return out;
}
static std::vector<Stage> solve_one_seeded(const Mat &kernel, int n_in, int n_out, std::string method0, std::string method1, int hard_dc, int decompose_dc, const std::vector<QI> &q, const std::vector<float> &lat, int adder_size, int carry_size, uint64_t mask) {
    if (method1 == "auto")
        method1 = (hard_dc >= 6 || ends_with(method0, "dc")) ? method0 : method0 + "-dc";
    if (hard_dc == 0 && !ends_with(method0, "dc"))
        method0 = method0 + "-dc";
    float min_lat = std::numeric_limits<float>::infinity();
    if (hard_dc >= 0)
        min_lat = minimal_latency(kernel, n_in, n_out, q, lat, carry_size, adder_size);
    float allowed = hard_dc + min_lat;
    int log2_n = (int)std::ceil(std::log2((float)n_in));
    decompose_dc = decompose_dc == -2 ? std::min(hard_dc, log2_n) : std::min({hard_dc, decompose_dc, log2_n});
    Stage s0, s1;
    while (true) {
        if (decompose_dc < 0 && hard_dc >= 0) {
            if (method0 != "dummy")
                method0 = method1 = "wmc-dc";
            else
                method0 = method1 = "dummy";
        }
        Mat m0, m1;
        kernel_decompose(kernel, n_in, n_out, decompose_dc, m0, m1);
        s0 = solve_single_seeded(m0, n_in, n_out, method0, q, lat, adder_size, carry_size, mask);
        std::vector<QI> q0;
        std::vector<float> l0;
        for (int64_t idx : s0.out_idxs) {
            l0.push_back(idx >= 0 ? s0.ops[idx].lat : 0.0f);
            q0.push_back(idx >= 0 ? s0.ops[idx].q : QI{0.0f, 0.0f, std::numeric_limits<float>::infinity()});
        }
        const bool both = method0 == "wmc-dc" && method1 == "wmc-dc";
        if (stage_max_lat(s0) > allowed && (!both || decompose_dc >= 0)) {
            decompose_dc--;
            continue;
        }
        s1 = solve_single_seeded(m1, n_out, n_out, method1, q0, l0, adder_size, carry_size, mask);
        if (stage_max_lat(s1) > allowed && (!both || decompose_dc >= 0)) {
            decompose_dc--;
            continue;
        }
        break;
    }
    return {s0, s1};
}
static std::vector<Stage> solve_seeded(const Mat &kernel, int n_in, int n_out, const std::string &method0, const std::string &method1, int hard_dc, int decompose_dc, std::vector<QI> q, std::vector<float> lat, int adder_size, int carry_size, bool search_all, uint64_t mask) {
    if (q.empty())
        q.assign(n_in, QI{-128.0f, 127.0f, 1.0f});
    if (lat.empty())
        lat.assign(n_in, 0.0f);
    if (!search_all)
        return solve_one_seeded(kernel, n_in, n_out, method0, method1, hard_dc, decompose_dc, q, lat, adder_size, carry_size, mask);
    int hd = hard_dc < 0 ? 1000000000 : hard_dc;
    int max_dc = std::min(hd, (int)std::ceil(std::log2((float)n_in)));
    std::vector<int> tries;
    for (int d = -1; d <= max_dc; ++d)
        tries.push_back(d);
    std::vector<std::vector<Stage>> cand(tries.size());
    std::vector<float> costs(tries.size());
    std::string err;
#pragma omp parallel for schedule(dynamic)
    for (size_t i = 0; i < tries.size(); ++i) {
        try {
            cand[i] = solve_one_seeded(kernel, n_in, n_out, method0, method1, hd, tries[i], q, lat, adder_size, carry_size, mask);
            float c = 0.0f;
            for (auto &s : cand[i])
                for (auto &op : s.ops)
                    c += op.cost;
            costs[i] = c;
        }
        catch (const std::exception &e) {
#pragma omp critical
            err = e.what();
        }
    }
    if (!err.empty())
        throw std::runtime_error(err);
    size_t best = 0;
    for (size_t i = 1; i < tries.size(); ++i)
        if (costs[i] < costs[best])
            best = i;
    return cand[best];
}

} // namespace orc

extern "C" {

uint64_t orc_tb_mask(uint64_t seed) { return orc::tb_mask(seed); }

void *orc_solve_seeded(const float *kernel, int64_t n_in, int64_t n_out, const char *method0, const char *method1, int hard_dc, int decompose_dc, const float *qint, const float *lat, int adder_size, int carry_size, int search_all, uint64_t seed) {
    try {
        auto *h = new Handle();
        h->stages = solve_seeded(to_mat(kernel, n_in, n_out), (int)n_in, (int)n_out, method0, method1, hard_dc, decompose_dc, to_q(qint, n_in), lat ? std::vector<float>(lat, lat + n_in) : std::vector<float>{}, adder_size, carry_size, search_all != 0, tb_mask(seed));
        return h;
    }
    catch (const std::exception &e) {
        g_err = e.what();
        return nullptr;
    }
}
void *orc_solve_single_seeded(const float *kernel, int64_t n_in, int64_t n_out, const char *method, const float *qint, const float *lat, int adder_size, int carry_size, uint64_t seed) {
    try {
        auto q = to_q(qint, n_in);
        if (q.empty())
            q.assign(n_in, QI{-128.0f, 127.0f, 1.0f});
        std::vector<float> l = lat ? std::vector<float>(lat, lat + n_in) : std::vector<float>(n_in, 0.0f);
        auto *h = new Handle();
        h->stages.push_back(solve_single_seeded(to_mat(kernel, n_in, n_out), (int)n_in, (int)n_out, method, q, l, adder_size, carry_size, tb_mask(seed)));
        return h;
    }
    catch (const std::exception &e) {
        g_err = e.what();
        return nullptr;
    }
}

} // extern "C"
