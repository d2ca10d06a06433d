// cmvm_num.cuh -- scalar numerics of the CMVM path, shared by device kernels and the host-side
// C-ABI helpers.  Every function names the reference lines whose arithmetic it reproduces
// bit-for-bit.  No fast-math, no FMA contraction: all float ops go through explicit _rn helpers.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>

#if defined(__CUDACC__)
#define DA_HD __host__ __device__ __forceinline__
#else
#define DA_HD inline
#endif

namespace da {

struct QInt {
    float min, max, step;
};

DA_HD uint32_t f2u(float x) {
#if defined(__CUDA_ARCH__)
    return __float_as_uint(x);
#else
    uint32_t u;
    memcpy(&u, &x, 4);
    return u;
#endif
}
DA_HD float u2f(uint32_t u) {
#if defined(__CUDA_ARCH__)
    return __uint_as_float(u);
#else
    float x;
    memcpy(&x, &u, 4);
    return x;
#endif
}
// IEEE round-to-nearest single ops that the compiler may not fuse into FMAs.
DA_HD float fadd(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fadd_rn(a, b);
#else
    volatile float r = a + b;
    return r;
#endif
}
DA_HD float fsub(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fsub_rn(a, b);
#else
    volatile float r = a - b;
    return r;
#endif
}
DA_HD float fmul(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fmul_rn(a, b);
#else
    volatile float r = a * b;
    return r;
#endif
}
DA_HD float fdiv(float a, float b) {
#if defined(__CUDA_ARCH__)
    return __fdiv_rn(a, b);
#else
    volatile float r = a / b;
    return r;
#endif
}
DA_HD float fmaxf_std(float a, float b) { return (a < b) ? b : a; } // std::max(a,b)
DA_HD float fminf_std(float a, float b) { return (b < a) ? b : a; } // std::min(a,b)

// 2^s as float for |s| small (std::pow(2.0, shift) cast to float: state_opr.cc:23,50)
DA_HD float pow2f(int64_t s) {
    if (s > 127)
        return u2f(0x7f800000u);
    if (s >= -126)
        return u2f((uint32_t)(s + 127) << 23);
    if (s >= -149)
        return u2f(1u << (s + 149));
    return 0.0f;
}

// glibc log2f stand-in.  glibc's log2f evaluates a double-precision polynomial and rounds once to
// float; (float)log2((double)x) agrees with it wherever a trunc()/ceil() of the result is taken in
// the reference (checked against glibc in tests/test_numerics.py over every exponent with
// mantissas adjacent to powers of two, where the two could differ).
DA_HD float log2f_ref(float x) { return (float)log2((double)x); }

// ceil(log2(y)) for finite y > 0, exact (replaces std::ceil(std::log2(double)) where the argument is
// never within rounding distance of a power of two unless it is one: bit_decompose.cc:25, mat_decompose.cc:19)
DA_HD int ceil_log2_pos(double y) {
    int e;
    double m = frexp(y, &e); // y = m * 2^e, m in [0.5,1)
    return (m == 0.5) ? e - 1 : e;
}

// static_cast<int64_t>(float) with x86 cvttss2si semantics for NaN/inf/out-of-range (cmvm_core.cc:137,187)
DA_HD int64_t trunc_i64(float v) {
    if (!(v > -9.2e18f && v < 9.2e18f))
        return INT64_MIN;
    return (int64_t)v;
}

// static_cast<int32_t>(float) with x86 cvttss2si semantics: INT32_MIN for NaN, +-inf and |v| >= 2^31 (bit_decompose.cc:59,
// mat_decompose.cc:81-82).  A plain cast on the device saturates instead, and gives 0 for NaN.
DA_HD int32_t trunc_i32(float v) {
    if (!(v > -2147483904.0f && v < 2147483648.0f)) // -2147483904 is the float below -2^31
        return INT32_MIN;
    return (int32_t)v;
}

// One step of the CSD digit loop (bit_decompose.cc:33-39) in the wrapping int32 arithmetic the reference compiles to:
// at n = 31 the threshold `_2pn * 2 / 3` is 0, at n = 30 it is -(2^31 / 3), and `x -= _2pn * d` wraps.  Returns the
// digit of weight 2^n and leaves the remainder in x.
DA_HD int csd_digit_i32(int32_t &x, int n) {
    const uint32_t p2 = 1u << n;
    const int32_t thres = (int32_t)(p2 * 2u) / 3;
    const int d = (x > thres) - (x < -thres);
    x = (int32_t)((uint32_t)x - p2 * (uint32_t)d);
    return d;
}

// |x| as it enters the width max (bit_decompose.cc:23): |INT32_MIN| wraps to itself there and never wins the max.
DA_HD int32_t csd_abs(int32_t x) { return x == INT32_MIN ? 0 : (x < 0 ? -x : x); }

// CSD width N of values whose largest csd_abs is max_abs (bit_decompose.cc:24-27)
DA_HD int csd_nbits(int32_t max_abs) {
    const int n = ceil_log2_pos((double)fmaxf((float)max_abs, 1.0f) * 1.5);
    return n > 1 ? n : 1;
}

// indexers.hh:12-18
DA_HD int8_t iceil_log2(float x) {
    uint32_t bits = f2u(x);
    uint8_t exp = (uint8_t)((bits >> 23) & 0xFF);
    uint32_t mant = bits & 0x7FFFFF;
    return (int8_t)(exp - 127 + (mant != 0));
}

// bit_decompose.cc:10-20
DA_HD int8_t get_lsb_loc(float x) {
    if (x == 0.0f)
        return 127;
    uint32_t bits = f2u(x);
    uint8_t exp = (uint8_t)((bits >> 23) & 0xFF);
    uint32_t mant = bits & 0x7FFFFF;
    uint32_t m = mant + (1u << 23);
#if defined(__CUDA_ARCH__)
    int mtz = __ffs(m) - 1;
#else
    int mtz = __builtin_ctz(m);
#endif
    return (int8_t)(exp + mtz - 150);
}

// state_opr.cc:8-29
DA_HD QInt qint_add(QInt q0, QInt q1, int64_t shift, bool sub0, bool sub1) {
    float min0 = q0.min, max0 = q0.max, step0 = q0.step;
    float min1 = q1.min, max1 = q1.max, step1 = q1.step;
    if (sub0) {
        float t = min0;
        min0 = -max0;
        max0 = -t;
    }
    if (sub1) {
        float t = min1;
        min1 = -max1;
        max1 = -t;
    }
    float s = pow2f(shift);
    min1 = fmul(min1, s);
    max1 = fmul(max1, s);
    step1 = fmul(step1, s);
    QInt r;
    r.min = fadd(min0, min1);
    r.max = fadd(max0, max1);
    r.step = fminf_std(step0, step1);
    return r;
}

// state_opr.cc:31-67; returns {dlat, cost}
DA_HD void cost_add(QInt q0, QInt q1, int64_t shift, bool sub, int adder_size, int carry_size, float &dlat, float &cost) {
    if (adder_size < 0 && carry_size < 0) {
        dlat = 1.0f;
        cost = 1.0f;
        return;
    }
    if (adder_size < 0)
        adder_size = 65535;
    if (carry_size < 0)
        carry_size = 65535;
    float min0 = q0.min, max0 = q0.max, step0 = q0.step;
    float min1 = q1.min, max1 = q1.max, step1 = q1.step;
    if (sub) {
        float t = min1;
        min1 = max1;
        max1 = t;
    }
    float sf = pow2f(shift);
    min1 = fmul(min1, sf);
    max1 = fmul(max1, sf);
    step1 = fmul(step1, sf);
    max0 = fadd(max0, step0);
    max1 = fadd(max1, step1);
    float f = -log2f_ref(fmaxf_std(step0, step1));
    // std::max({a,b,c,d}) = first maximal element, left fold with operator<
    float m = fabsf(min0);
    float c1 = fabsf(min1), c2 = fabsf(max0), c3 = fabsf(max1);
    if (m < c1)
        m = c1;
    if (m < c2)
        m = c2;
    if (m < c3)
        m = c3;
    float i = ceilf(log2f_ref(m));
    int k = (q0.min < 0 || q1.min < 0) ? 1 : 0;
    float n_accum = fadd(fadd((float)k, i), f);
    dlat = ceilf(fdiv(n_accum, (float)carry_size));
    cost = ceilf(fdiv(n_accum, (float)adder_size));
}

// indexers.cc:36-56
DA_HD void overlap_and_accum(QInt q0, QInt q1, int8_t &n_overlap, int8_t &n_accum) {
    float min0 = q0.min, max0 = q0.max, step0 = q0.step;
    float min1 = q1.min, max1 = q1.max, step1 = q1.step;
    max0 = fadd(max0, step0);
    max1 = fadd(max1, step1);
    int8_t f = (int8_t)(-(int)iceil_log2(fmaxf_std(step0, step1)));
    float a0 = fabsf(min0), a1 = fabsf(min1), b0 = fabsf(max0), b1 = fabsf(max1);
    float hi = a0;
    if (hi < a1)
        hi = a1;
    if (hi < b0)
        hi = b0;
    if (hi < b1)
        hi = b1;
    int8_t i_high = iceil_log2(hi);
    int8_t i_low = iceil_log2(fminf_std(fmaxf_std(a0, b0), fmaxf_std(a1, b1)));
    int8_t k = (q0.min < 0 || q1.min < 0) ? 1 : 0;
    n_accum = (int8_t)((int)k + (int)i_high + (int)f);
    n_overlap = (int8_t)((int)k + (int)i_low + (int)f);
}

// order-preserving map float -> uint32 (with -0 canonicalised and NaN excluded by the caller)
DA_HD uint32_t sortable_f32(float f) {
    uint32_t u = f2u(fadd(f, 0.0f));
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
DA_HD uint32_t sortable_i32(int32_t v) { return (uint32_t)v ^ 0x80000000u; }

enum Method : int { M_MC = 0, M_MC_DC = 1, M_MC_PDC = 2, M_WMC = 3, M_WMC_DC = 4, M_WMC_PDC = 5, M_DUMMY = 6 };

// Selector score of one histogram entry, as a sortable uint32 (indexers.cc:6-90).  Returns false
// when the entry can never be selected (NaN score).
DA_HD bool pair_score(int method, uint32_t count, QInt q0, float lat0, QInt q1, float lat1, uint32_t &key) {
    switch (method) {
    case M_MC: // idx_mc: size_t compare of the count
        key = sortable_i32((int32_t)count);
        return true;
    case M_MC_DC:
    case M_MC_PDC: { // idx_mc_dc: count - 1e9*|dlat| in float
        float score = fsub((float)count, fmul(1e9f, fabsf(fsub(lat0, lat1))));
        if (score != score)
            return false;
        key = sortable_f32(score);
        return true;
    }
    case M_WMC: { // idx_wmc: int64(count) * n_overlap
        int8_t ov, ac;
        overlap_and_accum(q0, q1, ov, ac);
        int64_t s = (int64_t)count * (int64_t)ov;
        if (s > 2147483647LL)
            s = 2147483647LL;
        if (s < -2147483647LL)
            s = -2147483647LL;
        key = sortable_i32((int32_t)s);
        return true;
    }
    case M_WMC_DC:
    case M_WMC_PDC: { // idx_wmc_dc: (uint32 * int8 -> unsigned wraparound) - 256*|dlat| in float
        int8_t ov, ac;
        overlap_and_accum(q0, q1, ov, ac);
        uint32_t prod = count * (uint32_t)(int32_t)ov;
        float score = fsub((float)prod, fmul(256.0f, fabsf(fsub(lat0, lat1))));
        if (score != score)
            return false;
        key = sortable_f32(score);
        return true;
    }
    default:
        return false;
    }
}

// smallest sortable score that the selector accepts (the `max_score` initial value)
DA_HD uint32_t method_threshold(int method) {
    switch (method) {
    case M_MC:
        return sortable_i32(0);
    case M_WMC:
        return sortable_i32(0);
    case M_MC_DC:
    case M_WMC_DC:
        return sortable_f32(0.0f);
    case M_MC_PDC:
    case M_WMC_PDC:
        return sortable_f32(u2f(0xff800000u)); // -inf
    default:
        return 0xffffffffu;
    }
}

// packed histogram key; integer order == Pair::operator< (types.hh:28-36): id1, id0, sub, shift
DA_HD uint64_t pack_key(uint32_t id0, uint32_t id1, int shift, int sub) {
    return ((uint64_t)id1 << 36) | ((uint64_t)id0 << 8) | ((uint64_t)(sub & 1) << 7) | (uint64_t)(shift + 64);
}
DA_HD uint32_t key_id1(uint64_t k) { return (uint32_t)(k >> 36); }
DA_HD uint32_t key_id0(uint64_t k) { return (uint32_t)(k >> 8) & 0x0fffffffu; }
DA_HD int key_sub(uint64_t k) { return (int)(k >> 7) & 1; }
DA_HD int key_shift(uint64_t k) { return (int)(k & 127) - 64; }

// Seeded tie-break (this project's extension; the reference has only seed 0).  Among entries of equal score the greedy
// selection takes the largest key ^ tb_mask(seed).  The mask covers the id0, sub and shift bits of pack_key and never
// id1, so the newest expression still wins ties; tb_mask(0) = 0 is the reference's order.
DA_HD uint64_t tb_mask(uint64_t seed) {
    if (seed == 0)
        return 0;
    uint64_t x = seed + 0x9E3779B97F4A7C15ull; // splitmix64
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    x ^= x >> 31;
    return x & ((1ull << 36) - 1);
}

// number of non-zero CSD digits of |x| (equals the digit count of bit_decompose.cc:22-42, which is
// the non-adjacent form; equivalence is checked exhaustively in tests/test_numerics.py)
DA_HD int csd_weight(int32_t x) {
    uint64_t u = x < 0 ? (uint64_t)(-(int64_t)x) : (uint64_t)x;
    uint64_t h = u >> 1;
    uint64_t t = u + h;
    uint64_t c = t ^ h;
#if defined(__CUDA_ARCH__)
    return __popcll(c);
#else
    return __builtin_popcountll(c);
#endif
}

// Non-zero digits of x among the nbits digits of the loop (csd_digit_i32).  Up to 30 digits and 3|x| <= 2^(nbits+1)
// that is the non-adjacent form's weight; otherwise (the wrapped thresholds of 31 and 32 digits, INT32_MIN, or a value
// whose float rounded down to a narrower width) the loop runs.
DA_HD int csd_count_i32(int32_t x, int nbits) {
    if (nbits <= 30 && x != INT32_MIN && 3 * (int64_t)csd_abs(x) <= (int64_t)2 << nbits)
        return csd_weight(x);
    int c = 0;
    for (int n = nbits - 1; n >= 0; --n)
        c += csd_digit_i32(x, n) != 0;
    return c;
}

} // namespace da
