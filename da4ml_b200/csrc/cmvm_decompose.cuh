// cmvm_decompose.cuh -- stage-1 graph decomposition W = M0 * M1 on the device
// (reference mat_decompose.cc:6-137; centring bit_decompose.hh:21-34).
//
//   center_kernel    power-of-two normalisation of columns then rows, augmented matrix [0 | centred]
//   dist_kernel      all-pairs column distance = min(CSD weight(a-b), CSD weight(a+b)) summed over rows, each weight
//                    at the CSD width of its whole array, as the reference counts it
//   mst_build_kernel one CTA per delay-constraint candidate: Prim MST with the reference's first-minimum
//                    tie-break, then the sequential construction of M0 (edge columns) and M1 (path matrix)
#pragma once
#include "cmvm_num.cuh"
#include "cmvm_types.cuh"

namespace da {

// aug: [n_in][n_out+1] float, column 0 is zero.  One CTA.
__global__ void __launch_bounds__(256) center_kernel(const float *kernel, int n_in, int n_out, float *aug, int8_t *shift0, int8_t *shift1) {
    const int tid = threadIdx.x, nt = blockDim.x, n = n_out + 1;
    for (int j = tid; j < n_out; j += nt) {
        int m = 127;
        for (int i = 0; i < n_in; ++i)
            m = min(m, (int)get_lsb_loc(kernel[(size_t)i * n_out + j]));
        shift1[j] = (int8_t)m;
    }
    __syncthreads();
    for (int i = tid; i < n_in; i += nt) {
        int m = 127;
        for (int j = 0; j < n_out; ++j) {
            float v = (float)((double)kernel[(size_t)i * n_out + j] * exp2(-(double)shift1[j]));
            m = min(m, (int)get_lsb_loc(v));
        }
        shift0[i] = (int8_t)m;
    }
    __syncthreads();
    for (int idx = tid; idx < n_in * n_out; idx += nt) {
        int i = idx / n_out, j = idx - i * n_out;
        float v = (float)((double)kernel[idx] * exp2(-(double)shift1[j]));
        v = (float)((double)v * exp2(-(double)shift0[i]));
        aug[(size_t)i * n + j + 1] = v;
    }
    for (int i = tid; i < n_in; i += nt)
        aug[(size_t)i * n] = 0.0f;
}

// The reference decomposes the whole [n_in][n][n] array of differences, and that of sums, each with one CSD width taken
// from its largest |int32| (mat_decompose.cc:81-84).  Every CTA first finds both maxima itself: one warp per row takes
// the row's max and min, which bound every difference and sum of the row.  Only a row whose bounds leave the int32 range
// (or that holds a NaN) is searched pair by pair, because its out-of-range values convert to INT32_MIN and take no part.
__device__ __forceinline__ void row_csd_maxima(const float *row, int n, int lane, int &m0, int &m1) {
    float hi = 0.0f, lo = 0.0f; // (column 0 is zero)
    bool bad = false;
    for (int a = lane; a < n; a += 32) {
        const float v = row[a];
        bad |= v != v;
        hi = fmaxf(hi, v);
        lo = fminf(lo, v);
    }
    for (int off = 16; off > 0; off >>= 1) {
        hi = fmaxf(hi, __shfl_xor_sync(0xffffffffu, hi, off));
        lo = fminf(lo, __shfl_xor_sync(0xffffffffu, lo, off));
        bad |= __shfl_xor_sync(0xffffffffu, (int)bad, off) != 0;
    }
    const float d = fsub(hi, lo), s_hi = fadd(hi, hi), s_lo = fadd(lo, lo); // rounding is monotone: the extremes
    if (!bad && d < 2147483648.0f && s_hi < 2147483648.0f && s_lo > -2147483648.0f) {
        m0 = max(m0, csd_abs(trunc_i32(d)));
        m1 = max(m1, max(csd_abs(trunc_i32(s_hi)), csd_abs(trunc_i32(s_lo))));
        return;
    }
    for (int a = lane; a < n; a += 32)
        for (int b = a; b < n; ++b) { // both are symmetric in (a, b)
            m0 = max(m0, csd_abs(trunc_i32(fsub(row[a], row[b]))));
            m1 = max(m1, csd_abs(trunc_i32(fadd(row[a], row[b]))));
        }
}

// dist[a][b] (int32) and sign[a][b] (int8), n = n_out + 1 (mat_decompose.cc:73-93)
__global__ void __launch_bounds__(256) dist_kernel(const float *aug, int n_in, int n, int *dist, int8_t *sign) {
#ifdef DA_CPU_SIM
    DA_SHARED_VAR(int, s_max0);
    DA_SHARED_VAR(int, s_max1);
#else
    __shared__ int s_max0, s_max1;
#endif
    const int tid = threadIdx.x, lane = tid & 31;
    if (tid == 0) {
        s_max0 = 0;
        s_max1 = 0;
    }
    __syncthreads();
    int m0 = 0, m1 = 0;
    for (int i = tid >> 5; i < n_in; i += blockDim.x >> 5)
        row_csd_maxima(aug + (size_t)i * n, n, lane, m0, m1);
    atomicMax(&s_max0, m0);
    atomicMax(&s_max1, m1);
    __syncthreads();
    const long long idx = (long long)blockIdx.x * blockDim.x + tid;
    if (idx >= (long long)n * n)
        return;
    const int a = (int)(idx / n), c = (int)(idx - (long long)a * n);
    const int nb0 = csd_nbits(s_max0), nb1 = csd_nbits(s_max1);
    long long d0 = 0, d1 = 0;
    for (int i = 0; i < n_in; ++i) {
        float x = aug[(size_t)i * n + a], y = aug[(size_t)i * n + c];
        d0 += csd_count_i32(trunc_i32(fsub(x, y)), nb0);
        d1 += csd_count_i32(trunc_i32(fadd(x, y)), nb1);
    }
    sign[idx] = (d1 - d0 < 0) ? -1 : 1;
    dist[idx] = (int)min(d0, d1);
}

struct DecompJob {
    int dc;
    float *m0; // [n_in][n_out]
    float *m1; // [n_out][n_out]
    int *mapping; // [n-1][2] scratch / output
};

__device__ __forceinline__ float lat_of(int cost) { return ceilf(log2f_ref((float)max(cost, 1))); }

// One CTA per job.  Dynamic shared memory: n * (8 + 4 + 4 + 1) bytes.
__global__ void __launch_bounds__(1024) mst_build_kernel(const float *aug, const int *dist, const int8_t *sign, const int8_t *shift0, const int8_t *shift1, int n_in, int n_out, const DecompJob *jobs) {
#ifdef DA_CPU_SIM
    DA_DYN_SHARED(smem_raw);
#else
    extern __shared__ unsigned char smem_raw[];
#endif
    const DecompJob job = jobs[blockIdx.x];
    const int n = n_out + 1, tid = threadIdx.x, nt = blockDim.x;
    const int dc = job.dc;
    long long *bestc = reinterpret_cast<long long *>(smem_raw);
    int *bestj = reinterpret_cast<int *>(bestc + n);
    int *latency = bestj + n;
    unsigned char *impl = reinterpret_cast<unsigned char *>(latency + n);
#ifdef DA_CPU_SIM
    struct Red {
        long long c[32];
        int i[32];
    };
    DA_SHARED_VAR(Red, s_red);
    long long *s_redc = s_red.c;
    int *s_redi = s_red.i;
    DA_SHARED_VAR(int, s_pick);
    DA_SHARED_VAR(int, s_cnt);
#else
    __shared__ long long s_redc[32];
    __shared__ int s_redi[32];
    __shared__ int s_pick;
    __shared__ int s_cnt;
#endif

    const long long PEN = 0x7fffffffffffffffLL / 2;
    float _dc = -1.0f;
    if (dc >= 0) {
        int mc = dist[0];
        for (int j = 1; j < n; ++j)
            mc = max(mc, dist[j]);
        double lg = (mc > 0) ? (double)ceil_log2_pos((double)(float)mc) : -106.0; // ceil(log2(0 + 1e-32)) = -106
        _dc = (float)((exp2((double)dc) - 1.0) + lg);
    }
    for (int i = tid; i < n; i += nt) {
        impl[i] = (i == 0);
        latency[i] = 0;
        long long c = dist[(size_t)i * n];
        if (dc >= 0) {
            float ml = fadd(fmaxf_std(lat_of(dist[(size_t)i * n]), 0.0f), 1.0f);
            if (ml > _dc)
                c = PEN;
        }
        bestc[i] = c;
        bestj[i] = 0;
    }
    __syncthreads();

    // ---- Prim (mat_decompose.cc:22-58): min over (cost, i, j) lexicographic == first minimum of the double loop
    for (int it = 1; it < n; ++it) {
        long long mc = 0x7fffffffffffffffLL;
        int mi = 0x7fffffff;
        for (int i = tid; i < n; i += nt) {
            if (!impl[i]) {
                long long c = bestc[i];
                if (c < mc || (c == mc && i < mi)) {
                    mc = c;
                    mi = i;
                }
            }
        }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
            long long oc = __shfl_xor_sync(0xffffffffu, mc, off);
            int oi = __shfl_xor_sync(0xffffffffu, mi, off);
            if (oc < mc || (oc == mc && oi < mi)) {
                mc = oc;
                mi = oi;
            }
        }
        if ((tid & 31) == 0) {
            s_redc[tid >> 5] = mc;
            s_redi[tid >> 5] = mi;
        }
        __syncthreads();
        if (tid == 0) {
            long long bc = s_redc[0];
            int bi = s_redi[0];
            for (int w = 1; w < (nt >> 5); ++w)
                if (s_redc[w] < bc || (s_redc[w] == bc && s_redi[w] < bi)) {
                    bc = s_redc[w];
                    bi = s_redi[w];
                }
            int j = bestj[bi];
            impl[bi] = 1;
            job.mapping[2 * (it - 1)] = j;
            job.mapping[2 * (it - 1) + 1] = bi;
            latency[bi] = (int)fadd(fmaxf_std(lat_of(dist[(size_t)bi * n + j]), (float)latency[j]), 1.0f);
            s_pick = bi;
        }
        __syncthreads();
        const int jn = s_pick;
        const float latj = (float)latency[jn];
        for (int i = tid; i < n; i += nt) {
            if (!impl[i]) {
                int d = dist[(size_t)i * n + jn];
                long long c = d;
                if (dc >= 0) {
                    float ml = fadd(fmaxf_std(lat_of(d), latj), 1.0f);
                    if (ml > _dc)
                        c = PEN;
                }
                if (c < bestc[i] || (c == bestc[i] && jn < bestj[i])) {
                    bestc[i] = c;
                    bestj[i] = jn;
                }
            }
        }
        __syncthreads();
    }

    // ---- build m0 / m1 (mat_decompose.cc:97-136)
    float *m0 = job.m0, *m1 = job.m1;
    for (int idx = tid; idx < n_in * n_out; idx += nt)
        m0[idx] = 0.0f;
    for (int idx = tid; idx < n_out * n_out; idx += nt)
        m1[idx] = 0.0f;
    __syncthreads();
    if (dc == -1) {
        for (int idx = tid; idx < n_in * n_out; idx += nt) {
            int i = idx / n_out, j = idx - i * n_out;
            m0[idx] = fmul(aug[(size_t)i * n + j + 1], pow2f(shift0[i]));
        }
        for (int j = tid; j < n_out; j += nt)
            m1[(size_t)j * n_out + j] = fmul(1.0f, pow2f(shift1[j]));
        return;
    }
    if (tid == 0)
        s_cnt = 0;
    __syncthreads();
    for (int k = 0; k < n - 1; ++k) {
        const int from = job.mapping[2 * k], to = job.mapping[2 * k + 1];
        const float sgn = (float)sign[(size_t)to * n + from];
        const int cnt = s_cnt;
        int any = 0;
        for (int i = tid; i < n_in; i += nt) {
            float c0 = fsub(aug[(size_t)i * n + to], fmul(aug[(size_t)i * n + from], sgn));
            any |= (c0 != 0.0f);
        }
        any = __syncthreads_or(any);
        if (any) {
            for (int i = tid; i < n_in; i += nt)
                m0[(size_t)i * n_out + cnt] = fsub(aug[(size_t)i * n + to], fmul(aug[(size_t)i * n + from], sgn));
        }
        for (int j = tid; j < n_out; j += nt) {
            float c1 = (from != 0) ? fmul(m1[(size_t)j * n_out + from - 1], sgn) : 0.0f;
            if (any && j == cnt)
                c1 = 1.0f;
            m1[(size_t)j * n_out + to - 1] = c1;
        }
        __syncthreads();
        if (tid == 0 && any)
            s_cnt = cnt + 1;
        __syncthreads();
    }
    for (int idx = tid; idx < n_in * n_out; idx += nt) {
        int i = idx / n_out;
        m0[idx] = fmul(m0[idx], pow2f(shift0[i]));
    }
    for (int idx = tid; idx < n_out * n_out; idx += nt) {
        int j = idx % n_out;
        m1[idx] = fmul(m1[idx], pow2f(shift1[j]));
    }
}

// Bitwise comparison of pairs of float matrices (one CTA per pair): out[pair] = 1 when all n words are equal.  Used by
// the host driver to find candidates whose decomposition produced the very same stage matrix.
struct MatPair {
    const uint32_t *a, *b;
    long long n;
};
__global__ void __launch_bounds__(256) mat_equal_kernel(const MatPair *pairs, int *out) {
    const MatPair pr = pairs[blockIdx.x];
    int same = 1;
    for (long long i = threadIdx.x; i < pr.n; i += blockDim.x)
        same &= pr.a[i] == pr.b[i] ? 1 : 0;
    same = __syncthreads_and(same);
    if (threadIdx.x == 0)
        out[blockIdx.x] = same;
}

} // namespace da
