// cmvm_prep.cuh -- centre + CSD-decompose the constant matrix into packed sign planes, one CTA per problem
// (bit_decompose.hh:21-34, bit_decompose.cc:22-62, state_opr.cc:92-97).
#pragma once
#include "solve_common.cuh"

namespace da {

// ------------------------------------------------------------------------------------------------
// prep: one CTA per problem

__global__ void __launch_bounds__(256) cmvm_prep_kernel(ProblemDesc *probs) {
    ProblemDesc &p = probs[blockIdx.x];
    const int n_in = p.n_in, n_out = p.n_out;
    const int tid = threadIdx.x, nt = blockDim.x;
#ifdef DA_CPU_SIM
    DA_SHARED_VAR(int, s_max);
    DA_SHARED_VAR(int, s_d0);
    DA_SHARED_VAR(int, s_colcap);
    DA_SHARED_VAR(int, s_dcolmax);
    DA_SHARED_VAR(int, s_rowsmax);
#else
    __shared__ int s_max, s_d0, s_colcap, s_dcolmax, s_rowsmax;
#endif
    if (tid == 0) {
        s_max = 0;
        s_d0 = 0;
        s_colcap = 0;
        s_dcolmax = 0;
        s_rowsmax = 0;
    }
    // column shifts (bit_decompose.hh:29): shift1[j] = min_i lsb(k[i,j])
    for (int j = tid; j < n_out; j += nt) {
        int m = 127;
        for (int i = 0; i < n_in; ++i)
            m = min(m, (int)get_lsb_loc(p.kernel[(size_t)i * n_out + j]));
        p.shift1[j] = (int8_t)m;
    }
    __syncthreads();
    // row shifts on the column-scaled matrix (bit_decompose.hh:31)
    for (int i = tid; i < n_in; i += nt) {
        int m = 127;
        for (int j = 0; j < n_out; ++j) {
            float v = (float)((double)p.kernel[(size_t)i * n_out + j] * exp2(-(double)p.shift1[j]));
            m = min(m, (int)get_lsb_loc(v));
        }
        p.shift0[i] = (int8_t)m;
    }
    __syncthreads();
    // global max |centred| -> CSD width (bit_decompose.cc:23-27)
    int lmax = 0;
    for (int idx = tid; idx < n_in * n_out; idx += nt) {
        int i = idx / n_out, j = idx - i * n_out;
        float v = (float)((double)p.kernel[idx] * exp2(-(double)p.shift1[j]));
        v = (float)((double)v * exp2(-(double)p.shift0[i]));
        lmax = max(lmax, csd_abs(trunc_i32(v)));
    }
    atomicMax(&s_max, lmax);
    __syncthreads();
    const int N = csd_nbits(s_max);
    // digits (bit_decompose.cc:29-38) -> sign planes; zero rows of zero-range inputs (state_opr.cc:92-97)
    for (int idx = tid; idx < n_in * n_out; idx += nt) {
        int i = idx / n_out, j = idx - i * n_out;
        float v = (float)((double)p.kernel[idx] * exp2(-(double)p.shift1[j]));
        v = (float)((double)v * exp2(-(double)p.shift0[i]));
        int32_t x = trunc_i32(v);
        uint32_t P = 0, Nn = 0;
        for (int n = N - 1; n >= 0; --n) {
            const int d = csd_digit_i32(x, n);
            if (d > 0)
                P |= 1u << n;
            if (d < 0)
                Nn |= 1u << n;
        }
        if (p.qint[3 * i] == 0.0f && p.qint[3 * i + 1] == 0.0f) {
            P = 0;
            Nn = 0;
        }
        p.masks0[idx] = make_uint2(P, Nn);
    }
    __syncthreads();
    for (int j = tid; j < n_out; j += nt) {
        int d = 0, rows = 0;
        for (int i = 0; i < n_in; ++i) {
            uint2 m = p.masks0[(size_t)i * n_out + j];
            int c = __popc(m.x) + __popc(m.y);
            d += c;
            rows += (c != 0);
        }
        p.col_digits[j] = d;
        atomicAdd(&s_d0, d);
        atomicMax(&s_colcap, d + n_in);
        atomicMax(&s_dcolmax, d);
        atomicMax(&s_rowsmax, rows);
    }
    __syncthreads();
    if (tid == 0) {
        p.prep_meta[PM_NBITS] = N;
        p.prep_meta[PM_D0] = s_d0;
        p.prep_meta[PM_COLCAP] = s_colcap;
        p.prep_meta[PM_DCOL_MAX] = s_dcolmax;
        p.prep_meta[PM_ROWS_MAX] = s_rowsmax;
    }
}



} // namespace da
