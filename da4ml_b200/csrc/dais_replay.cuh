// dais_replay.cuh -- the DAIS interpreter on the device (SURVEY.md section 8f, N2).
//
// Bit-exact port of the reference interpreter's op evaluation (reference src/da4ml/_binary/dais/DAISInterpreter.cc,
// `exec_ops` :291-388) for the whole opcode set: input load (-1), shift-add (0/1), relu (+-2), quantize (+-3), constant
// add (4), constant (5), MSB mux (+-6), multiply (7), lookup (8), bit unary (+-9) and bit binary (10); output scaling as
// `inference` :390-401.  Programs are the int32 words written by CombLogic.to_binary (reference types.py:500-541).
//
// The target is the reference's compiled x86-64 object code, including where its C++ is undefined:
//  - every shift masks its count the way x86 `shl`/`sar` do (5 bits for int32, 6 bits for int64); PTX shifts clamp
//    instead, so the masks below are explicit;
//  - int64 arithmetic wraps (two's complement), int32 arithmetic on the dtype fields wraps too;
//  - a double -> int64 conversion of NaN or an out-of-range value gives INT64_MIN (`cvttsd2si`), where PTX saturates;
//  - std::pow(2.0, e) of an integer is exact, so it is built from the exponent bits.
// dais_eval is the single definition of an op's value; it is __host__ __device__ so the CPU tests compile the same
// source with g++ (tests/simt/dais_eval_harness.cc).  The kernels below are thin loops around it (levels made of input
// loads and shift-adds only call its dais_input / dais_shift_add directly).
//
// Ops are levelised on the host (an op's level = 1 + max level of the ops it reads; inputs and constants sit at level
// 0); one launch per level, thread = (op of the level, sample) with the sample index fastest, so all buffer traffic is
// coalesced and a warp executes one opcode: the kernel family is plain HBM-bound streaming.
#pragma once
#include <climits>
#include <cmath>
#include <cstdint>
#include <cstring>

#ifdef __CUDACC__
#include <cuda_runtime.h>
#define DAIS_HD __host__ __device__ __forceinline__
#else
#define DAIS_HD inline
#endif

namespace da {

struct DaisOp { // layout of the reference's dais::Op (DAISInterpreter.hh:46-53)
    int32_t opcode, id0, id1, data_low, data_high;
    int32_t is_signed, integers, fractionals;
};

// wrapping int32 / int64 arithmetic (the reference's compiled code wraps; signed overflow is undefined in C++)
DAIS_HD int32_t dais_add32(int32_t a, int32_t b) { return (int32_t)((uint32_t)a + (uint32_t)b); }
DAIS_HD int32_t dais_sub32(int32_t a, int32_t b) { return (int32_t)((uint32_t)a - (uint32_t)b); }
DAIS_HD int64_t dais_add(int64_t a, int64_t b) { return (int64_t)((uint64_t)a + (uint64_t)b); }
DAIS_HD int64_t dais_sub(int64_t a, int64_t b) { return (int64_t)((uint64_t)a - (uint64_t)b); }
DAIS_HD int64_t dais_mul(int64_t a, int64_t b) { return (int64_t)((uint64_t)a * (uint64_t)b); }
DAIS_HD int64_t dais_neg(int64_t a) { return (int64_t)(0ull - (uint64_t)a); }
// x86 shifts: the count is taken modulo the operand width
DAIS_HD int64_t dais_shl(int64_t v, int32_t c) { return (int64_t)((uint64_t)v << (c & 63)); }
DAIS_HD int64_t dais_sar(int64_t v, int32_t c) { return v >> (c & 63); }
DAIS_HD int64_t dais_pow2_i64(int32_t c) { return (int64_t)(1ull << (c & 63)); } // 1LL << c

DAIS_HD int32_t dais_width(const DaisOp &o) { return dais_add32(dais_add32(o.integers, o.fractionals), o.is_signed ? 1 : 0); }

// std::pow(2.0, e) for an integer e: exact, subnormals included; 0 below 2^-1074, inf above 2^1023
DAIS_HD double dais_pow2(int32_t e) {
    if (e > 1023)
        return HUGE_VAL;
    if (e < -1074)
        return 0.0;
    const uint64_t bits = e >= -1022 ? (uint64_t)(e + 1023) << 52 : 1ull << (e + 1074);
    double d;
    memcpy(&d, &bits, sizeof(d));
    return d;
}

// static_cast<int64_t>(double) as x86 `cvttsd2si` executes it: NaN and out-of-range values give INT64_MIN
DAIS_HD int64_t dais_f2i(double y) { return (y >= -9223372036854775808.0 && y < 9223372036854775808.0) ? (int64_t)y : LLONG_MIN; }

// DAISInterpreter::quantize (:139-152): shift from f_from to the op's fractionals, then wrap into its range
DAIS_HD int64_t dais_quantize(int64_t value, int32_t f_from, const DaisOp &to) {
    value = dais_sar(value, dais_sub32(f_from, to.fractionals));
    const int32_t w = dais_width(to);
    const int64_t int_min = to.is_signed ? (int64_t)(int32_t)(0u - (1u << (dais_sub32(w, 1) & 31))) : 0; // DType::int_min, int32
    const int64_t mod = dais_pow2_i64(w);
    const int64_t av = value < 0 ? dais_neg(value) : value; // std::abs
    return dais_add(dais_add(dais_sub(value, int_min), dais_mul(dais_add(av / mod, 1), mod)) % mod, int_min);
}

// DAISInterpreter::get_msb (:177-181)
DAIS_HD bool dais_msb(int64_t v, const DaisOp &d) {
    if (d.is_signed)
        return v < 0;
    const int64_t t = dais_pow2_i64(dais_sub32(dais_width(d), 2));
    return v > (t > 0 ? t : 0);
}

// 64-bit constant of opcodes 4 / 5: data_high:data_low
DAIS_HD int64_t dais_const64(const DaisOp &op) { return (int64_t)(((uint64_t)(uint32_t)op.data_high << 32) | (uint32_t)op.data_low); }

// opcode -1 (:305-312): input x scaled by 2^(inp_shift + f), floored, wrapped into the op's range
DAIS_HD int64_t dais_input(const DaisOp &op, double x, int32_t inp_shift) {
    const int64_t v = dais_f2i(floor(x * dais_pow2(dais_add32(inp_shift, op.fractionals))));
    return dais_quantize(v, op.fractionals, op);
}

// opcodes 0 / 1, shift_add (:114-137); f0 / f1 are the fractionals of the operands
DAIS_HD int64_t dais_shift_add(const DaisOp &op, int32_t f0, int32_t f1, int64_t v0, int64_t v1) {
    const int32_t shift = op.data_low;
    const int32_t actual = dais_sub32(dais_add32(shift, f0), f1);
    const int64_t b = op.opcode == 1 ? dais_neg(v1) : v1;
    int64_t r = actual > 0 ? dais_add(v0, dais_shl(b, actual)) : dais_add(dais_shl(v0, dais_sub32(0, actual)), b);
    const int32_t c = dais_sub32(f1, shift);
    const int32_t gshift = dais_sub32(f0 > c ? f0 : c, op.fractionals);
    if (gshift > 0)
        r = dais_sar(r, gshift);
    return r;
}

// Value of op `op` for one sample.  o0 / o1 / oc are the ops named by id0 / id1 / the mux condition, v0 / v1 / vc their
// values (only those the opcode reads are meaningful); x is the input sample value of opcode -1 and inp_shift its
// input's shift; table / table_size the lookup table of opcode 8.  A lookup index out of range sets *oob, and the
// returned value then comes from the clamped index (so nothing outside the table is read).
DAIS_HD int64_t dais_eval(
    const DaisOp &op, const DaisOp &o0, const DaisOp &o1, const DaisOp &oc, int64_t v0, int64_t v1, int64_t vc, double x, int32_t inp_shift,
    const int32_t *table, int64_t table_size, bool *oob
) {
    switch (op.opcode) {
    case -1:
        return dais_input(op, x, inp_shift);
    case 0:
    case 1:
        return dais_shift_add(op, o0.fractionals, o1.fractionals, v0, v1);
    case 2:
    case -2: { // relu :154-162
        const int64_t v = op.opcode == -2 ? dais_neg(v0) : v0;
        return v < 0 ? 0 : dais_quantize(v, o0.fractionals, op);
    }
    case 3:
    case -3: // quantize
        return dais_quantize(op.opcode == -3 ? dais_neg(v0) : v0, o0.fractionals, op);
    case 4: // const_add :164-175
        return dais_add(dais_shl(v0, dais_sub32(op.fractionals, o0.fractionals)), dais_const64(op));
    case 5:
        return dais_const64(op);
    case 6:
    case -6: { // msb_mux :183-215 (the shift configuration is checked on the host; the quantize shift is 0)
        const int32_t shift1 = dais_add32(dais_sub32(op.fractionals, o1.fractionals), op.data_high);
        const int32_t shift0 = dais_sub32(op.fractionals, o0.fractionals);
        const int64_t r = dais_msb(vc, oc) ? dais_shl(v0, shift0) : dais_shl(op.opcode == -6 ? dais_neg(v1) : v1, shift1);
        return dais_quantize(r, op.fractionals, op);
    }
    case 7:
        return dais_mul(v0, v1);
    case 8: { // logic_lookup :217-237
        const int64_t zero = dais_mul((int64_t)(int32_t)(0u - (uint32_t)o0.is_signed), dais_pow2_i64(dais_sub32(dais_width(o0), 1)));
        int64_t index = dais_sub(dais_sub(v0, zero), (int64_t)op.data_high);
        if (index < 0 || index >= table_size) {
            *oob = true;
            if (table_size <= 0)
                return 0;
            index = index < 0 ? 0 : table_size - 1;
        }
#ifdef __CUDA_ARCH__
        return (int64_t)__ldg(table + index);
#else
        return (int64_t)table[index];
#endif
    }
    case 9:
    case -9: { // bit_unary :239-258 (unknown kinds are rejected on the host)
        const int64_t v = op.opcode == -9 ? dais_neg(v0) : v0;
        const int64_t mask = dais_sub(dais_pow2_i64(dais_width(o0)), 1);
        if (op.data_low == 0)
            return op.is_signed ? ~v : (~v & mask);
        if (op.data_low == 1)
            return v != 0;
        return (v & mask) == mask;
    }
    case 10: { // bit_binary :260-289
        const int32_t actual = dais_sub32(dais_add32(op.data_low, o0.fractionals), o1.fractionals);
        int64_t a = op.data_high & 1 ? dais_neg(v0) : v0;
        int64_t b = op.data_high & 2 ? dais_neg(v1) : v1;
        if (actual > 0)
            b = dais_shl(b, actual);
        else
            a = dais_shl(a, dais_sub32(0, actual));
        const int32_t kind = op.data_high >> 24;
        return kind == 0 ? (a & b) : kind == 1 ? (a | b) : (a ^ b);
    }
    default: // unknown opcodes are rejected on the host
        return 0;
    }
}

// inference :394-400: double(+-v) * 2^(out_shift - f); an output without an op (index -1) is 0
DAIS_HD double dais_output(int64_t v, int32_t neg, int32_t out_shift, int32_t fractionals) {
    return (double)(neg ? dais_neg(v) : v) * dais_pow2(dais_sub32(out_shift, fractionals));
}

// Opcodes whose operand fields name earlier ops (the program's checks are in dais_program.cuh).
DAIS_HD bool dais_reads_id0(int32_t opc) { return opc != -1 && opc != 5; }
DAIS_HD bool dais_reads_id1(int32_t opc) { return opc == 0 || opc == 1 || opc == 6 || opc == -6 || opc == 7 || opc == 10; }
DAIS_HD bool dais_reads_cond(int32_t opc) { return opc == 6 || opc == -6; }

#ifdef __CUDACC__
// Key of a failing lookup: the first (sample, op) in program order is the smallest key.
__device__ __forceinline__ unsigned long long dais_err_key(long long s, int i) { return ((unsigned long long)s << 32) | (unsigned)i; }

// buffer layout: [n_ops][S] int64, S = samples of the current chunk.  inputs: [S][n_in] float64 of the chunk.
// kAdder: every op of the level is an input load or a shift-add (the whole of a CMVM program): this instantiation
// carries none of the other opcodes' state and runs at the register count (and occupancy) of a plain adder replay.
template <bool kAdder>
__global__ void __launch_bounds__(256) dais_level_kernel(
    const DaisOp *__restrict__ ops, const int *__restrict__ order, int n_level_ops, const int *__restrict__ inp_shifts, const double *__restrict__ inputs,
    int n_in, long long S, long long *buffer, const int32_t *__restrict__ tables, const long long *__restrict__ table_off, unsigned long long *err
) {
    const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (tid >= (long long)n_level_ops * S)
        return;
    const int k = (int)(tid / S);
    const long long s = tid - (long long)k * S;
    const int i = order[k];
    const DaisOp op = ops[i];
    const int opc = op.opcode;
    if (kAdder) {
        buffer[(long long)i * S + s] = opc == -1 ? dais_input(op, inputs[s * n_in + op.id0], inp_shifts[op.id0])
                                                 : dais_shift_add(op, ops[op.id0].fractionals, ops[op.id1].fractionals, buffer[(long long)op.id0 * S + s],
                                                                  buffer[(long long)op.id1 * S + s]);
        return;
    }
    DaisOp o0 = op, o1 = op, oc = op;
    long long v0 = 0, v1 = 0, vc = 0;
    double x = 0.0;
    int inp_shift = 0;
    const int32_t *table = nullptr;
    long long table_size = 0;
    if (opc == -1) {
        x = inputs[s * n_in + op.id0];
        inp_shift = inp_shifts[op.id0];
    }
    else if (dais_reads_id0(opc)) {
        o0 = ops[op.id0];
        v0 = buffer[(long long)op.id0 * S + s];
        if (dais_reads_id1(opc)) {
            o1 = ops[op.id1];
            v1 = buffer[(long long)op.id1 * S + s];
        }
        if (dais_reads_cond(opc)) {
            oc = ops[op.data_low];
            vc = buffer[(long long)op.data_low * S + s];
        }
        if (opc == 8) {
            const long long t0 = table_off[op.data_low];
            table = tables + t0;
            table_size = table_off[op.data_low + 1] - t0;
        }
    }
    bool oob = false;
    buffer[(long long)i * S + s] = dais_eval(op, o0, o1, oc, v0, v1, vc, x, inp_shift, table, table_size, &oob);
    if (oob)
        atomicMin(err, dais_err_key(s, i));
}

__global__ void __launch_bounds__(256) dais_output_kernel(
    const DaisOp *__restrict__ ops, const int *__restrict__ out_idxs, const int *__restrict__ out_shifts, const int *__restrict__ out_negs, int n_out,
    long long S, const long long *__restrict__ buffer, double *__restrict__ outputs
) {
    const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (tid >= (long long)n_out * S)
        return;
    const int o = (int)(tid / S);
    const long long s = tid - (long long)o * S;
    const int idx = out_idxs[o];
    outputs[s * n_out + o] = idx >= 0 ? dais_output(buffer[(long long)idx * S + s], out_negs[o], out_shifts[o], ops[idx].fractionals) : 0.0;
}

// ---- op profiling: per-op statistics and dumps of the codes in the buffer, after a chunk's last level ----------------
// stats: [n_ops][3] int64 = {min, max, bitwise OR} of each op's codes, folded over every chunk of a call.
__global__ void dais_stats_init_kernel(long long *stats, int n_ops) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_ops)
        return;
    stats[3LL * i] = LLONG_MAX;
    stats[3LL * i + 1] = LLONG_MIN;
    stats[3LL * i + 2] = 0;
}

// grid (n_ops, sample blocks): each block reduces a slice of one op's row (contiguous, so the loads are coalesced) with
// warp shuffles and shared memory, then folds it into the op's accumulators with one atomic per statistic.
constexpr int kDaisStatsThreads = 256, kDaisStatsPerThread = 8;
__global__ void __launch_bounds__(kDaisStatsThreads) dais_stats_kernel(const long long *__restrict__ buffer, long long S, long long *stats) {
    const int i = blockIdx.x;
    const long long *row = buffer + (long long)i * S;
    long long mn = LLONG_MAX, mx = LLONG_MIN;
    unsigned long long bits = 0;
    constexpr long long kSpan = (long long)kDaisStatsThreads * kDaisStatsPerThread; // samples per block and pass
    for (long long s0 = (long long)blockIdx.y * kSpan + threadIdx.x; s0 < S; s0 += (long long)gridDim.y * kSpan) {
        long long v[kDaisStatsPerThread]; // all loads issued before any is used
#pragma unroll
        for (int k = 0; k < kDaisStatsPerThread; ++k) {
            const long long s = s0 + (long long)k * kDaisStatsThreads;
            v[k] = s < S ? __ldg(row + s) : row[s0];
        }
#pragma unroll
        for (int k = 0; k < kDaisStatsPerThread; ++k) {
            mn = min(mn, v[k]);
            mx = max(mx, v[k]);
            bits |= (unsigned long long)v[k];
        }
    }
    for (int off = 16; off > 0; off >>= 1) {
        mn = min(mn, __shfl_xor_sync(0xffffffffu, mn, off));
        mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, off));
        bits |= __shfl_xor_sync(0xffffffffu, bits, off);
    }
    __shared__ long long s_mn[kDaisStatsThreads / 32], s_mx[kDaisStatsThreads / 32];
    __shared__ unsigned long long s_bits[kDaisStatsThreads / 32];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) {
        s_mn[warp] = mn;
        s_mx[warp] = mx;
        s_bits[warp] = bits;
    }
    __syncthreads();
    if (warp)
        return;
    const bool live = lane < kDaisStatsThreads / 32;
    mn = live ? s_mn[lane] : LLONG_MAX;
    mx = live ? s_mx[lane] : LLONG_MIN;
    bits = live ? s_bits[lane] : 0;
    for (int off = kDaisStatsThreads / 64; off > 0; off >>= 1) {
        mn = min(mn, __shfl_xor_sync(0xffffffffu, mn, off));
        mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, off));
        bits |= __shfl_xor_sync(0xffffffffu, bits, off);
    }
    if (lane == 0) {
        long long *st = stats + 3LL * i;
        atomicMin(st, mn);
        atomicMax(st + 1, mx);
        atomicOr((unsigned long long *)(st + 2), bits);
    }
}

// values [S][n_sel] = codes of ops sel[0..n_sel) for the S samples of the chunk.  Block (32, 8), one 32-sample x 32-op
// tile at a time through shared memory: the reads run along the buffer's rows (samples), the writes along the output's
// rows (selected ops), so both are coalesced.  grid.x covers the samples, grid.y strides over the tiles of ops.
__global__ void __launch_bounds__(256) dais_dump_kernel(
    const long long *__restrict__ buffer, long long S, const int *__restrict__ sel, long long n_sel, long long *__restrict__ values
) {
    __shared__ long long tile[32][33]; // (+1 column: the transposed reads hit distinct banks)
    const long long s0 = (long long)blockIdx.x * 32;
    const long long n_tiles = (n_sel + 31) / 32;
    for (long long jt = blockIdx.y; jt < n_tiles; jt += gridDim.y) {
        const long long j0 = jt * 32;
        for (int r = threadIdx.y; r < 32; r += 8) {
            const long long j = j0 + r, s = s0 + threadIdx.x;
            if (j < n_sel && s < S)
                tile[r][threadIdx.x] = buffer[(long long)sel[j] * S + s];
        }
        __syncthreads();
        for (int r = threadIdx.y; r < 32; r += 8) {
            const long long j = j0 + threadIdx.x, s = s0 + r;
            if (j < n_sel && s < S)
                values[s * n_sel + j] = tile[threadIdx.x][r];
        }
        __syncthreads();
    }
}
#endif

} // namespace da
