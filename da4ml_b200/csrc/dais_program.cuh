// dais_program.cuh -- host side of the DAIS interpreter: parse, validate and levelise a program (plain C++, no CUDA, so
// the CPU tests compile it with g++ next to the evaluator of dais_replay.cuh).
//
// Everything that does not depend on the samples is checked here, before any device call, in the wording of the
// reference (DAISInterpreter.cc `load_from_binary` :10-91, `validate` :429-448, and the data-independent throws of
// `exec_ops` :291-388).  On top of that, what the reference indexes unchecked is checked too, so that a foreign file
// cannot make the device read outside its buffers: operand ids that are negative or out of range, table indices past
// n_tables, negative table sizes, out-of-range output indices, input ids and input / output shifts.
#pragma once
#include "dais_replay.cuh"

#include <algorithm>
#include <stdexcept>
#include <string>
#include <vector>

namespace da {

struct DaisProgramHost {
    int32_t n_in = 0, n_out = 0, n_ops = 0, n_tables = 0;
    std::vector<int32_t> header;        // inp_shifts[n_in], out_idxs[n_out], out_shifts[n_out], out_negs[n_out]
    std::vector<DaisOp> ops;
    std::vector<int32_t> tables;        // all lookup tables, concatenated
    std::vector<long long> table_off;   // [n_tables + 1] start of each table in `tables`
    std::vector<int> order, lvl_begin;  // ops sorted by level; level l is order[lvl_begin[l] .. lvl_begin[l + 1])
    std::vector<char> lvl_adder;        // level l holds input loads and shift-adds only
    int n_levels = 0, max_width = 0;
    bool has_lookup = false;

    const int32_t *inp_shifts() const { return header.data(); }
    const int32_t *out_idxs() const { return header.data() + n_in; }
    const int32_t *out_shifts() const { return header.data() + n_in + n_out; }
    const int32_t *out_negs() const { return header.data() + n_in + 2 * n_out; }
};

[[noreturn]] inline void dais_fail(const std::string &msg) { throw std::runtime_error(msg); }

// Header, size and the table block (load_from_binary :10-78), plus the index / shift ranges of the header arrays.
inline void dais_parse(const int32_t *w, int64_t n_words, DaisProgramHost &p) {
    if (!w || n_words < 6)
        dais_fail("Binary data too small to contain valid DAIS model file");
    if (w[0] != 1)
        dais_fail("DAIS version mismatch: expected version 1, got version " + std::to_string(w[0]));
    p.n_in = w[2];
    p.n_out = w[3];
    p.n_ops = w[4];
    p.n_tables = w[5];
    if (p.n_in < 0 || p.n_out < 0 || p.n_ops < 0 || p.n_tables < 0)
        dais_fail("Binary data header holds a negative count");
    const int64_t table_offset = 6 + (int64_t)p.n_in + 3LL * p.n_out + 8LL * p.n_ops;
    int64_t expect = table_offset;
    for (int64_t t = 0; t < p.n_tables; ++t) {
        if (table_offset + t >= n_words) { // the size words themselves are missing
            expect += p.n_tables - t;
            break;
        }
        const int32_t size = w[table_offset + t];
        if (size < 0)
            dais_fail("Lookup table " + std::to_string(t) + " has a negative size (" + std::to_string(size) + ")");
        expect += 1 + (int64_t)size;
    }
    if (expect != n_words)
        dais_fail("Binary data size mismatch: expected " + std::to_string(expect * 4) + " bytes , got " + std::to_string(n_words * 4) + " bytes");
    p.header.assign(w + 6, w + 6 + p.n_in + 3LL * p.n_out);
    p.ops.resize(p.n_ops);
    if (p.n_ops)
        memcpy(p.ops.data(), w + 6 + p.n_in + 3LL * p.n_out, sizeof(DaisOp) * p.n_ops);
    p.table_off.assign(p.n_tables + 1, 0);
    for (int32_t t = 0; t < p.n_tables; ++t)
        p.table_off[t + 1] = p.table_off[t] + w[table_offset + t];
    p.tables.assign(w + table_offset + p.n_tables, w + n_words);
    for (int i = 0; i < p.n_out; ++i)
        if (p.out_idxs()[i] < -1 || p.out_idxs()[i] >= p.n_ops)
            dais_fail("output index out of range at output " + std::to_string(i));
    for (int i = 0; i < p.n_in; ++i)
        if (p.inp_shifts()[i] < -1023 || p.inp_shifts()[i] > 1023)
            dais_fail("input shift out of range at input " + std::to_string(i));
    for (int i = 0; i < p.n_out; ++i)
        if (p.out_shifts()[i] < -1023 || p.out_shifts()[i] > 1023)
            dais_fail("output shift out of range at output " + std::to_string(i));
}

// Causality (validate :429-448), then, op by op in program order, what exec_ops throws whatever the data (unknown opcode,
// msb_mux shift configuration, bit-op kinds) together with the operand checks the reference leaves out.
inline void dais_validate(const DaisProgramHost &p) {
    const std::vector<DaisOp> &ops = p.ops;
    for (int i = 0; i < p.n_ops; ++i) {
        const DaisOp &op = ops[i];
        if (op.id0 >= i && op.opcode != -1)
            dais_fail("Operation " + std::to_string(i) + " has id0=" + std::to_string(op.id0) + "violating causality");
        if (op.id1 >= i)
            dais_fail("Operation " + std::to_string(i) + " has id1=" + std::to_string(op.id1) + " violating causality");
        if ((op.opcode == 6 || op.opcode == -6) && (op.data_low < 0 || op.data_low >= i))
            dais_fail("Operation " + std::to_string(i) + " has cond_idx=" + std::to_string(op.data_low) + " violating causality");
    }
    for (int i = 0; i < p.n_ops; ++i) {
        const DaisOp &op = ops[i];
        const int opc = op.opcode;
        const std::string at = std::to_string(i);
        if (opc < -10 || opc > 10 || opc == -4 || opc == -5 || opc == -7 || opc == -8 || opc == -10)
            dais_fail("Unknown opcode: " + std::to_string(opc) + " at index " + at);
        if (opc == -1 && (op.id0 < 0 || op.id0 >= p.n_in))
            dais_fail("input index out of range at operation " + at);
        if (dais_reads_id0(opc) && op.id0 < 0)
            dais_fail("Operation " + at + " has id0=" + std::to_string(op.id0) + " out of range");
        if (dais_reads_id1(opc) && op.id1 < 0)
            dais_fail("Operation " + at + " has id1=" + std::to_string(op.id1) + " out of range");
        if (opc == 6 || opc == -6) {
            const int32_t shift1 = dais_add32(dais_sub32(op.fractionals, ops[op.id1].fractionals), op.data_high);
            const int32_t shift0 = dais_sub32(op.fractionals, ops[op.id0].fractionals);
            if (shift1 != 0 && shift0 != 0)
                dais_fail("Unsupported msb_mux shift configuration: shift0=" + std::to_string(shift0) + ", shift1=" + std::to_string(shift1));
        }
        if (opc == 8 && (op.data_low < 0 || op.data_low >= p.n_tables))
            dais_fail("Operation " + at + " has table index " + std::to_string(op.data_low) + " out of range (" + std::to_string(p.n_tables) + " tables)");
        if ((opc == 9 || opc == -9) && (op.data_low < 0 || op.data_low > 2))
            dais_fail("Unknown bit unary operation with data_low=" + std::to_string(op.data_low));
        if (opc == 10 && ((op.data_high >> 24) < 0 || (op.data_high >> 24) > 2))
            dais_fail("Unknown bit binary operation with data_low=" + std::to_string(op.data_low));
    }
}

// Levels: inputs and constants at 0, every other op 1 + the highest level among the ops it reads (the mux condition
// included).  Also the largest op width and whether any op looks a table up.
inline void dais_levelise(DaisProgramHost &p) {
    std::vector<int> level(p.n_ops, 0);
    p.n_levels = p.n_ops ? 1 : 0;
    p.max_width = 0;
    p.has_lookup = false;
    for (int i = 0; i < p.n_ops; ++i) {
        const DaisOp &op = p.ops[i];
        p.max_width = std::max(p.max_width, (int)dais_width(op));
        p.has_lookup |= op.opcode == 8;
        if (!dais_reads_id0(op.opcode))
            continue;
        int l = level[op.id0];
        if (dais_reads_id1(op.opcode))
            l = std::max(l, level[op.id1]);
        if (dais_reads_cond(op.opcode))
            l = std::max(l, level[op.data_low]);
        level[i] = l + 1;
        p.n_levels = std::max(p.n_levels, level[i] + 1);
    }
    p.lvl_begin.assign(p.n_levels + 1, 0);
    p.order.resize(p.n_ops);
    for (int i = 0; i < p.n_ops; ++i)
        p.lvl_begin[level[i] + 1]++;
    for (int l = 0; l < p.n_levels; ++l)
        p.lvl_begin[l + 1] += p.lvl_begin[l];
    std::vector<int> fill(p.lvl_begin.begin(), p.lvl_begin.end() - 1);
    for (int i = 0; i < p.n_ops; ++i)
        p.order[fill[level[i]]++] = i;
    p.lvl_adder.assign(p.n_levels, 1);
    for (int i = 0; i < p.n_ops; ++i)
        if (p.ops[i].opcode < -1 || p.ops[i].opcode > 1)
            p.lvl_adder[level[i]] = 0;
}

// The reference's message for a lookup index out of range (logic_lookup :228-235), from the operand value v0.
inline std::string dais_lookup_error(const DaisProgramHost &p, int op_index, int64_t v0) {
    const DaisOp &op = p.ops[op_index];
    const DaisOp &o0 = p.ops[op.id0];
    const int64_t zero = dais_mul((int64_t)(int32_t)(0u - (uint32_t)o0.is_signed), dais_pow2_i64(dais_sub32(dais_width(o0), 1)));
    const int64_t index = dais_sub(dais_sub(v0, zero), (int64_t)op.data_high);
    const long long size = p.table_off[op.data_low + 1] - p.table_off[op.data_low];
    return "Logic lookup index out of bounds: index=" + std::to_string(index) + ", table_size=" + std::to_string(size) + ", zero=" + std::to_string(zero) +
           ", data_high=" + std::to_string(op.data_high) + ", v0=" + std::to_string(v0);
}

} // namespace da
