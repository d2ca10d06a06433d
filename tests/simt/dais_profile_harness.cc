// dais_profile_harness.cc -- TEST INFRASTRUCTURE ONLY.  The product's DAIS evaluator (da4ml_b200/csrc/dais_replay.cuh,
// `dais_eval`) and host checks (dais_program.cuh) compiled with g++, driven sample by sample and op by op in program
// order as in dais_eval_harness.cc, reporting the op codes themselves instead of the program's outputs: per-op
// statistics (`dp_profile`) and the codes of selected ops (`dp_dump`), for the CPU tests of DaisProgram.profile / dump.
#include "../../da4ml_b200/csrc/dais_program.cuh"

static thread_local std::string g_err;

// Evaluate every op of every sample in program order; after each sample, `emit(s, p, buf)` reads the op codes.
template <class Emit> static int replay(const int32_t *words, int64_t n_words, const double *inputs, int64_t n_samples, Emit &&emit) {
    try {
        da::DaisProgramHost p;
        da::dais_parse(words, n_words, p);
        da::dais_validate(p);
        da::dais_levelise(p);
        std::vector<int64_t> buf(p.n_ops);
        for (int64_t s = 0; s < n_samples; ++s) {
            const double *x = inputs + s * p.n_in;
            for (int i = 0; i < p.n_ops; ++i) {
                const da::DaisOp &op = p.ops[i];
                const int opc = op.opcode;
                const da::DaisOp &o0 = da::dais_reads_id0(opc) ? p.ops[op.id0] : op;
                const da::DaisOp &o1 = da::dais_reads_id1(opc) ? p.ops[op.id1] : op;
                const da::DaisOp &oc = da::dais_reads_cond(opc) ? p.ops[op.data_low] : op;
                const int32_t *table = nullptr;
                long long table_size = 0;
                if (opc == 8) {
                    table = p.tables.data() + p.table_off[op.data_low];
                    table_size = p.table_off[op.data_low + 1] - p.table_off[op.data_low];
                }
                bool oob = false;
                buf[i] = da::dais_eval(
                    op, o0, o1, oc, da::dais_reads_id0(opc) ? buf[op.id0] : 0, da::dais_reads_id1(opc) ? buf[op.id1] : 0,
                    da::dais_reads_cond(opc) ? buf[op.data_low] : 0, opc == -1 ? x[op.id0] : 0.0, opc == -1 ? p.inp_shifts()[op.id0] : 0, table, table_size, &oob
                );
                if (oob)
                    throw std::runtime_error(da::dais_lookup_error(p, i, buf[op.id0]));
            }
            emit(s, p, buf);
        }
        return 0;
    }
    catch (const std::exception &e) {
        g_err = e.what();
        return 1;
    }
}

extern "C" {
const char *dp_last_error() { return g_err.c_str(); }

// stats [n_ops][3] = {min, max, bitwise OR} of each op's codes over the samples; the caller initialises it (identity
// INT64_MAX, INT64_MIN, 0), so successive calls accumulate.
int dp_profile(const int32_t *words, int64_t n_words, const double *inputs, int64_t n_samples, int64_t *stats) {
    return replay(words, n_words, inputs, n_samples, [&](int64_t, const da::DaisProgramHost &p, const std::vector<int64_t> &buf) {
        for (int i = 0; i < p.n_ops; ++i) {
            stats[3 * i] = std::min(stats[3 * i], buf[i]);
            stats[3 * i + 1] = std::max(stats[3 * i + 1], buf[i]);
            stats[3 * i + 2] |= buf[i];
        }
    });
}

// values [n_samples][n_sel] = codes of ops op_ids[0..n_sel) (ids checked by the caller)
int dp_dump(const int32_t *words, int64_t n_words, const double *inputs, int64_t n_samples, const int32_t *op_ids, int64_t n_sel, int64_t *values) {
    return replay(words, n_words, inputs, n_samples, [&](int64_t s, const da::DaisProgramHost &, const std::vector<int64_t> &buf) {
        for (int64_t k = 0; k < n_sel; ++k)
            values[s * n_sel + k] = buf[op_ids[k]];
    });
}
}
