// dais_eval_harness.cc -- TEST INFRASTRUCTURE ONLY.  The product's DAIS evaluator (da4ml_b200/csrc/dais_replay.cuh,
// `dais_eval`) and host checks (dais_program.cuh) compiled with g++, driven sample by sample and op by op in program
// order the way the reference interpreter runs (DAISInterpreter.cc exec_ops), so the CPU tests can compare the
// evaluator's arithmetic and messages with stored reference answers without a GPU.
#include "../../da4ml_b200/csrc/dais_program.cuh"

static thread_local std::string g_err;

extern "C" {
const char *dh_last_error() { return g_err.c_str(); }

int dh_run(const int32_t *words, int64_t n_words, const double *inputs, int64_t n_samples, double *outputs) {
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
            for (int o = 0; o < p.n_out; ++o) {
                const int idx = p.out_idxs()[o];
                outputs[s * p.n_out + o] = idx >= 0 ? da::dais_output(buf[idx], p.out_negs()[o], p.out_shifts()[o], p.ops[idx].fractionals) : 0.0;
            }
        }
        return 0;
    }
    catch (const std::exception &e) {
        g_err = e.what();
        return 1;
    }
}
}
