/* da4ml_b200_cmvm.h -- C ABI of the B200-native CMVM solver (libda4ml_b200_cmvm.so).
 *
 * Drop-in boundary for the reference's nanobind module `da4ml._binary.cmvm_bin`
 * (reference src/da4ml/_binary/cmvm/bindings.cc:227-263).  Each entry point names the reference
 * interface it replaces.  Plain pointers and sizes only; all arrays are host memory unless noted,
 * dense C order.  Every compute entry point runs on the current CUDA device (cudaSetDevice /
 * torch.cuda.set_device) on the stream set with da4ml_cmvm_set_stream (default: stream 0) and
 * returns 0 on success; on failure it returns a non-zero DA4ML_E_* code and
 * da4ml_cmvm_last_error() describes it.  There is no CPU fallback: without a usable CUDA device the
 * compute calls fail with DA4ML_E_CUDA.
 */
#ifndef DA4ML_B200_CMVM_H
#define DA4ML_B200_CMVM_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum {
    DA4ML_OK = 0,
    DA4ML_E_INVALID = 1, /* bad argument; reference raises ValueError / std::invalid_argument  */
    DA4ML_E_RUNTIME = 2, /* e.g. "Unknown method: ..." (cmvm_core.cc:63), reference RuntimeError */
    DA4ML_E_CUDA = 3,    /* CUDA runtime failure or no device                                    */
    DA4ML_E_CAPACITY = 4 /* internal buffer could not be grown                                  */
};

typedef struct da4ml_pipeline da4ml_pipeline_t; /* opaque result, mirrors PipelineResult (types.hh:164-166) */

/* Message of the last failure on the calling thread. */
const char *da4ml_cmvm_last_error(void);

/* Library / device information: writes {abi_version, cuda_device_count, sm_count, sm_major, sm_minor}. */
int da4ml_cmvm_device_info(int32_t out[5]);

/* Stream (cudaStream_t as void*) used for every subsequent launch and copy issued by this library. */
int da4ml_cmvm_set_stream(void *cuda_stream);

/* Tuning knob: CTAs cooperating on one problem (0 = automatic). */
int da4ml_cmvm_set_group_size(int ctas_per_problem);

/* Launch geometry the solver would choose for a set of solve_single jobs on `co_resident_ctas` CTAs (132 on an H100 SXM),
 * without touching a device.  jobs: [n][8] int64 = {n_in, n_out, nbits, csd_digits, max_digits_per_column,
 * column_list_bound, f_mul, list_mul}; out: [12] int64 = {ctas_per_problem, concurrent_groups, columns_per_cta (adder
 * trees), list_rows_in_shared_memory, log2_chunk, chunk_slots, segment_entries_per_cta, log2_pair_counters,
 * dynamic_shared_bytes, shared_budget_bytes, narrow_rows (6-byte list rows), spill_rows}.  The histogram segment of a
 * CTA is a pool of pages: log2_chunk is the page size, segment_entries_per_cta the pool, chunk_slots its pages + 2.
 * Diagnostic; the reference has no counterpart. */
int da4ml_cmvm_plan(const int64_t *jobs, int64_t n_jobs, int co_resident_ctas, int group_override, int64_t out[12]);

/* Free the large device / pinned work buffers the library caches between calls (re-grown on demand; function-local
 * scratch of the small helper entry points is kept). */
int da4ml_cmvm_release(void);

/* Exact work accounting (sum over iterations of the live histogram size, needed for the algorithmic-bytes
 * figure): when on, every iteration re-reads the whole histogram instead of only the pages whose cached
 * maximum was invalidated.  Results are identical; only the counters and the speed change.  Off by default;
 * implied by a trace request. */
int da4ml_cmvm_set_accounting(int on);
/* The decompose_dc candidates of one call often decompose to byte-identical stage matrices; a solve_single job is a
 * pure function of its inputs, so by default identical jobs are solved once and the result shared (identical output to
 * the reference, which solves each candidate separately).  0 switches the sharing off. */
int da4ml_cmvm_set_job_sharing(int on);
/* Test-only capacity squeeze, so that small problems and the test suite reach the solve kernel's spill, multi-pass,
 * compaction, overflow and retry paths on the device.  caps[8] (NULL resets; a value < 0 keeps the planner's) =
 * {segment_entries (histogram entries per CTA, at least 4 pages), list_rows (shared-memory rows per owner list; 0 = every
 * row spills), spill_rows (global-memory rows per owner list), hash_log (log2 of the pair-counter table, 8..13),
 * wide_rows (> 0: 12-byte list rows), expr_cap (expression ids beyond the inputs), cell_pool (cells per CTA), poison
 * (> 0: every buffer the driver does not clear is filled with 0xA5)}.  A value only lowers the planner's; the retry after
 * a capacity status raises it as it raises the planner's (segment x f_mul, spill rows and cells x list_mul / 2; expr_cap
 * is dropped with the full expression table), and the work buffers keep the planner's sizes.  All knobs < 0 (the
 * default) leave every launch unchanged.  Results are unchanged too: a squeeze only makes the solver take longer paths. */
int da4ml_cmvm_set_capacity_override(const int64_t caps[8]);

/* ---- solve -------------------------------------------------------------------------------------
 * Replaces `solve` (bindings.cc:184-225 -> api.cc:147-250).
 *   kernel       [n_in, n_out] float32
 *   method0/1    "mc" "mc-dc" "mc-pdc" "wmc" "wmc-dc" "wmc-pdc" "dummy"; method1 may be "auto"
 *   qintervals   [n_in, 3] (min, max, step) or NULL  -> (-128, 127, 1)      (api.cc:161-167)
 *   latencies    [n_in] or NULL                     -> 0                   (api.cc:168-174)
 * Result: two stages (CombLogicResult, types.hh:153-162).  Free with da4ml_pipeline_free.          */
int da4ml_cmvm_solve(
    const float *kernel, int64_t n_in, int64_t n_out, const char *method0, const char *method1,
    int hard_dc, int decompose_dc, const float *qintervals, const float *latencies, int adder_size,
    int carry_size, int search_all_decompose_dc, da4ml_pipeline_t **out
);

/* Seeded tie-breaks (this library's extension; the reference has seed 0 only).  Among histogram entries of equal selector
 * score the greedy selection takes the one whose (packed key ^ tb_mask(seed)) is largest, where the packed key is
 * (id1 << 36 | id0 << 8 | sub << 7 | shift + 64) and tb_mask(0) = 0, tb_mask(s) = splitmix64(s) & (2^36 - 1): id1 is never
 * masked.  Seed 0 is the reference's rule exactly, and another seed is an equally valid greedy run with a different graph.
 * The seed applies to the greedy loop of both stages of every decompose_dc try; the decomposition, the latency retries,
 * the adder trees and the argmin over the tries are unchanged.  da4ml_cmvm_solve is the case seed = 0. */
int da4ml_cmvm_solve_seeded(
    const float *kernel, int64_t n_in, int64_t n_out, const char *method0, const char *method1,
    int hard_dc, int decompose_dc, const float *qintervals, const float *latencies, int adder_size,
    int carry_size, int search_all_decompose_dc, uint64_t seed, da4ml_pipeline_t **out
);

/* Batched form of da4ml_cmvm_solve: n independent problems solved concurrently on one GPU (the
 * reference has no batch API; its caller loops, trace/fixed_variable_array.py:368-371).  Per-problem
 * arrays of pointers; qintervals[i] / latencies[i] (or the arrays themselves) may be NULL.        */
int da4ml_cmvm_solve_batch(
    int64_t n_problems, const float *const *kernels, const int64_t *n_in, const int64_t *n_out,
    const char *method0, const char *method1, int hard_dc, int decompose_dc,
    const float *const *qintervals, const float *const *latencies, int adder_size, int carry_size,
    int search_all_decompose_dc, da4ml_pipeline_t **out /* [n_problems] */
);

/* Same as da4ml_cmvm_solve_batch but kernels_dev[i] are DEVICE pointers ([n_in, n_out] float32, dense): the
 * constant matrices are already resident in HBM (qintervals / latencies stay small host arrays). */
int da4ml_cmvm_solve_batch_device(
    int64_t n_problems, const float *const *kernels_dev, const int64_t *n_in, const int64_t *n_out,
    const char *method0, const char *method1, int hard_dc, int decompose_dc,
    const float *const *qintervals, const float *const *latencies, int adder_size, int carry_size,
    int search_all_decompose_dc, da4ml_pipeline_t **out /* [n_problems] */
);

/* One CSE stage on its own: `solve_single` (cmvm_core.cc:227-237).  One-stage pipeline.  When
 * trace_cap > 0, trace receives up to trace_cap rows of (id0, id1, shift, sub, |F|) per greedy
 * iteration (the reference's loop cmvm_core.cc:36-70) for step-level parity checks.              */
int da4ml_cmvm_solve_single(
    const float *kernel, int64_t n_in, int64_t n_out, const char *method, const float *qintervals,
    const float *latencies, int adder_size, int carry_size, int32_t *trace, int64_t trace_cap,
    da4ml_pipeline_t **out
);
/* The same under a tie-break seed (see da4ml_cmvm_solve_seeded); the trace reports the pairs the seeded run chose.
 * da4ml_cmvm_solve_single is the case seed = 0. */
int da4ml_cmvm_solve_single_seeded(
    const float *kernel, int64_t n_in, int64_t n_out, const char *method, const float *qintervals,
    const float *latencies, int adder_size, int carry_size, int32_t *trace, int64_t trace_cap, uint64_t seed,
    da4ml_pipeline_t **out
);

/* ---- sweep: one matrix under many option sets (the reference has no counterpart; its caller calls solve once per set) --
 * Option set s is {method0[s], method1[s], hard_dc[s], decompose_dc[s], search_all[s]}; the matrix, qintervals /
 * latencies (NULL -> defaults, as for da4ml_cmvm_solve) and the cost model (adder_size, carry_size) are shared.  Each set
 * expands into candidates as solve expands it (api.cc:176-201): with search_all, one per d in -1 .. min(H, ceil(log2
 * n_in)) with H = hard_dc (1e9 when hard_dc < 0), otherwise one with H = hard_dc, d = decompose_dc.  Candidate c is the
 * result of solve(kernel, method0, method1, H, d, search_all_decompose_dc = 0, ...) bit for bit; each set's winner (its
 * first candidate of minimum cost, api.cc:243-249) is the result of solve with the set itself.  Candidates are listed in
 * set order, then d order.  Candidates of different sets that start from the same state are solved once.  All jobs run
 * together, one launch per round.
 * The front: the candidates no other candidate dominates on (cost, latency_max), the first of exactly equal points only.
 * Op tables are kept for the winners and the front, or for every candidate with keep_all.  Arguments are checked on the
 * host before any device call (DA4ML_E_INVALID; an unknown method gives DA4ML_E_RUNTIME "Unknown method: ...").  If any
 * set fails as solve would fail, the call fails with that error and returns no result.  DA4ML_E_CAPACITY when the device
 * cannot hold the op tables of all jobs.  Free with da4ml_sweep_free. */
typedef struct da4ml_sweep da4ml_sweep_t; /* opaque sweep result */
int da4ml_cmvm_solve_sweep(
    const float *kernel, int64_t n_in, int64_t n_out, const float *qintervals, const float *latencies, int adder_size,
    int carry_size, int64_t n_sets, const char *const *method0, const char *const *method1, const int32_t *hard_dc,
    const int32_t *decompose_dc, const int32_t *search_all, int keep_all, da4ml_sweep_t **out
);
/* Many matrices under the same option sets in one GPU pass (a model's layers, say): every pending solve_single of every
 * candidate of every matrix runs in one launch per round.  Pointer arrays as for da4ml_cmvm_solve_batch; qintervals,
 * latencies or any entry of them may be NULL.  The option sets and the cost model are shared by the call, so costs of
 * different matrices can be summed.  out[p] is matrix p's result, exactly what da4ml_cmvm_solve_sweep returns for it
 * alone (candidates, winners, front and kept op tables within the matrix, n_solved of the matrix); its profile is the
 * whole call's.  Arguments are checked on the host before any device call and n_problems <= 0 gives DA4ML_E_INVALID.
 * If any set fails on any matrix, the call fails with that error and no out[p] is written.  da4ml_cmvm_solve_sweep is
 * the case n_problems = 1. */
int da4ml_cmvm_solve_sweep_batch(
    int64_t n_problems, const float *const *kernels, const int64_t *n_in, const int64_t *n_out, const float *const *qintervals,
    const float *const *latencies, int adder_size, int carry_size, int64_t n_sets, const char *const *method0,
    const char *const *method1, const int32_t *hard_dc, const int32_t *decompose_dc, const int32_t *search_all, int keep_all,
    da4ml_sweep_t **out /* [n_problems] */
);
/* The same with a tie-break seed per option set (seed[s], see da4ml_cmvm_solve_seeded; NULL = all 0).  Sets that differ
 * only in seed are distinct candidates; a candidate's seed is its set's.  Candidate c is the result of
 * da4ml_cmvm_solve_seeded(kernel, method0, method1, H, d, search_all_decompose_dc = 0, ..., seed[set]) bit for bit.
 * da4ml_cmvm_solve_sweep_batch is the case seed = NULL. */
int da4ml_cmvm_solve_sweep_batch_seeded(
    int64_t n_problems, const float *const *kernels, const int64_t *n_in, const int64_t *n_out, const float *const *qintervals,
    const float *const *latencies, int adder_size, int carry_size, int64_t n_sets, const char *const *method0,
    const char *const *method1, const int32_t *hard_dc, const int32_t *decompose_dc, const int32_t *search_all,
    const uint64_t *seed /* [n_sets] or NULL */, int keep_all, da4ml_sweep_t **out /* [n_problems] */
);
/* counts: {n_sets, n_candidates, n_kept (candidates with op tables), n_solved (distinct candidates solved)} */
int da4ml_sweep_counts(const da4ml_sweep_t *s, int64_t out[4]);
/* Profile of the sweep call, as da4ml_pipeline_profile: {device_ms, launches, solve_kernel_ms, solve_kernel_launches,
 * algorithmic_bytes, jobs_total, jobs_run, solve_retries}. */
int da4ml_sweep_profile(const da4ml_sweep_t *s, double out[8]);
/* Per candidate (either pointer may be NULL):
 *   ints   [n_candidates][12] int64 = {set, H, d (as started), method0, method1 (after api.cc:41-51 and any forced wmc-dc
 *          retry; 0 mc, 1 mc-dc, 2 mc-pdc, 3 wmc, 4 wmc-dc, 5 wmc-pdc, 6 dummy), final decompose_dc, adders, stage-0 ops,
 *          stage-1 ops, winner, front, kept}
 *   floats [n_candidates][3] float32 = {cost (float sum over both stages in op order, api.cc:222-227), latency_min,
 *          latency_max (Pipeline.latency: the last stage's output latencies)} */
int da4ml_sweep_summary(const da4ml_sweep_t *s, int64_t *ints, float *floats);
/* A kept candidate as an ordinary two-stage result (a copy; free with da4ml_pipeline_free).  DA4ML_E_INVALID for a
 * candidate that was not kept or is out of range. */
int da4ml_sweep_pipeline(const da4ml_sweep_t *s, int64_t candidate, da4ml_pipeline_t **out);
void da4ml_sweep_free(da4ml_sweep_t *s);
/* The front rule on its own (no device): front[i] = 1 when no j dominates i on (cost, latency_max), 0 otherwise. */
int da4ml_sweep_front(const float *cost, const float *latency_max, int64_t n, int8_t *front);

/* ---- result access (mirrors make_py_comblogic, bindings.cc:106-139) ---------------------------- */
void da4ml_pipeline_free(da4ml_pipeline_t *p);
int64_t da4ml_pipeline_n_stages(const da4ml_pipeline_t *p);
/* meta: {n_in, n_out, n_ops, carry_size, adder_size} */
int da4ml_pipeline_stage_meta(const da4ml_pipeline_t *p, int64_t stage, int64_t meta[5]);
/* inp_shifts[n_in], out_idxs/out_shifts/out_negs[n_out] int64;
 * ops_i [n_ops,4] int64 (id0,id1,opcode,data); ops_f [n_ops,5] float32 (qmin,qmax,qstep,latency,cost).
 * Any pointer may be NULL to skip that array. */
int da4ml_pipeline_stage_copy(
    const da4ml_pipeline_t *p, int64_t stage, int64_t *inp_shifts, int64_t *out_idxs,
    int64_t *out_shifts, int64_t *out_negs, int64_t *ops_i, float *ops_f
);
/* Work counters of one stage, int64[32]: see enum Meta in csrc/cmvm_types.cuh
 * (status, n_ops, T, sum|F_t|, sum R_t, F0, R0, D_final, F_max, compactions, ..., per-phase SM cycles). */
int da4ml_pipeline_stage_counters(const da4ml_pipeline_t *p, int64_t stage, int64_t counters[32]);
/* Diagnostic: 7 x 10 words, one group per milestone of 250 * 2^k greedy steps (k = 0..6): cumulative cycles CTA 0 of the
 * problem's group spent in each of the 8 phases of a greedy step, the cycles its refresh team spent counting digit pairs
 * of the recount, and the cycles since the loop started (zero for milestones the stage did not reach). */
int da4ml_pipeline_stage_milestones(const da4ml_pipeline_t *p, int64_t stage, int64_t out[70]);
/* Device milliseconds spent in this library's kernels for the call that produced p (CUDA events). */
double da4ml_pipeline_device_ms(const da4ml_pipeline_t *p);
/* Number of kernel launches issued for the call that produced p. */
int64_t da4ml_pipeline_launches(const da4ml_pipeline_t *p);
/* Profile of the call that produced p: {device_ms, launches, solve_kernel_ms, solve_kernel_launches,
 * algorithmic_bytes (all solve_single jobs of the call, exact in accounting mode), jobs_total, jobs_run,
 * solve_retries (solve_single jobs relaunched with larger capacities after a capacity status)}. */
int da4ml_pipeline_profile(const da4ml_pipeline_t *p, double out[8]);

/* ---- pipelined pricing ----------------------------------------------------------------------------
 * Price designs (solver results) as they will be pipelined under latency cutoffs: for every (design d, cutoff j), what
 * the reference computes by replaying d's stages through its symbolic tracer under HWConfig(adder_size, carry_size, c)
 * with the inputs at d's input latencies, gathering the result with comb_trace (dead ops dropped) and splitting it with
 * to_pipeline(comb, c, retiming=0); with retiming = 1, what retime_pipeline then keeps (every re-trace has its inputs at
 * latency 0, as the reference's re-trace of a split has them).
 * Designs are given as flat per-stage arrays, the stages of all designs concatenated in order: n_stages[n_designs];
 * stage_meta [total stages][5] = {n_in, n_out, n_ops, carry_size, adder_size} (da4ml_pipeline_stage_meta); inp_shifts,
 * out_idxs, out_shifts, out_negs, ops_i [.,4], ops_f [.,5] concatenated in the layout of da4ml_pipeline_stage_copy.
 * latencies: per design its first stage's n_in input latencies, concatenated (NULL: zeros).  cutoffs[n_cutoffs] > 0.
 * Outputs [n_designs][n_cutoffs]: status (0 ok, 1 an adder is slower than the cutoff -- the tracer's AssertionError,
 * 2 not supported -- a constant intermediate value), stages (len of the split), reg_bits (Pipeline.reg_bits of the
 * split), latency_max (the traced output latencies' maximum), cutoff_out (the cutoff retiming settled on; the cutoff
 * itself without retiming); out_latency (NULL to skip) [n_designs][n_cutoffs][n_out of the design] the traced output
 * latencies (0.0 for a dead column).  Not ok: stages = reg_bits = -1, latencies NaN.  profile (NULL to skip) =
 * {device_ms, launches}.  A design may also hold the relu / quantize ops of a chain design (opcodes +-2 / +-3: id0 an
 * earlier op, id1 -1, data 0, the op's interval on a power-of-two grid giving its (k, i, f); TRN / WRAP), replayed as
 * CombLogic.__call__ replays them, constant additions (opcode 4) and lookups (opcode 8: id0 an earlier op, id1 -1, data
 * its table's index in [0, 2^31), the op's interval the table's out_qint on a power-of-two grid).  The tables do not
 * cross this ABI: a lookup's cost and latency depend on intervals only, and the caller must check each lookup's index
 * against its own tables (the split hands the index back unchanged).  Arguments are checked on the host before any
 * device call: shapes, other opcodes,
 * operands, bad activation intervals, an activation of a non-zero constant and cutoffs <= 0 give DA4ML_E_INVALID. */
int da4ml_pipeline_price(
    int64_t n_designs, const int64_t *n_stages, const int64_t *stage_meta, const int64_t *inp_shifts,
    const int64_t *out_idxs, const int64_t *out_shifts, const int64_t *out_negs, const int64_t *ops_i,
    const float *ops_f, const double *latencies, const double *cutoffs, int64_t n_cutoffs, int retiming,
    int32_t *status, int64_t *stages, int64_t *reg_bits, double *latency_max, double *cutoff_out,
    double *out_latency, double profile[2]
);

/* Pipelined pricing that also builds and keeps the register stages (the split) of every ok task on the GPU: the
 * arguments and outputs of da4ml_pipeline_price, profile (NULL to skip) = {device_ms, launches, split launches, bytes of
 * op tables copied back}, and *out a handle to free with da4ml_split_free.  The split of task (d, j) is what the
 * reference's to_pipeline(comb, c, retiming) returns: without retiming, the split of the trace under d's input latencies;
 * with it, retime_pipeline's (the first split when no bisection round succeeded, else the last successful round's, at
 * cutoff_out with every input at latency 0).  Relu / quantize ops come back as the tracer writes them: (id0, -1, +-2 / +-3,
 * 0), negative for a negated operand.  Arguments are checked on the host before any device call. */
typedef struct da4ml_split da4ml_split_t; /* opaque split result */
int da4ml_pipeline_split(
    int64_t n_designs, const int64_t *n_stages, const int64_t *stage_meta, const int64_t *inp_shifts,
    const int64_t *out_idxs, const int64_t *out_shifts, const int64_t *out_negs, const int64_t *ops_i,
    const float *ops_f, const double *latencies, const double *cutoffs, int64_t n_cutoffs, int retiming,
    int32_t *status, int64_t *stages, int64_t *reg_bits, double *latency_max, double *cutoff_out,
    double *out_latency, double profile[4], da4ml_split_t **out
);
/* task = d * n_cutoffs + j: out = {status, n_stages, n_rows, n_outs}; status 0: split kept, 1: the task is not ok (no
 * split), 2: the reference's to_pipeline raises KeyError on the task (a stage would have no op or no output, as when
 * every input arrives after the first stage). */
int da4ml_split_info(const da4ml_split_t *s, int64_t task, int64_t out[4]);
/* A kept split's stages, concatenated in stage order: stage_meta [n_stages][3] = {n_in, n_out, n_ops}; out_idxs,
 * out_shifts, out_negs [n_outs] (shifts and negations are the design's in the last stage, 0 before); ops_i [n_rows][4];
 * ops_f [n_rows][5] in float64 (copy latencies c * (j + 1) and traced latencies are doubles).  inp_shifts are all 0. */
int da4ml_split_copy(const da4ml_split_t *s, int64_t task, int64_t *stage_meta, int64_t *out_idxs, int64_t *out_shifts,
                     int64_t *out_negs, int64_t *ops_i, double *ops_f);
/* Both accessors give DA4ML_E_INVALID, with the reason in da4ml_cmvm_last_error, for a null handle or array, a task out
 * of range, or (da4ml_split_copy) a task without a split. */
void da4ml_split_free(da4ml_split_t *s);

/* ---- DAIS interpreter (SURVEY 8f N2) ----------------------------------------------------------------
 * Replaces `run_interp` of the reference's second native module (dais/bindings.cc:30-131 -> DAISInterpreter.cc) for
 * every DAIS program: all opcodes of DAISInterpreter::exec_ops and lookup tables.  Programs are the int32 words of
 * CombLogic.to_binary (types.py:500-541); inputs [n_samples, n_in] float64, outputs [n_samples, n_out] float64, both
 * row-major.  Bit-exact int64 fixed-point semantics of the reference interpreter's compiled code. */
typedef struct da4ml_dais_program da4ml_dais_program_t; /* opaque loaded program */

/* Parse and validate a program on the host (no device call): size, version and table block, causality, opcodes, operand
 * ids, table indices, mux shift configurations, bit-op kinds.  Errors return DA4ML_E_RUNTIME with the reference's
 * wording where it has one.  Free with da4ml_dais_program_free. */
int da4ml_dais_program_load(const int32_t *words, int64_t n_words, da4ml_dais_program_t **out);
/* info: {n_in, n_out, n_ops, n_tables, n_levels, max op width} */
int da4ml_dais_program_info(const da4ml_dais_program_t *p, int64_t info[6]);
/* Run on n_samples rows on the stream set with da4ml_cmvm_set_stream.  device_ptrs = 1: inputs / outputs are device
 * pointers, used in place, and the call returns without waiting unless the program has lookups.  Runs of any programs on
 * any streams are executed one after the other on the device (they share the library's scratch buffer), each ordered
 * after the work already queued on its own stream.  A lookup index out of range fails with the reference's message for
 * the first failing sample (lowest sample, then lowest op); outputs of the chunk that failed and of later chunks are
 * then unspecified. */
int da4ml_dais_program_run(da4ml_dais_program_t *p, const double *inputs, int64_t n_samples, double *outputs, int device_ptrs);
/* Same, on the given stream (cudaStream_t as void*) instead of the library's stream, which stays as it is. */
int da4ml_dais_program_run_stream(
    da4ml_dais_program_t *p, const double *inputs, int64_t n_samples, double *outputs, int device_ptrs, void *cuda_stream
);
/* Profiling: an op's code is its int64 value in the interpreter (its real value is code * 2^-fractionals).  Both calls
 * run the program as da4ml_dais_program_run_stream does, on the given stream, with the same ordering and lookup errors,
 * and check their arguments on the host before any device call (DA4ML_E_INVALID). */
/* Per-op statistics of the op codes over n_samples rows, on the given stream: stats [n_ops][3] int64 host =
 * {min, max, bitwise OR}; identity {INT64_MAX, INT64_MIN, 0} for zero samples.  Synchronises.  On a lookup error the
 * reference's message is returned and stats is not written. */
int da4ml_dais_program_profile(da4ml_dais_program_t *p, const double *inputs, int64_t n_samples, int device_ptrs,
                               void *cuda_stream, int64_t *stats);
/* Codes of ops op_ids[0..n_sel) for every row: values [n_samples][n_sel] int64 (device pointer when device_ptrs).
 * op_ids is host memory; ids may repeat.  Returns without waiting under the same conditions as a run. */
int da4ml_dais_program_dump(da4ml_dais_program_t *p, const double *inputs, int64_t n_samples, const int32_t *op_ids,
                            int64_t n_sel, int64_t *values, int device_ptrs, void *cuda_stream);
void da4ml_dais_program_free(da4ml_dais_program_t *p);

/* The programs the CMVM path produces only (opcodes -1, 0, 1; no lookup tables), host arrays; any other program is
 * refused.  Same engine as da4ml_dais_program_run. */
int da4ml_dais_run(const int32_t *program, int64_t n_words, const double *inputs, int64_t n_samples, double *outputs);

/* ---- helpers exported by the reference module -------------------------------------------------- */
/* `csd_decompose` (bindings.cc:63-103 -> bit_decompose.cc:44-62).  csd must hold n_in*n_out*32 int8;
 * *n_bits receives N, the caller reads csd as [n_in, n_out, N].  shift0[n_in], shift1[n_out] int8. */
int da4ml_cmvm_csd_decompose(
    const float *kernel, int64_t n_in, int64_t n_out, int center, int8_t *csd, int8_t *shift0,
    int8_t *shift1, int64_t *n_bits
);
/* `int_arr_to_csd` (bindings.cc:43-61 -> bit_decompose.cc:22-42): flat int32[n] -> int8[n, N]. */
int da4ml_cmvm_int_arr_to_csd(const int32_t *x, int64_t n, int8_t *csd, int64_t *n_bits);
/* `kernel_decompose` (mat_decompose.cc:62-137): m0 [n_in,n_out], m1 [n_out,n_out]. */
int da4ml_cmvm_kernel_decompose(const float *kernel, int64_t n_in, int64_t n_out, int dc, float *m0, float *m1);
/* scalar helpers (bit_decompose.cc:10-20, indexers.hh:12-18, state_opr.cc:31-67) */
int da4ml_cmvm_get_lsb_loc(float x);
int da4ml_cmvm_iceil_log2(float x);
int da4ml_cmvm_cost_add(
    const float q0[3], const float q1[3], int64_t shift, int sub, int adder_size, int carry_size,
    float out[2] /* (latency increment, cost) */
);

#ifdef __cplusplus
}
#endif
#endif
