// cmvm_kernels.cuh -- sm_90a kernels of the CMVM greedy common-subexpression solver.
//
//   cmvm_prep_kernel    centre + CSD-decompose the constant matrix into packed sign planes
//                       (bit_decompose.hh:21-34, bit_decompose.cc:22-62, state_opr.cc:92-97)
//   cmvm_solve_kernel   persistent kernel (cmvm_kernel_own.cuh); a group of G CTAs owns one problem:
//                       build the lists + initial pair histogram (state_opr.cc:100-144),
//                       greedy loop = select / substitute / recount (cmvm_core.cc:36-70,
//                       indexers.cc, state_opr.cc:227-345), adder-tree finisher (cmvm_core.cc:89-225)
//
// Formulation (differs from the reference by design, results are identical):
//   * a row of an expression in one output column is two sign planes, so a pair count is a
//     handful of AND/shift/popc and substitution is a mask operation;
//   * the histogram is an unordered, append-only log of (score, stamp, packed key) split into one
//     segment per CTA.  The reference's "erase every entry touching id0/id1" (state_opr.cc:291-294)
//     is lazy: each expression carries the step at which it was last rewritten, an entry is live iff
//     its creation stamp is not older than either operand's rewrite step.  The argmax keeps a
//     per-chunk cached maximum in shared memory and re-reads a chunk only when its cached winner
//     died; order independence comes from reducing on the composite (score, key), whose order is
//     exactly the reference's "last maximum in sorted order";
//   * expression e is owned by CTA e mod G, which keeps the rows of its expressions as per-column lists in
//     shared memory and counts the digit pairs of a step in a shared-memory hash table (solve_owned.cuh).
#pragma once
#include "cmvm_prep.cuh"
#include "solve_finish.cuh"
#include "solve_histogram.cuh"
