// Host-side planning for the shared-memory ("cooperative") kernels: dependency segments, history
// analysis, slot assignment.
//
// The reference does the equivalent bookkeeping for its compact mode: taylor_segment_dc()
// (src/taylor_02.cpp:105-207) splits the decomposition into segments of mutually independent u variables,
// and the tape holds every u variable at every order (src/taylor_02.cpp:1227-1233). Here the tape has to
// fit in the 227 KB of shared memory of an SM, so only what is re-read at a LATER order keeps its history:
//   H  ("history")   operands of convolution-type recurrences: p (or p + 1) slots, one per order
//   SV (state var)   two slots, ping-pong on the order's parity (order n is built from order n - 1)
//   T  ("transient") everything that is only consumed at the order at which it is produced: one slot
// The coefficients of the state variables of every order are streamed to the tc array in HBM (they are
// needed again only once, for the step-size estimate and the state update).
#ifndef HEYOKA_B200_CSRC_SMEM_PLAN_HPP
#define HEYOKA_B200_CSRC_SMEM_PLAN_HPP

#include <cstdint>
#include <vector>

#include "program.hpp"

namespace heyoka_b200::detail
{

// Packed row reference (30 bits): (mask code << 27) | first slot. The order-o coefficient of a row lives in
// slot `first + (o & mask)`, mask = sign-extended mask code: 0 (T, one slot), 1 (SV, two slots on the parity of
// the order), ~0 (H, one slot per order). The device decodes the mask with one shift pair.
constexpr std::uint32_t ROW_T = 0u, ROW_SV = 1u, ROW_H = 7u;
constexpr std::uint32_t ROW_SLOT_BITS = 27u;

// Superinstructions (internal to the plan, never part of a hy_program): opcodes >= HY_FOP_FIRST.
//   HY_FOP_NBODY_PAIR  the gravitational pair interaction of model::nbody (src/model/nbody.cpp:97-153): 3 sub,
//                      sum_sq, pow, optional scaling, 3 products, optional 3 scalings run by ONE work item.
//                      op.a = offset into aux (33 words, see make_smem_plan()), op.b = kind of the scaling of
//                      r^alpha (0 none, 1 constant, 2 negation), op.c = 1 if the products are rescaled.
//   HY_FOP_SUM_T       a sum whose terms are all single-slot rows (argument table entries = slots).
constexpr std::uint32_t HY_FOP_FIRST = 0x100u, HY_FOP_NBODY_PAIR = 0x100u, HY_FOP_SUM_T = 0x101u;
// Words per HY_FOP_NBODY_PAIR entry in aux: 27 operand words + 6 offsets into svout (m_0..2, n_0..2; 0 = none).
constexpr std::uint32_t HY_FOP_NBODY_PAIR_AUX = 33u;

struct smem_plan {
    std::uint32_t n_slots = 0;  // doubles of shared memory per lane
    // Doubles per lane of the overflow tape in HBM/L2: when shared memory is the limit on the number of
    // resident warps, the rows that only a superinstruction reads (r^2 and r^alpha histories of the pair
    // interaction) are moved out of shared memory (spill_private).
    std::uint32_t n_gslots = 0;
    std::uint32_t n_segments = 0;
    std::uint32_t max_seg_width = 0;
    // Ops in execution order (segment by segment, grouped by opcode inside a segment); operand fields that
    // referred to u variables are row references.
    std::vector<hy_op> ops;
    std::vector<std::uint32_t> dst;         // row reference of the u variable each op defines
    std::vector<std::uint32_t> seg_offsets; // n_segments + 1 offsets into ops
    std::vector<std::uint32_t> args;        // n-ary argument table, variable entries -> row references
    std::vector<std::uint32_t> sv_defs;     // idem for the state variables' derivatives
    std::vector<std::uint32_t> sv_rows;     // row reference of each state variable
    std::vector<std::uint32_t> aux;         // operand tables of the superinstructions
    std::uint32_t n_fused = 0;              // number of superinstructions
    // Constants appended to the program's pool (indices start at n_consts): per distinct exponent alpha of the
    // pair interactions, the table j * (alpha + 1), j = 0..order, of the pow recurrence.
    std::vector<double> extra_consts;
    // State-variable propagation fused into the producers. When u^[n] is the right-hand side of state variable
    // s, the work item that produces it also writes x_s^[n+1] = u^[n] / (n + 1) (and x_s2^[n+2] for a state
    // variable s2 whose derivative is s, e.g. positions whose derivative is a velocity): no separate pass and
    // no synchronisation for those. svout: [count, (sv, row, depth) x count] lists, addressed by svo[] (one
    // per op, 0 = none, else offset + 1). sv_cover[s]: 0 = handled by the generic per-order pass, 1 / 2 = depth
    // of the fused propagation; sv_parent[s]: the state variable s derives from (depth 2).
    std::vector<std::uint32_t> svout, svo, sv_cover, sv_parent, sv_phase;
};

smem_plan make_smem_plan(const hy_program &, bool fuse = true, bool fuse_sv = true, bool spill_private = false);

} // namespace heyoka_b200::detail

#endif
