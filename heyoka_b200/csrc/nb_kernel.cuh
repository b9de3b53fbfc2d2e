// k_nb: the dedicated sm_90a kernel for N-body-shaped programs (nb_plan.hpp): model::nbody of the outer Solar System
// (6 bodies, 15 pair interactions), the two-body step benchmark, model::nbody with 32 bodies (496 pair interactions).
//
// Same persistent structure as k_coop (kernels.cuh): a team (a warp, or the whole CTA when one lane has hundreds of pair
// interactions) owns LT lanes, claims chunks of LT lanes from an atomic counter and runs a chunk's whole
// propagate_until() loop; the state update and the per-lane bookkeeping are the functions of kernels.cuh. What
// differs is the jet:
//   * the orders are walked two at a time (nb_core.hpp), two synchronisations per PAIR of orders;
//   * a thread is bound to one (pair interaction, lane) for the whole kernel: its operands' shared-memory addresses
//     and constants live in registers, nothing is decoded per order;
//   * its private history rows are stored as (even order, odd order) pairs in shared memory, interleaved by thread
//     ([order pair][row][thread], one 16-byte access per thread, conflict-free); with CTA teams, when the five rows of
//     512 threads do not fit in shared memory (model::nbody with 32 bodies), r^2, d_2 and r^alpha go to a per-CTA
//     slab of global memory that stays in L2 (OFFCHIP = true; same interleaving, coalesced);
//   * shared memory otherwise only holds what threads exchange: the positions of the current order pair and the
//     outputs of the pair interactions / partial sums ([role][pair][lane] so that a warp writes consecutive slots);
//   * what a thread does in the summation phase is a pre-decoded 32-byte record (nb_role) per round;
//   * the three infinity norms of the step-size estimate are gathered while the coefficients are produced: no second
//     pass over the coefficients for h. Warp teams of the 256-thread instantiations keep each thread's maxima in
//     registers and reduce them with warp shuffles after the jet; the others use shared-memory atomic maxima on the
//     bit patterns of |x|.
// All shared-memory accesses use 32-bit shared-window addresses (ld.shared / st.shared): no generic addressing, no
// 64-bit pointer arithmetic in the hot loops.
// Replaces, for these programs: the JIT'd step function (src/taylor_00.cpp:712-865) and the propagate loop
// (src/taylor_adaptive_batch.cpp:1136-1534), like k_coop.
#ifndef HEYOKA_B200_CSRC_NB_KERNEL_CUH
#define HEYOKA_B200_CSRC_NB_KERNEL_CUH

#include <cstdint>

#include <cuda_runtime.h>

#include "kernels.cuh"
#include "nb_core.hpp"
#include "nb_desc.hpp"

namespace heyoka_b200::dev
{

// Systems with ONE pair interaction run one thread per lane (k_nb1, nb1_kernel.cuh). Slot s = 3 * side + k: side 0 /
// 1 = the body whose positions are the pair's pa / pb, k = coordinate. The accelerations of a side's velocities v_sv
// (whose position children are x_sv) are the pair outputs m_k (kind 0), n_k (kind 1) or the number 0 (kind 2).
// sv0_slot / sv0_is_x: where state variable 0 sits (its NaNs are the ones the step-size norms let through).
struct nb1_tab {
    std::uint32_t v_sv[6], x_sv[6], kind[2];
    std::uint32_t sv0_slot, sv0_is_x;
};

// Device-side view of an nb_plan (arrays in global memory) + the shared-memory layout chosen by the host.
struct nb_dev_plan {
    const detail::nb_pair_desc *pairs;
    const uint4 *roles; // n_rounds x TT records of 2 x uint4
    const double *consts, *fac;
    std::uint32_t n_pairs, n_pos, n_out, n_consts, npp, fac_stride;
    std::uint32_t n_rounds, round_level_end; // rounds of the summation phase; bit r: round r ends a level
    double alpha;
    std::uint32_t pow_algo;
    std::uint32_t roles_in_smem;  // 1: the role table is copied to shared memory
    std::uint32_t shared_doubles; // CTA-shared tables: fac | rcp | consts | roles
    std::uint32_t team_doubles;   // per team: positions | outputs | private rows | norms | scalars
    std::uint32_t n_slots_equiv;  // team region (without the scalars) expressed in coop_smem<LT> slots
    double *offchip;              // OFFCHIP kernels: per CTA, [order pair][3 rows][thread] pairs of doubles
    nb1_tab l1;                   // k_nb1 only
};

// Per-phase cycle attribution of k_nb (warp teams, PROP), compiled in with -DHY_NB_PHASE_CLOCK only
// (tools/nb_phase_profile.py): thread 0 of every team adds the clock64() cycles between the phase boundaries to
// nb_phase_cycles[team][phase], and counts the team's warp-steps and its lifetime. The sub-phases split the pair and
// summation phases of thread 0 further: each ends where the instructions of its part have been issued, so the latency
// of a load is charged to the sub-phase that first uses the value; what is left of a phase after its sub-phases is the
// wait at the synchronisation that ends it. Without the macro the object has no state and emits no code.
enum nb_phase : int {
    NB_PH_PAIR,      // pair_block() of an order pair, and the sync after it
    NB_PH_SUM,       // the summation rounds of an order pair and their syncs
    NB_PH_INIT,      // role_init(): order 0 from the state, and the sync after it
    NB_PH_STEP_SIZE, // the step size (norm reduction, nb_step_size() or nb_rho()), and the sync after it
    NB_PH_UPDATE,    // coop_update_state() and the reduction of its non-finite mask
    NB_PH_PROP,      // the lane_prop bookkeeping, the loop test and chunk changes
    NB_PH_STEPS,     // (count of warp-steps)
    NB_PH_LIFE,      // (cycles from the first chunk claim to the end of the kernel)
    // Sub-phases of NB_PH_PAIR (nb::pair_block):
    NB_PH_PAIR_SS,   //   d_k and the sum_sq loop, the rows d_k and r^2 stored
    NB_PH_PAIR_MAIN, //   the main loop (pow recurrence and products)
    NB_PH_PAIR_Q,    //   the two quotients of the pow recurrence, r^alpha stored
    NB_PH_PAIR_OUT,  //   the last terms of the products and the output stores
    // Sub-phases of NB_PH_SUM (per round, nb::role_block):
    NB_PH_SUM_ROLE,  //   the role record
    NB_PH_SUM_LOAD,  //   the term loads
    NB_PH_SUM_ARITH, //   the sum and the quotients
    NB_PH_SUM_STORE, //   the coefficient / position / partial-sum stores and the round's sync
    NB_PH_SLOTS
};
#if defined(HY_NB_PHASE_CLOCK)
constexpr std::uint32_t nb_phase_teams = 4096u;
namespace
{
__device__ unsigned long long nb_phase_cycles[nb_phase_teams][NB_PH_SLOTS];
}
struct nb_phase_clock {
    unsigned long long *acc;
    long long t, t0, ts;
    __device__ __forceinline__ void start(std::size_t team, bool leader)
    {
        acc = leader && team < nb_phase_teams ? nb_phase_cycles[team] : nullptr;
        ts = t0 = t = clock64();
    }
    __device__ __forceinline__ void lap(nb_phase ph)
    {
        const long long now = clock64();
        if (acc != nullptr) {
            atomicAdd(acc + ph, static_cast<unsigned long long>(now - t));
        }
        ts = t = now;
    }
    // A sub-phase: the cycles since the last lap() or sub().
    __device__ __forceinline__ void sub(nb_phase ph)
    {
        const long long now = clock64();
        if (acc != nullptr) {
            atomicAdd(acc + ph, static_cast<unsigned long long>(now - ts));
        }
        ts = now;
    }
    __device__ __forceinline__ void step()
    {
        if (acc != nullptr) {
            atomicAdd(acc + NB_PH_STEPS, 1ull);
        }
    }
    __device__ __forceinline__ void finish()
    {
        if (acc != nullptr) {
            atomicAdd(acc + NB_PH_LIFE, static_cast<unsigned long long>(clock64() - t0));
        }
    }
};
#else
struct nb_phase_clock {
    __device__ __forceinline__ void start(std::size_t, bool) {}
    __device__ __forceinline__ void lap(nb_phase) {}
    __device__ __forceinline__ void sub(nb_phase) {}
    __device__ __forceinline__ void step() {}
    __device__ __forceinline__ void finish() {}
};
#endif

namespace nbk
{

using nb::d2;

__device__ __forceinline__ std::uint32_t saddr(const void *p)
{
    return static_cast<std::uint32_t>(__cvta_generic_to_shared(p));
}
// Pins a loop-invariant value in a register: without it the compiler re-derives shared-window addresses and kernel
// parameters (a dozen uniform-datapath instructions each) inside the per-order-pair code instead of keeping them.
__device__ __forceinline__ void keep(std::uint32_t &x)
{
    asm volatile("" : "+r"(x));
}
__device__ __forceinline__ d2 lds2(std::uint32_t a)
{
    d2 v;
    asm volatile("ld.shared.v2.f64 {%0, %1}, [%2];" : "=d"(v.x), "=d"(v.y) : "r"(a));
    return v;
}
__device__ __forceinline__ double lds1(std::uint32_t a)
{
    double v;
    asm volatile("ld.shared.f64 %0, [%1];" : "=d"(v) : "r"(a));
    return v;
}
__device__ __forceinline__ uint4 lds4u(std::uint32_t a)
{
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a));
    return v;
}
__device__ __forceinline__ void sts2(std::uint32_t a, const d2 &v)
{
    asm volatile("st.shared.v2.f64 [%0], {%1, %2};" ::"r"(a), "d"(v.x), "d"(v.y) : "memory");
}
__device__ __forceinline__ void red_max_u64(std::uint32_t a, unsigned long long v)
{
    asm volatile("red.shared.max.u64 [%0], %1;" ::"r"(a), "l"(v) : "memory");
}
__device__ __forceinline__ d2 from_words(std::uint32_t a, std::uint32_t b, std::uint32_t c, std::uint32_t d)
{
    return d2{__hiloint2double(static_cast<int>(b), static_cast<int>(a)),
              __hiloint2double(static_cast<int>(d), static_cast<int>(c))};
}

// Storage policy of pair_block() (nb_core.hpp). TT = threads per team. All members are shared-window addresses.
// Private rows in shared memory: element (order pair op, row r) of this thread at drow + (op * NSR + r) * TT * 16,
// rows d_0, d_1 (+ d_2, r^2, r^alpha when OFFCHIP is false). Off chip: element (op, r) of this thread at
// grow[(op * 3 + r) * TT], rows r^2, d_2, r^alpha.
template <int TT, bool OFFCHIP>
struct pair_mem {
    static constexpr int NSR = OFFCHIP ? 2 : 5;
    // pair_block()'s reciprocals ahead of the main loop (nb_core.hpp, early_den()): not with the rows off chip, where
    // the reload of r2^[0]'s terms is an L2 access and the 512-thread kernel has no registers to spare.
    static constexpr bool EARLY_DEN = !OFFCHIP;
    static constexpr std::uint32_t OPB = static_cast<std::uint32_t>(NSR) * TT * 16u; // bytes per order pair
    static constexpr std::uint32_t RB = TT * 16u;                                    // bytes per row
    std::uint32_t pa[3], pb[3]; // the six positions this pair reads (this thread's lane)
    std::uint32_t om, kstride;  // output m_0 of this (pair, lane); m_k / n_k are k / (3 + k) strides further
    std::uint32_t drow;         // this thread's slice of the private rows
    std::uint32_t fac_, fac_stride_b;
    double2 *grow; // OFFCHIP: this thread's element (0, 0)
    std::uint32_t flags; // bit 0: active (owns a pair), bits 1-3: n_k exists
#if defined(HY_NB_PHASE_CLOCK)
    nb_phase_clock *clk;
    __device__ __forceinline__ void lap(int k) const
    {
        clk->sub(static_cast<nb_phase>(NB_PH_PAIR_SS + k));
    }
#endif

    __device__ __forceinline__ d2 gld(std::uint32_t op, std::uint32_t r) const
    {
        const double2 v = grow[(op * 3u + r) * TT];
        return d2{v.x, v.y};
    }
    __device__ __forceinline__ void gst(std::uint32_t op, std::uint32_t r, const d2 &v) const
    {
        grow[(op * 3u + r) * TT] = make_double2(v.x, v.y);
    }
    __device__ __forceinline__ d2 pos_a(int k) const
    {
        return lds2(pa[k]);
    }
    __device__ __forceinline__ d2 pos_b(int k) const
    {
        return lds2(pb[k]);
    }
    __device__ __forceinline__ void st_d(std::uint32_t m, const d2 (&D)[3]) const
    {
        const std::uint32_t p = drow + m * OPB;
        sts2(p, D[0]);
        sts2(p + RB, D[1]);
        if constexpr (OFFCHIP) {
            gst(m, 1u, D[2]);
        } else {
            sts2(p + 2u * RB, D[2]);
        }
    }
    __device__ __forceinline__ void st_r2(std::uint32_t m, const d2 &r) const
    {
        if constexpr (OFFCHIP) {
            gst(m, 0u, r);
        } else {
            sts2(drow + m * OPB + 3u * RB, r);
        }
    }
    __device__ __forceinline__ void st_q(std::uint32_t m, const d2 &q) const
    {
        if constexpr (OFFCHIP) {
            gst(m, 2u, q);
        } else {
            sts2(drow + m * OPB + 4u * RB, q);
        }
    }
    __device__ __forceinline__ void ld_ss(std::uint32_t ai, std::uint32_t li, d2 (&A)[3], d2 (&Lo)[3]) const
    {
        const std::uint32_t pa_ = drow + ai * OPB, pl = drow + li * OPB;
        if constexpr (OFFCHIP) {
            A[2] = gld(ai, 1u);
            Lo[2] = gld(li, 1u);
            A[0] = lds2(pa_);
            A[1] = lds2(pa_ + RB);
            Lo[0] = lds2(pl);
            Lo[1] = lds2(pl + RB);
        } else {
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                A[k] = lds2(pa_ + k * RB);
                Lo[k] = lds2(pl + k * RB);
            }
        }
    }
    __device__ __forceinline__ void ld_a(std::uint32_t ai, d2 (&A)[3]) const
    {
        const std::uint32_t pa_ = drow + ai * OPB;
        if constexpr (OFFCHIP) {
            A[2] = gld(ai, 1u);
            A[0] = lds2(pa_);
            A[1] = lds2(pa_ + RB);
        } else {
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                A[k] = lds2(pa_ + k * RB);
            }
        }
    }
    __device__ __forceinline__ void ld_main(std::uint32_t qi, std::uint32_t li, d2 &Q, d2 &Rlo, d2 (&Dlo)[3]) const
    {
        const std::uint32_t pl = drow + li * OPB;
        if constexpr (OFFCHIP) {
            Rlo = gld(li, 0u);
            Dlo[2] = gld(li, 1u);
            Q = gld(qi, 2u);
            Dlo[0] = lds2(pl);
            Dlo[1] = lds2(pl + RB);
        } else {
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                Dlo[k] = lds2(pl + k * RB);
            }
            Rlo = lds2(pl + 3u * RB);
            Q = lds2(drow + qi * OPB + 4u * RB);
        }
    }
    __device__ __forceinline__ d2 fac(std::uint32_t n, std::uint32_t j) const
    {
        return lds2(fac_ + n * fac_stride_b + j * 8u);
    }
    __device__ __forceinline__ double fac1(std::uint32_t n, std::uint32_t j) const
    {
        return lds1(fac_ + n * fac_stride_b + j * 8u);
    }
    __device__ __forceinline__ void out(int k, const d2 &v) const
    {
        if ((flags & 1u) != 0u) {
            sts2(om + static_cast<std::uint32_t>(k) * kstride, v);
        }
    }
    __device__ __forceinline__ void out_n(int k, const d2 &v) const
    {
        if ((flags & (2u << k)) != 0u) {
            sts2(om + static_cast<std::uint32_t>(3 + k) * kstride, v);
        }
    }
};

// Storage policy of role_block() / role_init(): the thread's NL lanes start at lane l0 of the team's LT lanes (the
// records' units already include l0).
// REGN: the thread keeps its maxima of the step-size norms in registers (nrm), reduced over the team with warp
// shuffles once the jet is done (norms_reduce); otherwise they go to the team's norm slots in shared memory by atomic
// maxima, which sm_90 executes as compare-and-swap loops.
template <int NL, bool REGN>
struct role_mem {
    std::uint32_t pos_b, out_b;   // team bases
    std::uint32_t consts, rcp_;   // CTA tables
    std::uint32_t norms;          // team norms: [3][LT] u64 (|x^[0]|, |x^[p]|, |x^[p-1]|), + lane l0 of this thread
    std::uint32_t lt8;            // copies * LT * 8: stride between the three norms
    mutable double nrm[3][NL];    // REGN: this thread's maxima (|x^[0]|, |x^[p]|, |x^[p-1]|) of its lanes
    const double *state0;         // D.state + first global lane of this thread (clamped)
    std::size_t n_batch;
    double *cbase;                // coefficient store + lane offset of lane 0 of this thread
    std::size_t stride_sv, stride_o;
    std::uint32_t p;
    bool pub, track;
    bool lane_ok[NL];
    std::uint32_t ldelta; // offset (in doubles) between the thread's lanes in state / public store (0 if clamped)
#if defined(HY_NB_PHASE_CLOCK)
    nb_phase_clock *clk;
    __device__ __forceinline__ void lap(int k) const
    {
        clk->sub(static_cast<nb_phase>(NB_PH_SUM_LOAD + k));
    }
#endif

    __device__ __forceinline__ d2 out_u(std::uint32_t unit, int l) const
    {
        return lds2(out_b + (unit + l) * 16u);
    }
    __device__ __forceinline__ void out_st_u(std::uint32_t unit, int l, const d2 &v) const
    {
        sts2(out_b + (unit + l) * 16u, v);
    }
    __device__ __forceinline__ void pos_st_u(std::uint32_t unit, int l, const d2 &v) const
    {
        sts2(pos_b + (unit + l) * 16u, v);
    }
    __device__ __forceinline__ double cst(std::uint32_t i) const
    {
        return lds1(consts + i * 8u);
    }
    __device__ __forceinline__ double rcp(std::uint32_t n) const
    {
        return lds1(rcp_ + n * 8u);
    }
    // Norms of the step-size estimate: NaN-skipping maximum of |v| (bit patterns of non-negative doubles order like
    // unsigned integers). which: 0 = order 0, 1 = order p, 2 = order p - 1.
    // (REGN: fmax() skips the NaN and, on non-negative values, picks the same value as the maximum of the bit
    // patterns, so the result is the same bits.)
    __device__ __forceinline__ void norm(std::uint32_t which, int l, double v) const
    {
        if constexpr (REGN) {
            // (Constant indices: a register, not a local-memory array.)
            if (which == 0u) {
                nrm[0][l] = fmax(nrm[0][l], fabs(v));
            } else if (which == 1u) {
                nrm[1][l] = fmax(nrm[1][l], fabs(v));
            } else {
                nrm[2][l] = fmax(nrm[2][l], fabs(v));
            }
        } else if (v == v) {
            red_max_u64(norms + which * lt8 + l * 8u,
                        static_cast<unsigned long long>(__double_as_longlong(v)) & 0x7fffffffffffffffull);
        }
    }
    __device__ __forceinline__ void norms_reset() const
    {
        if constexpr (!REGN) {
            return;
        }
#pragma unroll
        for (int w = 0; w < 3; ++w) {
#pragma unroll
            for (int l = 0; l < NL; ++l) {
                nrm[w][l] = 0.;
            }
        }
    }
    // REGN, warp teams of LT lanes: the maxima of lane tid (< LT) of the team, for its owner thread. Threads whose
    // indices differ by a multiple of GS = LT / NL hold the same lanes: a butterfly over those strides gives each of
    // them the team's maxima. Every thread of the warp takes part.
    template <int LT>
    __device__ __forceinline__ void norms_reduce(std::uint32_t tid, double (&m3)[3]) const
    {
        constexpr int GS = LT / NL;
#pragma unroll
        for (int off = GS; off < 32; off *= 2) {
#pragma unroll
            for (int w = 0; w < 3; ++w) {
#pragma unroll
                for (int l = 0; l < NL; ++l) {
                    nrm[w][l] = fmax(nrm[w][l], __shfl_xor_sync(0xffffffffu, nrm[w][l], off));
                }
            }
        }
        // Lane tid is element tid % NL of the threads with thread index % GS == tid / NL.
        const int src = static_cast<int>((tid % LT) / NL);
#pragma unroll
        for (int w = 0; w < 3; ++w) {
            double v = __shfl_sync(0xffffffffu, nrm[w][0], src);
            if constexpr (NL == 2) {
                const double v1 = __shfl_sync(0xffffffffu, nrm[w][1], src);
                v = (tid % 2u) != 0u ? v1 : v;
            }
            m3[w] = v;
        }
    }
    __device__ __forceinline__ void track_order(std::uint32_t order, const double (&a)[NL]) const
    {
        if (order == 0u || order == p || order + 1u == p) {
            const std::uint32_t which = order == 0u ? 0u : (order == p ? 1u : 2u);
#pragma unroll
            for (int l = 0; l < NL; ++l) {
                norm(which, l, a[l]);
            }
        }
    }
    // One order of state variable sv for the thread's lanes at element index idx of the coefficient store.
    template <typename I>
    __device__ __forceinline__ void store_lanes(I idx, const double (&a)[NL]) const
    {
        if constexpr (NL == 2) {
            if (!pub) {
                // Private store: the two lanes are adjacent and 16-byte aligned.
                *reinterpret_cast<double2 *>(cbase + idx) = make_double2(a[0], a[1]);
                return;
            }
        }
#pragma unroll
        for (int l = 0; l < NL; ++l) {
            if (lane_ok[l]) {
                cbase[idx + (pub ? l * ldelta : l)] = a[l];
            }
        }
    }
    __device__ __forceinline__ void coef_pair(std::uint32_t sv, std::uint32_t order, const double (&a)[NL],
                                              const double (&b)[NL]) const
    {
        if (pub) {
            const std::size_t idx = sv * stride_sv + order * stride_o;
            if (order <= p) {
                store_lanes(idx, a);
            }
            if (order + 1u <= p) {
                store_lanes(idx + stride_o, b);
            }
        } else {
            // (The private store has fewer than 2^32 elements.)
            const std::uint32_t so = static_cast<std::uint32_t>(stride_o);
            const std::uint32_t idx = sv * static_cast<std::uint32_t>(stride_sv) + order * so;
            if (order <= p) {
                store_lanes(idx, a);
            }
            if (order + 1u <= p) {
                store_lanes(idx + so, b);
            }
        }
        if (track) {
            track_order(order, a);
            track_order(order + 1u, b);
        }
    }
    __device__ __forceinline__ void coef_one(std::uint32_t sv, std::uint32_t order, const double (&a)[NL]) const
    {
        store_lanes(sv * stride_sv + order * stride_o, a);
        if (track) {
            track_order(order, a);
        }
    }
    __device__ __forceinline__ double state(std::uint32_t sv, int l) const
    {
        return state0[static_cast<std::size_t>(sv) * n_batch + l * ldelta];
    }
};

} // namespace nbk

// Step size of one lane from the norms gathered during the jet (norms[0], norms[lt], norms[2 lt]: bit patterns of the
// NaN-skipping maxima of |x^[0]|, |x^[p]|, |x^[p-1]|; reset to 0 here) and the coefficients of the first state
// variable: the sequential reference loop m = (m < |x|) ? |x| : m, started from |x_0|, yields NaN iff x_0 is NaN and
// ignores every other NaN (src/taylor_00.cpp:102-273). Once per lane and step: out of line. (The program's constants
// come as values: a reference to the kernel's program would park a copy of it in local memory, read back from L2 at
// every step.)
// norms == nullptr: the maxima come in m0, mp, mp1 (reduced in registers, role_mem::norms_reduce()).
static __device__ __noinline__ double nb_step_size(double inv_p, double inv_pm1, double rhofac, unsigned long long *norms,
                                                   std::uint32_t lt, double m0, double mp, double mp1, const double *c,
                                                   std::size_t off_p, std::size_t off_pm1, double max_delta_t)
{
    if (norms != nullptr) {
        // norms[(which * copies + r) * lt]: the maximum over the copies, which are reset.
        const std::uint32_t copies = detail::nb_norm_copies(lt);
        unsigned long long n3[3];
        for (std::uint32_t w = 0; w < 3u; ++w) {
            unsigned long long v = 0ull;
            for (std::uint32_t r = 0; r < copies; ++r) {
                unsigned long long *q = norms + (w * copies + r) * lt;
                v = *q > v ? *q : v;
                *q = 0ull;
            }
            n3[w] = v;
        }
        m0 = __longlong_as_double(static_cast<long long>(n3[0]));
        mp = __longlong_as_double(static_cast<long long>(n3[1]));
        mp1 = __longlong_as_double(static_cast<long long>(n3[2]));
    }
    const double f0 = fabs(c[0]), fp = fabs(c[off_p]), fp1 = fabs(c[off_pm1]);
    return h_from_norms(inv_p, inv_pm1, rhofac, isnan(f0) ? f0 : m0, isnan(fp) ? fp : mp, isnan(fp1) ? fp1 : mp1,
                        max_delta_t);
}
// One of the two radii of convergence of nb_step_size() (order p: inv = 1 / p, order p - 1: inv = 1 / (p - 1)) from the
// maxima m0 (order 0) and m (that order), with the same NaN rule: c0, c = the coefficients of state variable 0 at
// order 0 and at that order. Out of line: one copy of pow() in the kernel.
static __device__ __noinline__ double nb_rho(double inv, double m0, double m, double c0, double c)
{
    const double f0 = fabs(c0), f = fabs(c);
    return rho_from_norm(isnan(f0) ? f0 : m0, isnan(f) ? f : m, inv);
}

// LT: lanes per team; CTA: a team is the whole CTA (else a warp); OFFCHIP: r^2, d_2, r^alpha rows in NP.offchip.
template <int LT, bool CTA, bool OFFCHIP, bool PROP, int MAXT>
__global__ void __launch_bounds__(MAXT, 1) k_nb(program P, nb_dev_plan NP, batch D, run_args R)
{
    static_assert(!OFFCHIP || CTA, "off-chip private rows are laid out per CTA");
    using T = team<CTA>;
    constexpr int TT = CTA ? MAXT : 32; // threads per team (CTA teams are launched with exactly MAXT threads)
    constexpr int NL = LT >= 2 ? 2 : 1; // lanes per thread in the summation phase
    constexpr std::uint32_t GS = LT / NL;
    extern __shared__ __align__(16) double smem_raw[];

    // ---- CTA-shared tables: fac | rcp | consts | roles ----
    const std::uint32_t p = P.order;
    double *fac_s = smem_raw;
    const std::uint32_t n_fac = (p + 1u) * NP.fac_stride;
    double *rcp_s = fac_s + n_fac;
    const std::uint32_t n_rcp = (p + 5u) & ~1u;
    double *consts_s = rcp_s + n_rcp;
    const std::uint32_t n_cst = (NP.n_consts + 1u) & ~1u;
    uint4 *roles_s = reinterpret_cast<uint4 *>(consts_s + n_cst);
    for (std::uint32_t i = threadIdx.x; i < n_fac; i += blockDim.x) {
        fac_s[i] = __ldg(NP.fac + i);
    }
    for (std::uint32_t i = threadIdx.x; i < n_rcp; i += blockDim.x) {
        rcp_s[i] = i == 0u ? 0. : 1. / static_cast<double>(i);
    }
    for (std::uint32_t i = threadIdx.x; i < NP.n_consts; i += blockDim.x) {
        consts_s[i] = __ldg(NP.consts + i);
    }
    if (NP.roles_in_smem != 0u) {
        for (std::uint32_t i = threadIdx.x; i < NP.n_rounds * TT * 2u; i += blockDim.x) {
            roles_s[i] = __ldg(NP.roles + i);
        }
    }
    __syncthreads();

    const std::uint32_t tid = T::tid();
    double *region = smem_raw + NP.shared_doubles
                     + (CTA ? 0u : static_cast<std::size_t>(threadIdx.x >> 5) * NP.team_doubles);
    const coop_smem<LT> S(region, NP.n_slots_equiv);
    std::uint32_t pos_b = nbk::saddr(region);
    std::uint32_t out_b = pos_b + NP.n_pos * LT * 16u;
    const std::uint32_t drow_b = out_b + NP.n_out * LT * 16u;
    const std::uint32_t norms_b = drow_b + NP.npp * nbk::pair_mem<TT, OFFCHIP>::OPB;
    nbk::keep(pos_b);
    nbk::keep(out_b);
    unsigned long long *norms_p
        = reinterpret_cast<unsigned long long *>(region + (static_cast<std::size_t>(NP.n_pos) + NP.n_out) * LT * 2u
                                                 + static_cast<std::size_t>(NP.npp) * nbk::pair_mem<TT, OFFCHIP>::OPB / 8u);

    // ---- this thread's pair interaction ----
    nbk::pair_mem<TT, OFFCHIP> PM;
    nb::pair_consts PC;
    {
        const std::uint32_t n_pt = NP.n_pairs * LT;
        const bool active = tid < n_pt;
        // Idle threads shadow pair 0 / lane 0 (they skip the pair phase).
        const std::uint32_t pi = active ? tid / LT : 0u, l = active ? tid % LT : 0u;
        const uint4 *dp = reinterpret_cast<const uint4 *>(NP.pairs + pi);
        const uint4 w0 = __ldg(dp), w1 = __ldg(dp + 1), w2 = __ldg(dp + 2), w3 = __ldg(dp + 3);
        // u16 fields: pa[3] pb[3] om[3] on[3] = words w0.x .. w1.y; flags = w1.z; c1 = w2.xy; c2[3] = w2.zw, w3.xy, w3.zw
        const std::uint32_t h[6] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y};
        const auto u16 = [&](int i) { return (h[i >> 1] >> ((i & 1) * 16)) & 0xffffu; };
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            PM.pa[k] = pos_b + (u16(k) * LT + l) * 16u;
            PM.pb[k] = pos_b + (u16(3 + k) * LT + l) * 16u;
        }
        PM.om = out_b + (u16(6) * LT + l) * 16u; // om[k] = k * n_pairs + pair, on[k] = (3 + k) * n_pairs + pair
        PM.kstride = NP.n_pairs * LT * 16u;
        PM.flags = (active ? 1u : 0u);
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            if (active && u16(9 + k) != 0xffffu) {
                PM.flags |= 2u << k;
            }
        }
        PC.c1 = __hiloint2double(static_cast<int>(w2.y), static_cast<int>(w2.x));
        PC.c2[0] = __hiloint2double(static_cast<int>(w2.w), static_cast<int>(w2.z));
        PC.c2[1] = __hiloint2double(static_cast<int>(w3.y), static_cast<int>(w3.x));
        PC.c2[2] = __hiloint2double(static_cast<int>(w3.w), static_cast<int>(w3.z));
        PC.alpha = NP.alpha;
        PC.pow_algo = NP.pow_algo;
        PC.have_n = (w1.z & 1u) != 0u;
        PM.drow = drow_b + tid * 16u;
        PM.fac_ = nbk::saddr(fac_s);
        PM.fac_stride_b = NP.fac_stride * 8u;
        PM.grow = nullptr;
        if constexpr (OFFCHIP) {
            PM.grow = reinterpret_cast<double2 *>(NP.offchip)
                      + static_cast<std::size_t>(blockIdx.x) * NP.npp * 3u * TT + threadIdx.x;
        }
    }
    // ---- this thread's lanes in the summation phase ----
    const std::uint32_t l0 = (tid % GS) * NL;
    // (The 384- and 512-thread instantiations have no registers to spare for the maxima.)
    constexpr bool REGN = !CTA && MAXT <= 256;
    nbk::role_mem<NL, REGN> RM;
    RM.pos_b = pos_b;
    RM.out_b = out_b;
    RM.consts = nbk::saddr(consts_s);
    RM.rcp_ = nbk::saddr(rcp_s);
    constexpr std::uint32_t NC = detail::nb_norm_copies(LT);
    RM.norms = norms_b + ((tid % NC) * LT + l0) * 8u;
    RM.lt8 = NC * LT * 8u;
    RM.n_batch = D.n;
    RM.p = p;
    const std::size_t team_global = T::index();
    const coef_view cv{R.coef_base + team_global * R.coef_warp_stride, static_cast<std::size_t>(R.coef_stride_sv),
                       static_cast<std::size_t>(R.coef_stride_o), R.coef_pub != 0, !PROP && R.skip != nullptr};
    RM.stride_sv = cv.stride_sv;
    RM.stride_o = cv.stride_o;
    RM.pub = cv.pub;
    std::uint32_t roles_sa = nbk::saddr(roles_s) + tid * 32u;
    nbk::keep(roles_sa);
    nbk::keep(RM.consts);
    nbk::keep(RM.rcp_);
    nbk::keep(PM.fac_);
    const std::uint32_t n_rounds = NP.n_rounds, level_end = NP.round_level_end, roles_smem = NP.roles_in_smem;
    const uint4 *roles_g = NP.roles + tid * 2u;

    const std::uint32_t n_chunks = (D.n + LT - 1u) / LT;
    const bool owner = tid < LT;
    const std::uint32_t n_blocks = NP.npp;
    nb_phase_clock clk;
#if defined(HY_NB_PHASE_CLOCK)
    PM.clk = &clk;
    RM.clk = &clk;
#endif

    const auto load_role = [&](std::uint32_t rd, std::uint32_t (&w)[8]) {
        uint4 a, b;
        if (roles_smem != 0u) {
            a = nbk::lds4u(roles_sa + rd * (TT * 32u));
            b = nbk::lds4u(roles_sa + rd * (TT * 32u) + 16u);
        } else {
            a = __ldg(roles_g + static_cast<std::size_t>(rd) * (TT * 2u));
            b = __ldg(roles_g + static_cast<std::size_t>(rd) * (TT * 2u) + 1);
        }
        w[0] = a.x, w[1] = a.y, w[2] = a.z, w[3] = a.w, w[4] = b.x, w[5] = b.y, w[6] = b.z, w[7] = b.w;
    };

    double nm3[3] = {0., 0., 0.}; // REGN: the maxima of the owner's lane after a jet
    const auto jet = [&](std::uint32_t lane0) {
        // The thread's lanes: global indices (clamped), offsets into the coefficient store.
        {
            const std::uint32_t la = lane0 + l0, lb = la + (NL - 1);
            const std::uint32_t ga = la < D.n ? la : D.n - 1u, gb = lb < D.n ? lb : D.n - 1u;
            // (A step with a skip mask leaves the lanes that are not running untouched, tc included.)
            RM.lane_ok[0] = la < D.n && !(cv.mask_idle && S.running[l0] == 0);
            if constexpr (NL == 2) {
                RM.lane_ok[1] = lb < D.n && !(cv.mask_idle && S.running[l0 + 1] == 0);
            }
            RM.ldelta = gb - ga;
            RM.state0 = D.state + ga;
            RM.cbase = cv.base + cv.lane_off(ga, l0);
        }
        RM.track = true;
        RM.norms_reset();
        for (std::uint32_t rd = 0; rd < n_rounds; ++rd) {
            std::uint32_t w[8];
            load_role(rd, w);
            nb::role_init<NL>(RM, w);
        }
        T::sync();
        clk.lap(NB_PH_INIT);
        for (std::uint32_t m = 0; m < n_blocks; ++m) {
            if ((PM.flags & 1u) != 0u) {
                nb::pair_block(PM, PC, m);
            }
            T::sync();
            clk.lap(NB_PH_PAIR);
            RM.track = m + 2u >= n_blocks;
            for (std::uint32_t rd = 0; rd < n_rounds; ++rd) {
                std::uint32_t w[8];
                load_role(rd, w);
                clk.sub(NB_PH_SUM_ROLE);
                nb::role_block<NL>(RM, w, m, p);
                if (((level_end >> rd) & 1u) != 0u) {
                    T::sync();
                }
                clk.sub(NB_PH_SUM_STORE);
            }
            clk.lap(NB_PH_SUM);
        }
    };

    // Step size from the norms gathered during the jet; resets the norms. Every thread of the team calls it; the owner
    // threads get the step size of their lane.
    // PAIRED (warp teams of at most 16 lanes with the maxima in registers): the two radii of convergence of a lane are
    // computed side by side, the order-p one by the lane's owner tid and the order-(p - 1) one by thread tid + LT, in
    // the same instructions; a shuffle brings the second to the owner. The coefficients of state variable 0 that the
    // NaN rule reads are loaded before the shuffle reduction of the maxima, which hides their latency.
    constexpr bool PAIRED = REGN && 2 * LT <= 32;
    const auto step_size = [&](std::uint32_t lane0, double max_delta_t) {
        const std::uint32_t o = PAIRED ? tid % LT : tid; // the lane's owner
        const std::uint32_t lane_raw = lane0 + o, lane = lane_raw < D.n ? lane_raw : D.n - 1u;
        const double *c = cv.base + cv.lane_off(lane, o);
        if constexpr (PAIRED) {
            const bool ord_p = owner; // (threads beyond 2 LT repeat the order-(p - 1) radius of their lane)
            const double c0 = c[0], cq = c[(ord_p ? p : p - 1u) * cv.stride_o];
            RM.template norms_reduce<LT>(tid, nm3);
            const double rho = nb_rho(ord_p ? P.inv_p : P.inv_pm1, nm3[0], ord_p ? nm3[1] : nm3[2], c0, cq);
            const double rho_m1 = __shfl_down_sync(0xffffffffu, rho, LT);
            return h_from_rho(rho, rho_m1, P.rhofac, max_delta_t);
        } else {
            if constexpr (REGN) {
                RM.template norms_reduce<LT>(tid, nm3);
            }
            double h = 0.;
            if (owner) {
                h = nb_step_size(P.inv_p, P.inv_pm1, P.rhofac, REGN ? nullptr : norms_p + tid, LT, nm3[0], nm3[1],
                                 nm3[2], c, p * cv.stride_o, (p - 1u) * cv.stride_o, max_delta_t);
            }
            return h;
        }
    };
    if (owner) {
        for (std::uint32_t i = 0; i < 3u * NC; ++i) {
            norms_p[i * LT + tid] = 0ull;
        }
    }
    // The per-lane bookkeeping of propagate_until() is parked in shared memory while the jet runs (it would otherwise
    // hold ~26 registers of every thread across the hot loops).
    static_assert(sizeof(lane_prop) <= 128u && alignof(lane_prop) <= 8u);
    lane_prop *const park = reinterpret_cast<lane_prop *>(norms_p + 3u * NC * LT) + (owner ? tid : 0u);

    clk.start(team_global, !CTA && PROP && tid == 0u);
    for (std::uint32_t chunk = T::claim(R.counter); chunk < n_chunks; chunk = T::claim(R.counter)) {
        const std::uint32_t lane0 = chunk * LT;
        const std::uint32_t lane_raw = lane0 + tid;
        bool valid = owner && lane_raw < D.n;
        const std::uint32_t lane = (owner && lane_raw < D.n) ? lane_raw : D.n - 1u;

        if constexpr (!PROP) {
            if (owner) {
                const bool skipped = R.skip != nullptr && R.skip[lane] != 0u;
                valid = valid && !skipped;
                S.time[tid] = D.t_hi[lane];
                S.running[tid] = skipped ? 0 : 1;
            }
            T::sync();
            jet(lane0);
            double mdt = 0.;
            if (owner) {
                mdt = R.max_delta_t != nullptr ? R.max_delta_t[lane] : R.default_max_delta_t;
            }
            const double h = step_size(lane0, mdt);
            if (owner) {
                S.h[tid] = h;
            }
            T::sync();
            unsigned nf_mask = 0u;
            coop_update_state<LT, CTA>(P, D, S, cv, lane0, nf_mask);
            nf_mask = T::template reduce_or<LT>(nf_mask);
            if (valid) {
                const dfl nt = dfl_add(dfl{D.t_hi[lane], D.t_lo[lane]}, dfl{h, 0.});
                D.t_hi[lane] = nt.hi;
                D.t_lo[lane] = nt.lo;
                D.last_h[lane] = h;
                const bool nf = !(isfinite(nt.hi) && isfinite(nt.lo)) || ((nf_mask >> tid) & 1u) != 0u;
                D.step_outcome[lane]
                    = nf ? HY_OUTCOME_ERR_NF_STATE : (h == mdt ? HY_OUTCOME_TIME_LIMIT : HY_OUTCOME_SUCCESS);
            }
        } else {
            bool running = false;
            if (owner) {
                lane_prop lp;
                lp.init(D, R, lane);
                *park = lp;
                running = lp.running;
            }
            while (T::any(running)) {
                if (owner) {
                    S.time[tid] = park->t.hi;
                    S.running[tid] = running ? 1 : 0;
                }
                T::sync();
                clk.lap(NB_PH_PROP);
                clk.step();
                jet(lane0);
                double cur_max = 0.;
                if (owner) {
                    cur_max = park->cur_max();
                }
                const double h = step_size(lane0, cur_max);
                if (owner) {
                    S.h[tid] = h;
                }
                T::sync();
                clk.lap(NB_PH_STEP_SIZE);
                unsigned nf_mask = 0u;
                coop_update_state<LT, CTA>(P, D, S, cv, lane0, nf_mask);
                nf_mask = T::template reduce_or<LT>(nf_mask);
                clk.lap(NB_PH_UPDATE);
                if (running) {
                    lane_prop lp = *park;
                    lp.advance(h, cur_max, ((nf_mask >> tid) & 1u) != 0u, R, valid);
                    *park = lp;
                    running = lp.running;
                }
            }
            if (valid) {
                park->store(D, lane);
                park->report_iters(R);
            }
        }
        T::sync();
        clk.lap(NB_PH_PROP);
    }
    clk.finish();
}

} // namespace heyoka_b200::dev

#endif
