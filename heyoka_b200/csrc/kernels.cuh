// The sm_90a kernels of the batch Taylor integrator.
//
// k_coop (the product path): warp-cooperative. A warp owns L lanes and their compact derivative tape ([slot][L]
//   doubles; only what is re-read at later orders keeps its history, see smem_plan.hpp). Its 32 threads share the
//   work of every dependency level: one work item = one u variable (or one superinstruction, fused.cuh) x N
//   adjacent lanes; items of a level are independent, a __syncwarp() separates levels and orders (the structure of
//   the reference's compact mode, src/taylor_02.cpp:1147-1185, with its parallel mode's idea of spreading a
//   segment over workers, src/taylor_01.cpp:1220-1247). Warps are persistent, claim groups of L lanes from an
//   atomic counter and run a group's whole propagate_until() loop in one go; they never wait for each other.
//   Where the tape lives is the kernel's MODE:
//     0 / 1  shared memory (0: superinstruction-only programs, no interpreter of the elementary recurrences);
//     4 / 5  a slab of global memory per team, tables read in place (systems too large for shared memory);
//            4: a team is a warp, 5: a team is the whole CTA (wide levels, few lanes; see team<>).
//   HBM traffic per step: the state in and out (the state variables' coefficients go to a private L2-resident
//   store, or to the public tc array on request).
//
// k_hbm (the first kernel of the round, kept selectable): one thread per lane, a warp owns 32 consecutive lanes,
//   every access is a coalesced 256-byte row of the warp's private slab in HBM.
//
// Replaces: the JIT'd step function (src/taylor_00.cpp:712-865), step_impl() bookkeeping
// (src/taylor_adaptive_batch.cpp:632-727), propagate_until_impl() (:1136-1534), d_out_f
// (src/taylor_01.cpp:1015-1185).
#ifndef HEYOKA_B200_CSRC_KERNELS_CUH
#define HEYOKA_B200_CSRC_KERNELS_CUH

#include <cstdint>

#include <cuda_runtime.h>
#include <math_constants.h>

#include "device_program.cuh"
#include "recurrences.cuh"
#include "fused.cuh"

namespace heyoka_b200::dev
{

// Arguments of a step / propagate launch.
struct run_args {
    // step
    const double *max_delta_t; // per lane, or nullptr
    double default_max_delta_t;
    // propagate
    const double *tf_hi, *tf_lo;
    unsigned long long iter_cap; // 0 = unlimited
    int replay;
    int write_tc;
    run_flags *flags;
    unsigned int *counter;
    // Cooperative kernels: where the state variables' coefficients of the current step go (dev::coef_view). Either
    // the public tc array (coef_pub = 1, warp stride 0) or a private store of coef_warp_stride doubles per warp,
    // used when write_tc == 0. Filled in by hy_batch::launch().
    double *coef_base;
    unsigned long long coef_warp_stride, coef_stride_sv, coef_stride_o;
    int coef_pub;
    // step: lanes flagged here are left untouched (no state, time, outcome or tc write). Used for the zero-length
    // re-expansion of the lanes that finished a propagate_until() early (see batch.cu::propagate_finish()).
    const unsigned char *skip;
};

// ================================================================================================
// Per-lane bookkeeping shared by both strategies.
// ================================================================================================

// State of one lane inside propagate_until() (src/taylor_adaptive_batch.cpp:1256-1273, :1402-1460).
struct lane_prop {
    dfl t, rem, tf;
    double mdt, min_h, max_h, last_h;
    unsigned long long ts_count, iter;
    long long outcome;
    bool dir, running;

    __device__ __forceinline__ void init(const batch &D, const run_args &R, std::uint32_t lane)
    {
        tf = dfl{R.tf_hi[lane], R.tf_lo != nullptr ? R.tf_lo[lane] : 0.};
        mdt = R.max_delta_t != nullptr ? R.max_delta_t[lane] : CUDART_INF;
        t = dfl{D.t_hi[lane], D.t_lo[lane]};
        rem = dfl_sub(tf, t);
        dir = dfl_ge0(rem); // fixed at the start
        ts_count = 0;
        iter = 0;
        min_h = CUDART_INF;
        max_h = 0.;
        last_h = 0.;
        outcome = HY_OUTCOME_TIME_LIMIT;
        running = true;
    }

    // The signed limit of the next step; 0 for a lane that is done (zero-length step, nothing written).
    __device__ __forceinline__ double cur_max() const
    {
        return running ? step_limit(dir, rem, mdt) : 0.;
    }

    // After a step of size h (state already written); nf = non-finite state detected.
    __device__ __forceinline__ void advance(double h, double used_max, bool state_nf, const run_args &R, bool valid)
    {
        t = dfl_add(t, dfl{h, 0.});
        last_h = h;
        ++iter;
        const bool nf = !(isfinite(t.hi) && isfinite(t.lo)) || state_nf;
        if (nf) {
            outcome = HY_OUTCOME_ERR_NF_STATE;
            running = false;
            if (valid) {
                atomicOr(&R.flags->any_nf, 1u);
                atomicMin(&R.flags->min_nf_iter, iter);
            }
            return;
        }
        const bool time_limit = (h == used_max);
        outcome = time_limit ? HY_OUTCOME_TIME_LIMIT : HY_OUTCOME_SUCCESS;
        ts_count += (h != 0.) ? 1u : 0u;
        if (!time_limit) {
            const double ah = fabs(h);
            min_h = fmin(min_h, ah);
            max_h = fmax(max_h, ah);
        }
        if (h == rem.hi) {
            // Final time reached (the outcome is necessarily time_limit).
            rem = dfl{0., 0.};
            running = false;
        } else {
            rem = dfl_sub(tf, t);
            if (iter == R.iter_cap) {
                running = false;
                if (!R.replay) {
                    outcome = HY_OUTCOME_STEP_LIMIT;
                    if (valid) {
                        atomicOr(&R.flags->any_limit, 1u);
                    }
                }
            }
        }
    }

    __device__ __forceinline__ void store(const batch &D, std::uint32_t lane) const
    {
        D.t_hi[lane] = t.hi;
        D.t_lo[lane] = t.lo;
        D.last_h[lane] = last_h;
        D.prop_outcome[lane] = outcome;
        D.prop_min_h[lane] = min_h;
        D.prop_max_h[lane] = max_h;
        D.prop_n_steps[lane] = ts_count;
        D.prop_iters[lane] = iter;
    }
    // (Separate from store(): needs the launch's flags.)
    __device__ __forceinline__ void report_iters(const run_args &R) const
    {
        atomicMax(&R.flags->max_iter, iter);
    }
};

__device__ __forceinline__ bool lane_state_nonfinite(const program &P, const batch &D, std::uint32_t lane)
{
    bool nf = false;
    for (std::uint32_t i = 0; i < P.n_eq; ++i) {
        nf = nf || !isfinite(D.state[static_cast<std::size_t>(i) * D.n + lane]);
    }
    return nf;
}

// ================================================================================================
// "hbm" strategy.
// ================================================================================================
struct hbm_tape {
    double *base; // warp slab + lane-in-warp
    std::uint32_t pp1;
    const double *pars;
    std::uint32_t batch, lane;
    double tm;
    const std::uint32_t *args;
    const double *consts;

    __device__ __forceinline__ std::uint32_t arg(std::uint32_t i) const
    {
        return __ldg(args + i);
    }
    __device__ __forceinline__ double cst(std::uint32_t i) const
    {
        return __ldg(consts + i);
    }

    struct row_t {
        double *p;
        static constexpr std::uint32_t stride = 32u;
        __device__ __forceinline__ static vd<1> load(const double *q)
        {
            return vd<1>{{*q}};
        }
        __device__ __forceinline__ const double *hptr(std::uint32_t o) const
        {
            return p + static_cast<std::size_t>(o) * 32u;
        }
        __device__ __forceinline__ vd<1> at(std::uint32_t o) const
        {
            return vd<1>{{p[static_cast<std::size_t>(o) * 32u]}};
        }
        __device__ __forceinline__ void set(std::uint32_t o, const vd<1> &v) const
        {
            p[static_cast<std::size_t>(o) * 32u] = v.v[0];
        }
    };
    __device__ __forceinline__ row_t row(std::uint32_t u) const
    {
        return row_t{base + static_cast<std::size_t>(u) * pp1 * 32u};
    }
    __device__ __forceinline__ vd<1> par(std::uint32_t idx) const
    {
        return vd<1>{{__ldg(pars + static_cast<std::size_t>(idx) * batch + lane)}};
    }
    __device__ __forceinline__ vd<1> time() const
    {
        return vd<1>{{tm}};
    }
};

// The whole jet of the lane: orders 0..p-1 of every u variable, order p of the state variables
// (evaluation order of src/taylor_02.cpp:1147-1185: per order, state variables first, then the others).
__device__ __forceinline__ void hbm_jet(const program &P, const hbm_tape &t, const double *state)
{
    for (std::uint32_t i = 0; i < P.n_eq; ++i) {
        t.row(i).set(0u, vd<1>{{state[static_cast<std::size_t>(i) * t.batch + t.lane]}});
    }
    for (std::uint32_t n = 0; n < P.order; ++n) {
        if (n > 0u) {
            const double nd = static_cast<double>(n), rcp = 1. / nd;
            for (std::uint32_t i = 0; i < P.n_eq; ++i) {
                t.row(i).set(n, sv_diff<1>(P, t, __ldg(P.sv_defs + i), n, nd, rcp));
            }
        }
        for (std::uint32_t k = 0; k < P.n_ops; ++k) {
            const uint4 op = __ldg(P.ops + k);
            const auto self = t.row(P.n_eq + k);
            self.set(n, diff_op<1>(P, t, op, self, n));
        }
    }
    {
        const double nd = static_cast<double>(P.order), rcp = 1. / nd;
        for (std::uint32_t i = 0; i < P.n_eq; ++i) {
            t.row(i).set(P.order, sv_diff<1>(P, t, __ldg(P.sv_defs + i), P.order, nd, rcp));
        }
    }
}

__device__ __forceinline__ double hbm_determine_h(const program &P, const hbm_tape &t, double max_delta_t)
{
    const std::uint32_t p = P.order;
    double m0, mp, mp1;
    {
        const auto r = t.row(0);
        m0 = fabs(r.at(0).v[0]);
        mp = fabs(r.at(p).v[0]);
        mp1 = fabs(r.at(p - 1u).v[0]);
    }
    for (std::uint32_t i = 1; i < P.n_eq; ++i) {
        const auto r = t.row(i);
        m0 = std_max(m0, fabs(r.at(0).v[0]));
        mp = std_max(mp, fabs(r.at(p).v[0]));
        mp1 = std_max(mp1, fabs(r.at(p - 1u).v[0]));
    }
    return h_from_norms(P, m0, mp, mp1, max_delta_t);
}

__device__ __forceinline__ void hbm_update_state(const program &P, const hbm_tape &t, double h, double *state, double *tc,
                                                 bool write)
{
    const std::uint32_t pp1 = P.order + 1u;
    for (std::uint32_t i = 0; i < P.n_eq; ++i) {
        const auto r = t.row(i);
        const double res = eval_poly(P, [&r](std::uint32_t o) { return r.at(o).v[0]; }, h);
        if (write) {
            state[static_cast<std::size_t>(i) * t.batch + t.lane] = res;
            if (tc != nullptr) {
                for (std::uint32_t o = 0; o < pp1; ++o) {
                    tc[(static_cast<std::size_t>(i) * pp1 + o) * t.batch + t.lane] = r.at(o).v[0];
                }
            }
        }
    }
}

__device__ __forceinline__ std::uint32_t claim_chunk_warp(unsigned int *counter)
{
    unsigned int c = 0;
    if ((threadIdx.x & 31u) == 0u) {
        c = atomicAdd(counter, 1u);
    }
    return __shfl_sync(0xffffffffu, c, 0);
}

// The threads that work together on one chunk of L lanes: a warp (the default) or, for systems with hundreds of
// independent items per level and too few lanes to fill the GPU with warps, the whole CTA (kernel MODE 5: the
// latency of a lane-step drops by the number of warps, and the tapes in flight nearly fit in L2).
template <bool CTA>
struct team {
    __device__ __forceinline__ static std::uint32_t tid()
    {
        return CTA ? threadIdx.x : (threadIdx.x & 31u);
    }
    __device__ __forceinline__ static std::uint32_t size()
    {
        return CTA ? blockDim.x : 32u;
    }
    // Index of the team in the grid (slab / private store index).
    __device__ __forceinline__ static std::size_t index()
    {
        return CTA ? static_cast<std::size_t>(blockIdx.x)
                   : ((static_cast<std::size_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5);
    }
    __device__ __forceinline__ static void sync()
    {
        if constexpr (CTA) {
            __syncthreads();
        } else {
            __syncwarp();
        }
    }
    __device__ __forceinline__ static bool any(bool pred)
    {
        if constexpr (CTA) {
            return __syncthreads_or(pred ? 1 : 0) != 0;
        } else {
            return __any_sync(0xffffffffu, pred) != 0;
        }
    }
    // Bitwise OR of a per-lane mask (bit l = lane l) over the team.
    template <int L>
    __device__ __forceinline__ static unsigned reduce_or(unsigned mask)
    {
        if constexpr (CTA) {
            unsigned r = 0u;
#pragma unroll
            for (int l = 0; l < L; ++l) {
                r |= __syncthreads_or(static_cast<int>((mask >> l) & 1u)) != 0 ? (1u << l) : 0u;
            }
            return r;
        } else {
            return __reduce_or_sync(0xffffffffu, mask);
        }
    }
    __device__ __forceinline__ static std::uint32_t claim(unsigned int *counter)
    {
        if constexpr (CTA) {
            __shared__ unsigned int claimed;
            if (threadIdx.x == 0u) {
                claimed = atomicAdd(counter, 1u);
            }
            __syncthreads();
            const unsigned int c = claimed;
            __syncthreads();
            return c;
        } else {
            return claim_chunk_warp(counter);
        }
    }
};

template <bool PROP>
__global__ void __launch_bounds__(256) k_hbm(program P, batch D, run_args R, double *scratch, std::size_t slab_doubles)
{
    const std::uint32_t lane_in_warp = threadIdx.x & 31u;
    const std::size_t warp_global = (static_cast<std::size_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    double *slab = scratch + warp_global * slab_doubles + lane_in_warp;
    const std::uint32_t n_chunks = (D.n + 31u) / 32u;

    for (std::uint32_t chunk = claim_chunk_warp(R.counter); chunk < n_chunks; chunk = claim_chunk_warp(R.counter)) {
        const std::uint32_t lane_raw = chunk * 32u + lane_in_warp;
        bool valid = lane_raw < D.n;
        const std::uint32_t lane = valid ? lane_raw : D.n - 1u;
        if constexpr (!PROP) {
            valid = valid && !(R.skip != nullptr && R.skip[lane] != 0u);
        }
        hbm_tape tape{slab, P.order + 1u, D.pars, D.n, lane, 0., P.args, P.consts};

        if constexpr (!PROP) {
            const double mdt = R.max_delta_t != nullptr ? R.max_delta_t[lane] : R.default_max_delta_t;
            const dfl t0{D.t_hi[lane], D.t_lo[lane]};
            tape.tm = t0.hi;
            hbm_jet(P, tape, D.state);
            const double h = hbm_determine_h(P, tape, mdt);
            hbm_update_state(P, tape, h, D.state, R.write_tc ? D.tc : nullptr, valid);
            if (valid) {
                const dfl nt = dfl_add(t0, dfl{h, 0.});
                D.t_hi[lane] = nt.hi;
                D.t_lo[lane] = nt.lo;
                D.last_h[lane] = h;
                const bool nf = !(isfinite(nt.hi) && isfinite(nt.lo)) || lane_state_nonfinite(P, D, lane);
                D.step_outcome[lane]
                    = nf ? HY_OUTCOME_ERR_NF_STATE : (h == mdt ? HY_OUTCOME_TIME_LIMIT : HY_OUTCOME_SUCCESS);
            }
        } else {
            lane_prop lp;
            lp.init(D, R, lane);
            while (__any_sync(0xffffffffu, lp.running)) {
                // A lane that is done takes a zero-length step: the jet is computed (the warp stays
                // converged) but nothing is written.
                const double cur_max = lp.cur_max();
                tape.tm = lp.t.hi;
                hbm_jet(P, tape, D.state);
                const double h = hbm_determine_h(P, tape, cur_max);
                hbm_update_state(P, tape, h, D.state, R.write_tc ? D.tc : nullptr, lp.running && valid);
                if (lp.running) {
                    lp.advance(h, cur_max, lane_state_nonfinite(P, D, lane), R, valid);
                }
            }
            if (valid) {
                lp.store(D, lane);
                lp.report_iters(R);
            }
        }
    }
}

// ================================================================================================
// "coop" strategy: warp-cooperative, tape in shared memory.
// A warp owns L lanes and a private slice of shared memory; its 32 threads are (32 / G) workers x G lane
// groups of N lanes (G = L / N). Levels and orders are separated by __syncwarp() only: warps never wait
// for each other, the SM interleaves them. The program tables (ops, argument tables, constants) are copied
// once per CTA into shared memory, so that no global-memory latency sits on the per-item critical path.
// ================================================================================================

// Word offsets into the plan blob (see make_plan_blob() in batch.cu); the blob starts with this header.
struct coop_header {
    std::uint32_t n_words, n_items, n_segments, n_eq;
    std::uint32_t off_ops, off_seg, off_args, off_aux;
    std::uint32_t off_consts, off_sv, n_slots, off_svout;
    std::uint32_t off_svphase, n_svphase, off_rcp, n_gslots;
    std::uint32_t reserved0, reserved1, reserved2, reserved3;
};

template <int L, int N>
struct smem_tape {
    double *base;  // the warp's tape + first lane of this thread's group
    double *gbase; // idem for the overflow tape in global memory (nullptr if unused)
    const std::uint32_t *args;
    const double *consts;
    const double *pars;
    std::uint32_t batch;
    std::uint32_t glane[N]; // global lane indices (clamped to valid lanes)
    vd<N> tm;

    __device__ __forceinline__ std::uint32_t arg(std::uint32_t i) const
    {
        return args[i];
    }
    __device__ __forceinline__ double cst(std::uint32_t i) const
    {
        return consts[i];
    }

    struct row_t {
        double *p;
        std::uint32_t mask;
        static constexpr std::uint32_t stride = L;
        __device__ __forceinline__ static vd<N> load(const double *q)
        {
            vd<N> r;
            if constexpr (N == 2) {
                const double2 x = *reinterpret_cast<const double2 *>(q);
                r.v[0] = x.x;
                r.v[1] = x.y;
            } else if constexpr (N == 4) {
                const double2 x = *reinterpret_cast<const double2 *>(q);
                const double2 y = *reinterpret_cast<const double2 *>(q + 2);
                r.v[0] = x.x;
                r.v[1] = x.y;
                r.v[2] = y.x;
                r.v[3] = y.y;
            } else {
#pragma unroll
                for (int i = 0; i < N; ++i) {
                    r.v[i] = q[i];
                }
            }
            return r;
        }
        __device__ __forceinline__ static void store(double *q, const vd<N> &v)
        {
            if constexpr (N == 2) {
                *reinterpret_cast<double2 *>(q) = make_double2(v.v[0], v.v[1]);
            } else if constexpr (N == 4) {
                *reinterpret_cast<double2 *>(q) = make_double2(v.v[0], v.v[1]);
                *reinterpret_cast<double2 *>(q + 2) = make_double2(v.v[2], v.v[3]);
            } else {
#pragma unroll
                for (int i = 0; i < N; ++i) {
                    q[i] = v.v[i];
                }
            }
        }
        // Address of the order-o coefficient of a HISTORY row (convolution operands always are).
        __device__ __forceinline__ const double *hptr(std::uint32_t o) const
        {
            return p + o * L;
        }
        __device__ __forceinline__ vd<N> at(std::uint32_t o) const
        {
            return load(p + (o & mask) * L);
        }
        __device__ __forceinline__ void set(std::uint32_t o, const vd<N> &v) const
        {
            store(p + (o & mask) * L, v);
        }
    };
    // ref = (mask code << 27) | first slot (see smem_plan.hpp): mask = sign extension of the 3-bit code.
    __device__ __forceinline__ row_t row(std::uint32_t ref) const
    {
        const std::uint32_t mask = static_cast<std::uint32_t>(static_cast<std::int32_t>(ref << 2) >> 29);
        return row_t{base + (ref & 0x7ffffffu) * L, mask};
    }
    // A row known to be a history row / a single-slot row (superinstructions): no mask decoding.
    __device__ __forceinline__ row_t hrow(std::uint32_t ref) const
    {
        return row_t{base + (ref & 0x7ffffffu) * L, 0xffffffffu};
    }
    // A history row of the overflow tape.
    __device__ __forceinline__ row_t grow(std::uint32_t ref) const
    {
        return row_t{gbase + (ref & 0x7ffffffu) * L, 0xffffffffu};
    }
    __device__ __forceinline__ vd<N> par(std::uint32_t idx) const
    {
        vd<N> r;
#pragma unroll
        for (int i = 0; i < N; ++i) {
            r.v[i] = __ldg(pars + static_cast<std::size_t>(idx) * batch + glane[i]);
        }
        return r;
    }
    __device__ __forceinline__ vd<N> time() const
    {
        return tm;
    }
};

// Shared memory of one warp: tape[n_slots][L], then per-lane scalars.
template <int L>
struct coop_smem {
    double *tape;
    double *time, *h;
    int *running;

    __device__ __forceinline__ coop_smem(double *warp_region, std::uint32_t n_slots)
    {
        tape = warp_region;
        time = tape + static_cast<std::size_t>(n_slots) * L;
        h = time + L;
        running = reinterpret_cast<int *>(h + L);
    }
    // Doubles of shared memory per warp (tape + scalars, kept 16-byte aligned).
    __host__ __device__ static constexpr std::size_t warp_doubles(std::uint32_t n_slots)
    {
        return (static_cast<std::size_t>(n_slots) * L + 2u * L + (L + 1u) / 2u + 1u) / 2u * 2u;
    }
};

// Where the state variables' coefficients of the current step go (they are needed once more, for the step size
// and the state update): the public tc array, [(sv * (p + 1) + o) * batch + lane], when the caller asked for it
// (write_tc), otherwise a private per-warp store [(o * n_eq + sv) * L + l] that stays in L2 and is read back with
// contiguous accesses. One addressing formula serves both: base + sv * stride_sv + o * stride_o + lane offset.
struct coef_view {
    double *base;
    std::size_t stride_sv, stride_o;
    bool pub;
    bool mask_idle = false; // lanes that are not running do not write to the store either (step with a skip mask)
    __device__ __forceinline__ std::size_t lane_off(std::uint32_t glane, std::uint32_t l) const
    {
        return pub ? glane : l;
    }
};

// Writes of state-variable coefficients: into the tape row and, streamed, into the coefficient store.
template <int L, int N>
struct sv_writer {
    const smem_tape<L, N> &t;
    coef_view cv;
    const std::uint32_t *svout;
    const double *rcp;
    std::uint32_t p;
    std::size_t loff[N]; // lane offsets into the coefficient store
    bool lane_ok[N];

    // Stream the coefficient of state variable sv at order n (valid lanes only).
    __device__ __forceinline__ void write_tc(std::uint32_t sv, std::uint32_t n, const vd<N> &v) const
    {
        double *dst = cv.base + sv * cv.stride_sv + n * cv.stride_o;
#pragma unroll
        for (int i = 0; i < N; ++i) {
            if (lane_ok[i]) {
                dst[loff[i]] = v.v[i];
            }
        }
    }
    // State variables whose derivative is the value v = u^[n] just produced: x^[n+1] = v / (n + 1), and
    // x2^[n+2] = x^[n+1] / (n + 2) for the state variables x2 that derive from x (see smem_plan.hpp).
    // (Must stay inline: an out-of-line call would force the tape object into local memory.)
    __device__ __forceinline__ void operator()(std::uint32_t off, const vd<N> &v, std::uint32_t n) const
    {
        const std::uint32_t *so = svout + off;
        const std::uint32_t cnt = so[0];
        vd<N> v1 = v;
        for (std::uint32_t e = 0; e < cnt; ++e) {
            const std::uint32_t sv = so[1u + 3u * e], rw = so[2u + 3u * e], depth = so[3u + 3u * e];
            if (depth == 1u) {
                v1 = div_small_int(v, n + 1u, static_cast<double>(n + 1u), rcp[n + 1u]);
                t.row(rw).set(n + 1u, v1);
                write_tc(sv, n + 1u, v1);
            } else if (n + 2u <= p) {
                const vd<N> v2 = div_small_int(v1, n + 2u, static_cast<double>(n + 2u), rcp[n + 2u]);
                t.row(rw).set(n + 2u, v2);
                write_tc(sv, n + 2u, v2);
            }
        }
    }
};

// Jet of the L lanes starting at global lane `lane0`; the state variables' coefficients go to tc.
// MODE: 1 = the program contains elementary ops; 0 = superinstructions only (the interpreter of the elementary
// recurrences is compiled out, which keeps the hot code small); 4 / 5 = tape in global memory.
template <int L, int N, int MODE>
__device__ __forceinline__ void coop_jet(const program &P, const coop_header &H, const std::uint32_t *tab,
                                         const batch &D, const coop_smem<L> &S, std::uint32_t lane0, double *gtape,
                                         const coef_view &cv)
{
    constexpr bool GEN = MODE == 1 || MODE == 4 || MODE == 5;
    using T = team<MODE == 5>;
    constexpr std::uint32_t G = L / N; // lane groups per warp
    const std::uint32_t tid = T::tid();
    const std::uint32_t nthr = T::size();
    const std::uint32_t p = P.order;
    const uint4 *ops = reinterpret_cast<const uint4 *>(tab + H.off_ops);
    const std::uint32_t *seg = tab + H.off_seg;
    const std::uint32_t *aux = tab + H.off_aux;
    const std::uint32_t *svout = tab + H.off_svout;
    const std::uint32_t *svphase = tab + H.off_svphase;
    const double *rcp = reinterpret_cast<const double *>(tab + H.off_rcp);
    const uint4 *svt = reinterpret_cast<const uint4 *>(tab + H.off_sv); // {row, rhs reference, cover, parent}

    // This thread always works on the same lane group: g = tid % G.
    smem_tape<L, N> t;
    const std::uint32_t g = tid % G;
    t.base = S.tape + g * N;
    t.gbase = gtape != nullptr ? gtape + g * N : nullptr;
    t.args = tab + H.off_args;
    t.consts = reinterpret_cast<const double *>(tab + H.off_consts);
    t.pars = D.pars;
    t.batch = D.n;
    bool lane_ok[N];
#pragma unroll
    for (int i = 0; i < N; ++i) {
        const std::uint32_t l = lane0 + g * N + i;
        lane_ok[i] = l < D.n && !(cv.mask_idle && S.running[g * N + i] == 0);
        t.glane[i] = l < D.n ? l : D.n - 1u;
        t.tm.v[i] = S.time[g * N + i];
    }
    sv_writer<L, N> sv_out_{t, cv, svout, rcp, p, {}, {}};
#pragma unroll
    for (int i = 0; i < N; ++i) {
        sv_out_.lane_ok[i] = lane_ok[i];
        sv_out_.loff[i] = cv.lane_off(t.glane[i], g * N + i);
    }
    const sv_writer<L, N> &sv_out = sv_out_;
    const auto write_tc = [&](std::uint32_t sv, std::uint32_t n, const vd<N> &v) { sv_out.write_tc(sv, n, v); };

    // Order 0 of the state variables: the state itself; order 1 of those that derive from another state
    // variable (x^[1] = v^[0]). (it % G == g because nthr is a multiple of G.)
    for (std::uint32_t it = tid; it < P.n_eq * G; it += nthr) {
        const std::uint32_t sv = it / G;
        const uint4 e = svt[sv];
        vd<N> v;
#pragma unroll
        for (int i = 0; i < N; ++i) {
            v.v[i] = D.state[static_cast<std::size_t>(sv) * D.n + t.glane[i]];
        }
        const auto r = t.row(e.x);
        r.set(0u, v);
        write_tc(sv, 0u, v);
        if (e.z == 2u) {
            vd<N> vp;
#pragma unroll
            for (int i = 0; i < N; ++i) {
                vp.v[i] = D.state[static_cast<std::size_t>(e.w) * D.n + t.glane[i]];
            }
            r.set(1u, vp);
            write_tc(sv, 1u, vp);
        }
    }
    T::sync();

    // The generic per-order pass for the state variables that no producer takes care of.
    const auto sv_pass = [&](std::uint32_t n) {
        const double nd = static_cast<double>(n), rc = rcp[n];
        for (std::uint32_t it = tid; it < H.n_svphase * G; it += nthr) {
            const std::uint32_t sv = svphase[it / G];
            const uint4 e = svt[sv];
            const vd<N> v = sv_diff<N>(P, t, e.y, n, nd, rc);
            t.row(e.x).set(n, v);
            write_tc(sv, n, v);
        }
        T::sync();
    };

    for (std::uint32_t n = 0; n < p; ++n) {
        if (n > 0u && H.n_svphase != 0u) {
            sv_pass(n);
        }
        // The other u variables, one dependency level at a time.
        for (std::uint32_t s = 0; s < H.n_segments; ++s) {
            const std::uint32_t b = seg[s], e = seg[s + 1u];
            for (std::uint32_t it = tid; it < (e - b) * G; it += nthr) {
                const std::uint32_t k = b + it / G;
                const uint4 op = ops[2u * k];
                if (op.x == FOP_NBODY_PAIR) {
                    if (H.n_gslots != 0u) {
                        fused_nbody_pair<N, true>(P, t, aux + op.y, op.z, op.w != 0u, n, sv_out);
                    } else {
                        fused_nbody_pair<N, false>(P, t, aux + op.y, op.z, op.w != 0u, n, sv_out);
                    }
                } else {
                    const uint4 op2 = ops[2u * k + 1u];
                    const auto self = t.row(op2.x);
                    vd<N> v;
                    if (!GEN || op.x == FOP_SUM_T) {
                        v = sum_single_slot<N>(t, op.y, op.z);
                    } else if constexpr (GEN) {
                        v = diff_op<N>(P, t, op, self, n);
                    }
                    self.set(n, v);
                    if (op2.y != 0u) {
                        sv_out(op2.y, v, n);
                    }
                }
            }
            T::sync();
        }
    }
    if (H.n_svphase != 0u) {
        sv_pass(p);
    }
}

// Step-size estimate of the warp's lanes from the coefficients streamed to tc: the three infinity norms are
// gathered by the whole warp (thread -> lane tid % L, state variables tid / L, tid / L + 32 / L, ...) and
// reduced with shuffles; the owner threads (tid < L) get the step size of lane tid.
// The sequential reference loop m = (m < |x|) ? |x| : m, started from |x_0|, yields NaN iff x_0 is NaN and
// ignores every other NaN: that is fmax() over all the elements plus a check of the first one.
template <int L>
__device__ __forceinline__ double coop_determine_h(const program &P, const batch &D, const coef_view &cv,
                                                   std::uint32_t lane0, double max_delta_t)
{
    const std::uint32_t tid = threadIdx.x & 31u, l = tid % L;
    const std::uint32_t p = P.order;
    const std::uint32_t glane = lane0 + l < D.n ? lane0 + l : D.n - 1u;
    const double *tc = cv.base + cv.lane_off(glane, l);
    const std::size_t so = cv.stride_o;
    double m0 = 0., mp = 0., mp1 = 0.;
    for (std::uint32_t sv = tid / L; sv < P.n_eq; sv += 32u / L) {
        const double *c = tc + sv * cv.stride_sv;
        m0 = fmax(m0, fabs(c[0]));
        mp = fmax(mp, fabs(c[p * so]));
        mp1 = fmax(mp1, fabs(c[(p - 1u) * so]));
    }
#pragma unroll
    for (std::uint32_t off = 16u; off >= L; off >>= 1) {
        m0 = fmax(m0, __shfl_xor_sync(0xffffffffu, m0, off));
        mp = fmax(mp, __shfl_xor_sync(0xffffffffu, mp, off));
        mp1 = fmax(mp1, __shfl_xor_sync(0xffffffffu, mp1, off));
    }
    double h = 0.;
    if (tid < L) {
        // (tid < L: this thread handled state variable 0 of its lane.)
        const double f0 = fabs(tc[0]), fp = fabs(tc[p * so]), fp1 = fabs(tc[(p - 1u) * so]);
        h = h_from_norms(P, isnan(f0) ? f0 : m0, isnan(fp) ? fp : mp, isnan(fp1) ? fp1 : mp1, max_delta_t);
    }
    return h;
}

// State update of the warp's lanes: item = (state variable, lane); S.h holds the step sizes, S.running
// which lanes may be written. Sets bit l of nf_mask if this thread produced a non-finite value for lane l.
// A thread evaluates up to three polynomials side by side (their coefficients come from L2).
template <int L, bool CTA = false>
__device__ __forceinline__ void coop_update_state(const program &P, const batch &D, const coop_smem<L> &S,
                                                  const coef_view &cv, std::uint32_t lane0, unsigned &nf_mask)
{
    constexpr int K = 3;
    const std::uint32_t tid = CTA ? threadIdx.x : (threadIdx.x & 31u), nthr = CTA ? blockDim.x : 32u;
    const std::uint32_t l = tid % L, n_items = P.n_eq * L;
    const std::uint32_t glane_raw = lane0 + l;
    const bool lane_active = glane_raw < D.n && S.running[l] != 0;
    const std::uint32_t glane = glane_raw < D.n ? glane_raw : D.n - 1u;
    const double h = S.h[l];
    const std::size_t n = D.n;
    for (std::uint32_t base = tid; base < n_items; base += nthr * K) {
        const double *c[K];
        bool act[K];
#pragma unroll
        for (int k = 0; k < K; ++k) {
            const std::uint32_t it = base + nthr * static_cast<std::uint32_t>(k);
            act[k] = it < n_items;
            const std::uint32_t sv = act[k] ? it / L : 0u;
            c[k] = cv.base + sv * cv.stride_sv + cv.lane_off(glane, l);
        }
        double res[K];
        eval_poly_k<K>(P, c, cv.stride_o, h, res);
#pragma unroll
        for (int k = 0; k < K; ++k) {
            if (act[k] && lane_active) {
                const std::uint32_t sv = (base + nthr * static_cast<std::uint32_t>(k)) / L;
                D.state[static_cast<std::size_t>(sv) * n + glane] = res[k];
                if (!isfinite(res[k])) {
                    nf_mask |= 1u << l;
                }
            }
        }
    }
}

// MAXT: upper bound on the threads per CTA. With at most 8 resident warps (tapes of more than ~14 KB per warp)
// the 256-thread instantiation lets the compiler use up to 255 registers per thread instead of 128.
template <int L, int N, bool PROP, int MAXT, int MODE>
__global__ void __launch_bounds__(MAXT, 1)
    k_coop(program P, const std::uint32_t *blob, batch D, run_args R, double *gscratch)
{
    // MODE 4: systems whose compact tape does not fit in shared memory. Same kernel, but the warp's tape lives in
    // a per-warp slab of global memory (gscratch) and the program tables are read in place (L1 / L2).
    constexpr bool GLOBAL = MODE == 4 || MODE == 5;
    // MODE 5: idem, and the whole CTA works on one chunk of lanes (see team<>).
    constexpr bool CTA = MODE == 5;
    using T = team<CTA>;
    extern __shared__ __align__(16) double smem_raw[];
    const std::uint32_t n_words = __ldg(blob);
    const std::uint32_t *tab = blob;
    if constexpr (!GLOBAL) {
        // Program tables: global -> shared, once per CTA.
        std::uint32_t *stab = reinterpret_cast<std::uint32_t *>(smem_raw);
        for (std::uint32_t i = threadIdx.x; i < n_words; i += blockDim.x) {
            stab[i] = __ldg(blob + i);
        }
        tab = stab;
    }
    __syncthreads();
    const coop_header H = *reinterpret_cast<const coop_header *>(tab);

    const std::uint32_t tid = T::tid();
    const std::size_t warp_global = T::index();
    // Shared memory: tables rounded up to 16 bytes, then one region per warp. Global mode: one slab per warp.
    const std::size_t tab_doubles = static_cast<std::size_t>(n_words + 3u) / 4u * 2u;
    const coop_smem<L> S(GLOBAL ? gscratch + warp_global * coop_smem<L>::warp_doubles(H.n_slots)
                                : smem_raw + tab_doubles
                                      + static_cast<std::size_t>(threadIdx.x >> 5)
                                            * coop_smem<L>::warp_doubles(H.n_slots),
                         H.n_slots);
    const std::uint32_t n_chunks = (D.n + L - 1u) / L;
    const bool owner = tid < L;
    // The warp's slice of the overflow tape.
    double *gtape = (!GLOBAL && H.n_gslots != 0u)
                        ? gscratch
                              + warp_global * (static_cast<std::size_t>(H.n_gslots) * L)
                        : nullptr;

    // Coefficient store: public tc or the warp's private slice (see coef_view; strides precomputed by the host).
    const coef_view cv{R.coef_base + warp_global * R.coef_warp_stride,
                       static_cast<std::size_t>(R.coef_stride_sv), static_cast<std::size_t>(R.coef_stride_o),
                       R.coef_pub != 0, !PROP && R.skip != nullptr};

    for (std::uint32_t chunk = T::claim(R.counter); chunk < n_chunks; chunk = T::claim(R.counter)) {
        const std::uint32_t lane0 = chunk * L;
        // Owner threads (one per lane) do the scalar bookkeeping of their lane.
        const std::uint32_t lane_raw = lane0 + tid;
        bool valid = owner && lane_raw < D.n;
        const std::uint32_t lane = valid ? lane_raw : D.n - 1u;

        if constexpr (!PROP) {
            double mdt = 0.;
            dfl t0{0., 0.};
            if (owner) {
                const bool skipped = R.skip != nullptr && R.skip[lane] != 0u;
                valid = valid && !skipped;
                mdt = R.max_delta_t != nullptr ? R.max_delta_t[lane] : R.default_max_delta_t;
                t0 = dfl{D.t_hi[lane], D.t_lo[lane]};
                S.time[tid] = t0.hi;
                S.running[tid] = skipped ? 0 : 1;
            }
            T::sync();
            coop_jet<L, N, MODE>(P, H, tab, D, S, lane0, gtape, cv);
            const double h = (!CTA || threadIdx.x < 32u) ? coop_determine_h<L>(P, D, cv, lane0, mdt) : 0.;
            if (owner) {
                S.h[tid] = h;
            }
            T::sync();
            unsigned nf_mask = 0u;
            coop_update_state<L, CTA>(P, D, S, cv, lane0, nf_mask);
            nf_mask = T::template reduce_or<L>(nf_mask);
            if (valid) {
                const dfl nt = dfl_add(t0, dfl{h, 0.});
                D.t_hi[lane] = nt.hi;
                D.t_lo[lane] = nt.lo;
                D.last_h[lane] = h;
                const bool nf = !(isfinite(nt.hi) && isfinite(nt.lo)) || ((nf_mask >> tid) & 1u) != 0u;
                D.step_outcome[lane]
                    = nf ? HY_OUTCOME_ERR_NF_STATE : (h == mdt ? HY_OUTCOME_TIME_LIMIT : HY_OUTCOME_SUCCESS);
            }
        } else {
            lane_prop lp;
            lp.running = false;
            if (owner) {
                lp.init(D, R, lane);
            }
            while (T::any(owner && lp.running)) {
                double cur_max = 0.;
                if (owner) {
                    cur_max = lp.cur_max();
                    S.time[tid] = lp.t.hi;
                    S.running[tid] = lp.running ? 1 : 0;
                }
                T::sync();
                coop_jet<L, N, MODE>(P, H, tab, D, S, lane0, gtape, cv);
                const double h = (!CTA || threadIdx.x < 32u) ? coop_determine_h<L>(P, D, cv, lane0, cur_max) : 0.;
                if (owner) {
                    S.h[tid] = h;
                }
                T::sync();
                unsigned nf_mask = 0u;
                coop_update_state<L, CTA>(P, D, S, cv, lane0, nf_mask);
                nf_mask = T::template reduce_or<L>(nf_mask);
                if (owner && lp.running) {
                    lp.advance(h, cur_max, ((nf_mask >> tid) & 1u) != 0u, R, valid);
                }
            }
            if (valid) {
                lp.store(D, lane);
                lp.report_iters(R);
            }
        }
        T::sync();
    }
}

} // namespace heyoka_b200::dev

#endif
