// k_nb1: the N-body kernel for systems with ONE pair interaction (the two-body step benchmark,
// benchmark/two_body_step_batch.cpp: model::nbody(2, masses = {1, 0})): one thread per lane, nothing exchanged between
// threads.
//
// k_nb (nb_kernel.cuh) with 32 lanes per warp already gives every thread one (pair interaction, lane), but its
// summation phase is written for sums whose terms come from OTHER threads: positions and pair outputs go through shared
// memory, what a thread adds up is a pre-decoded record per round, the norms of the step-size estimate are shared-memory
// atomics, and two warp synchronisations separate the phases of every order pair: 80 % of the instructions of a
// two-body step. With one pair interaction per lane every "sum" is a single pair output (or a number: the accelerations
// of a body that only massless bodies pull on), so the thread that owns the lane keeps everything in registers:
//   * the six positions of the current order pair, the outputs m_k / n_k of the pair interaction (nb_core.hpp's
//     pair_block() with a register policy), v^[n+1] = a^[n] / (n + 1), x^[n+2] = v^[n+1] / (n + 2) in straight-line code;
//   * its history rows d_0, d_1 in shared memory and r^2, d_2, r^alpha in tensor memory, exactly as in k_nb;
//   * the state variables' coefficients (velocities: orders 1..p, positions: 2..p; the lower ones are the state) go to
//     a private per-warp store [order][slot][32 lanes] with compile-time strides (one store instruction per
//     coefficient, 256-byte rows, 1 KB per lane of the two-body benchmark: the stores of all resident warps, 54 MB, stay in
//     L2), read back for the step-size norms, the state update and the public tc array when the caller asks for it.
//     A body that nothing pulls on (right-hand side 0) stores nothing: its rows are (v_0, 0, ...), (x_0, v_0, 0, ...).
//     (HY_NB1_STORE_X=0: only the velocities are stored and the positions' coefficients x^[o] = v^[o-1] / o are
//     recomputed - correctly rounded either way, hence identical - where they are needed again.)
// No exchange between threads; a __syncwarp() per order pair only keeps the warp converged for the tensor-memory
// accesses. Same arithmetic, same order of operations as k_nb / k_coop: bit-identical results (tests/test_gpu_parity.py
// runs both on the same inputs).
// Replaces, for these programs: the JIT'd step function (src/taylor_00.cpp:712-865) and the propagate loop
// (src/taylor_adaptive_batch.cpp:1136-1534).
#ifndef HEYOKA_B200_CSRC_NB1_KERNEL_CUH
#define HEYOKA_B200_CSRC_NB1_KERNEL_CUH

#include <cstdint>

#include <cuda_runtime.h>

#include "nb_kernel.cuh"

namespace heyoka_b200::dev
{

namespace nbk
{

// pair_block()'s storage policy for a thread that owns its lane: positions in, pair outputs out are registers; the
// private history rows are those of pair_mem<32, OFFCHIP>.
template <bool OFFCHIP>
struct pair_mem1 : pair_mem<32, OFFCHIP> {
    d2 xa[3], xb[3];   // (x^[n], x^[n+1]) of the two bodies
    d2 om_[3], on_[3]; // (m_k^[n], m_k^[n+1]), (n_k^[n], n_k^[n+1])

    __device__ __forceinline__ d2 pos_a(int k) const
    {
        return xa[k];
    }
    __device__ __forceinline__ d2 pos_b(int k) const
    {
        return xb[k];
    }
    __device__ __forceinline__ void out(int k, const d2 &v)
    {
        om_[k] = v;
    }
    __device__ __forceinline__ void out_n(int k, const d2 &v)
    {
        on_[k] = v;
    }
};

} // namespace nbk

// NaN-skipping running maximum of |v| on the bit patterns (non-negative doubles order like unsigned integers).
__device__ __forceinline__ void nb1_track(unsigned long long &m, double v)
{
    if (v == v) {
        const unsigned long long b = static_cast<unsigned long long>(__double_as_longlong(v)) & 0x7fffffffffffffffull;
        m = b > m ? b : m;
    }
}
// x / n for the recomputed position coefficients: the correctly rounded quotient whichever path produced it in the jet.
__device__ __forceinline__ double nb1_div(double x, std::uint32_t n, double nd, double rcp)
{
    if (n <= 64u && nb::div_si_in_range(x)) {
        return nb::div_si_fast(x, nd, rcp);
    }
    return x == 0. ? x : nb::div_cold(x, nd);
}

template <bool OFFCHIP, bool PROP, int MAXT>
__global__ void __launch_bounds__(MAXT, 1) k_nb1(program P, nb_dev_plan NP, batch D, run_args R)
{
    using nb::d2;
    extern __shared__ __align__(16) double smem_raw[];
#if !defined(HY_NB1_STORE_X)
#define HY_NB1_STORE_X 1
#endif
    // SX: the positions' coefficients (orders 2..p) are stored next to the velocities' instead of being recomputed where
    // they are needed again (1 KB per lane instead of 0.5 KB, 60 quotients per lane-step less).
    constexpr bool SX = HY_NB1_STORE_X != 0;
    constexpr std::uint32_t SO = (SX ? 12u : 6u) * 32u; // doubles per order of the private store: [order - 1][slot][lane]
    constexpr std::uint32_t XO = 6u * 32u;              // X(o, s) at cb[(o - 1) * SO + XO + s * 32] (SX)

    // ---- CTA-shared tables: fac | rcp ----
    const std::uint32_t p = P.order;
    double *fac_s = smem_raw;
    const std::uint32_t n_fac = (p + 1u) * NP.fac_stride;
    double *rcp_s = fac_s + n_fac;
    const std::uint32_t n_rcp = (p + 5u) & ~1u;
    for (std::uint32_t i = threadIdx.x; i < n_fac; i += blockDim.x) {
        fac_s[i] = __ldg(NP.fac + i);
    }
    for (std::uint32_t i = threadIdx.x; i < n_rcp; i += blockDim.x) {
        rcp_s[i] = i == 0u ? 0. : 1. / static_cast<double>(i);
    }
    static_assert(!OFFCHIP, "the one-thread-per-lane kernel keeps its private rows in shared memory");
    __syncthreads();

    const std::uint32_t tid = threadIdx.x & 31u, warp = threadIdx.x >> 5;
    double *region = smem_raw + NP.shared_doubles + static_cast<std::size_t>(warp) * NP.team_doubles;
    using PM_t = nbk::pair_mem1<OFFCHIP>;
    PM_t PM;
    nb::pair_consts PC;
    {
        const uint4 *dp = reinterpret_cast<const uint4 *>(NP.pairs);
        const uint4 w1 = __ldg(dp + 1), w2 = __ldg(dp + 2), w3 = __ldg(dp + 3);
        PC.c1 = __hiloint2double(static_cast<int>(w2.y), static_cast<int>(w2.x));
        PC.c2[0] = __hiloint2double(static_cast<int>(w2.w), static_cast<int>(w2.z));
        PC.c2[1] = __hiloint2double(static_cast<int>(w3.y), static_cast<int>(w3.x));
        PC.c2[2] = __hiloint2double(static_cast<int>(w3.w), static_cast<int>(w3.z));
        PC.alpha = NP.alpha;
        PC.pow_algo = NP.pow_algo;
        PC.have_n = (w1.z & 1u) != 0u;
        PM.drow = nbk::saddr(region) + tid * 16u;
        PM.fac_ = nbk::saddr(fac_s);
        PM.fac_stride_b = NP.fac_stride * 8u;
        PM.flags = 0u;
        PM.grow = nullptr;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            PM.on_[k] = d2{0., 0.};
        }
    }
    std::uint32_t rcp_a = nbk::saddr(rcp_s);
    nbk::keep(rcp_a);
    nbk::keep(PM.fac_);
    nbk::keep(PM.drow);
    lane_prop *const park
        = reinterpret_cast<lane_prop *>(region + static_cast<std::size_t>(NP.npp) * PM_t::OPB / 8u) + tid;
    static_assert(sizeof(lane_prop) <= 128u && alignof(lane_prop) <= 8u);

    const std::size_t team_global = (static_cast<std::size_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    // The private store of this thread's lane: V(o, s) = v_s^[o] (o = 1..p) at cb[(o - 1) * SO + s * 32].
    double *const cb = R.coef_base + team_global * R.coef_warp_stride + tid;
    const bool pub = R.coef_pub != 0;
    const std::uint32_t n_chunks = (D.n + 31u) / 32u;
    const std::uint32_t n_blocks = NP.npp;
    const nb1_tab &TB = NP.l1;
    const std::size_t nb = D.n;

    // The jet of this thread's lane (glane: clamped global lane). Returns the NaN-skipping maximum of the order-0
    // coefficients (bit pattern).
    const auto jet = [&](std::uint32_t glane) {
        unsigned long long m0 = 0ull;
#pragma unroll
        for (int s = 0; s < 6; ++s) {
            const double x0 = D.state[static_cast<std::size_t>(TB.x_sv[s]) * nb + glane];
            const double v0 = D.state[static_cast<std::size_t>(TB.v_sv[s]) * nb + glane];
            nb1_track(m0, x0);
            nb1_track(m0, v0);
            (s < 3 ? PM.xa[s % 3] : PM.xb[s % 3]) = d2{x0, v0};
        }
        double *vp = cb; // V(n + 1, 0)
        for (std::uint32_t m = 0; m < n_blocks; ++m) {
            __syncwarp();
            nb::pair_block(PM, PC, m);
            const std::uint32_t n = 2u * m;
            const double n1 = static_cast<double>(n + 1u), n2 = static_cast<double>(n + 2u),
                         n3 = static_cast<double>(n + 3u);
            const double r1 = nbk::lds1(rcp_a + (n + 1u) * 8u), r2 = nbk::lds1(rcp_a + (n + 2u) * 8u),
                         r3 = nbk::lds1(rcp_a + (n + 3u) * 8u);
            const bool two = n + 2u <= p;
#pragma unroll
            for (int side = 0; side < 2; ++side) {
                const std::uint32_t kind = TB.kind[side];
                if (kind == 2u) {
                    // Right-hand side 0: v = (v_0, 0, ...), x = (x_0, v_0, 0, ...).
#pragma unroll
                    for (int k = 0; k < 3; ++k) {
                        (side == 0 ? PM.xa[k] : PM.xb[k]) = d2{0., 0.};
                    }
                    continue;
                }
#pragma unroll
                for (int k = 0; k < 3; ++k) {
                    const d2 a = kind == 1u ? PM.on_[k] : PM.om_[k];
                    // (Every quotient takes its own range check: the coefficients of a circular orbit are zero at
                    // every other order, and a zero next to a regular value must not send both to the true division.)
                    const double va = nb1_div(a.x, n + 1u, n1, r1); // v^[n+1]
                    const double vb = nb1_div(a.y, n + 2u, n2, r2); // v^[n+2]
                    const double xa = nb1_div(va, n + 2u, n2, r2);  // x^[n+2]
                    const double xb = nb1_div(vb, n + 3u, n3, r3);  // x^[n+3]
                    vp[(side * 3 + k) * 32] = va;
                    if (two) {
                        vp[SO + (side * 3 + k) * 32] = vb;
                        if constexpr (SX) {
                            vp[SO + XO + (side * 3 + k) * 32] = xa;
                            if (n + 3u <= p) {
                                vp[2u * SO + XO + (side * 3 + k) * 32] = xb;
                            }
                        }
                    }
                    (side == 0 ? PM.xa[k] : PM.xb[k]) = d2{xa, xb};
                }
            }
            vp += 2u * SO;
        }
        return m0;
    };

    // Step size (nb_step_size()'s semantics: NaN-skipping maxima over the state variables of the orders 0, p, p - 1; a NaN
    // in the FIRST state variable makes the norm a NaN).
    const auto step_size = [&](std::uint32_t glane, unsigned long long m0, double max_delta_t) {
        unsigned long long mp = 0ull, mp1 = 0ull;
        double fp = 0., fp1 = 0.;
        const double pd = static_cast<double>(p), pd1 = static_cast<double>(p - 1u);
        const double rp = nbk::lds1(rcp_a + p * 8u), rp1 = nbk::lds1(rcp_a + (p - 1u) * 8u);
        const double *top = cb + static_cast<std::size_t>(p - 1u) * SO; // V(p, 0)
#pragma unroll 1
        for (std::uint32_t side = 0; side < 2u; ++side) {
            if (TB.kind[side] == 2u) {
                continue;
            }
#pragma unroll
            for (std::uint32_t k = 0; k < 3u; ++k) {
                const std::uint32_t s = side * 3u + k;
                const double *c = top + s * 32u;
                const double vp_ = c[0], vp1_ = *(c - SO);
                double xp_, xp1_;
                if constexpr (SX) {
                    xp_ = c[XO];
                    xp1_ = *(c + XO - SO);
                } else {
                    const double vp2_ = *(c - 2u * SO);
                    xp_ = nb1_div(vp1_, p, pd, rp);
                    xp1_ = nb1_div(vp2_, p - 1u, pd1, rp1);
                }
                nb1_track(mp, vp_);
                nb1_track(mp, xp_);
                nb1_track(mp1, vp1_);
                nb1_track(mp1, xp1_);
                if (s == TB.sv0_slot) {
                    fp = fabs(TB.sv0_is_x != 0u ? xp_ : vp_);
                    fp1 = fabs(TB.sv0_is_x != 0u ? xp1_ : vp1_);
                }
            }
        }
        const double f0 = fabs(D.state[glane]);
        return h_from_norms(P, isnan(f0) ? f0 : __longlong_as_double(static_cast<long long>(m0)),
                            isnan(fp) ? fp : __longlong_as_double(static_cast<long long>(mp)),
                            isnan(fp1) ? fp1 : __longlong_as_double(static_cast<long long>(mp1)), max_delta_t);
    };

    // The public Taylor coefficients of the lane (write_tc): tc[(sv (p + 1) + o) batch + lane].
    const auto publish = [&](std::uint32_t glane) {
        const std::size_t so = nb, ssv = static_cast<std::size_t>(p + 1u) * nb;
#pragma unroll 1
        for (std::uint32_t s = 0; s < 6u; ++s) {
            const bool stored = TB.kind[s / 3u] != 2u;
            const std::uint32_t vs = TB.v_sv[s], xs = TB.x_sv[s];
            double prev = D.state[static_cast<std::size_t>(vs) * nb + glane];
            double *tv = D.tc + vs * ssv + glane, *tx = D.tc + xs * ssv + glane;
            tv[0] = prev;
            tx[0] = D.state[static_cast<std::size_t>(xs) * nb + glane];
            const double *c = cb + s * 32u;
            for (std::uint32_t o = 1; o <= p; ++o) {
                const double cur = stored ? c[static_cast<std::size_t>(o - 1u) * SO] : 0.;
                tv[o * so] = cur;
                if (SX && o >= 2u) {
                    tx[o * so] = stored ? c[static_cast<std::size_t>(o - 1u) * SO + XO] : 0.;
                } else {
                    tx[o * so] = nb1_div(prev, o, static_cast<double>(o), nbk::lds1(rcp_a + o * 8u));
                }
                prev = cur;
            }
        }
    };

    // State update of the lane (Horner / compensated summation of recurrences.cuh::eval_poly(), the three coordinates
    // of a body side by side, velocity and position chains fed by the same loads); returns true if a non-finite
    // value was produced.
    const auto update = [&](std::uint32_t glane, bool write, double h) {
        bool nf = false;
#pragma unroll 1
        for (std::uint32_t side = 0; side < 2u; ++side) {
            const bool stored = TB.kind[side] != 2u;
            double v0[3], x0[3], rv[3], rx[3];
            const double *c[3];
#pragma unroll
            for (std::uint32_t k = 0; k < 3u; ++k) {
                const std::uint32_t s = side * 3u + k;
                v0[k] = D.state[static_cast<std::size_t>(TB.v_sv[s]) * nb + glane];
                x0[k] = D.state[static_cast<std::size_t>(TB.x_sv[s]) * nb + glane];
                c[k] = cb + s * 32u;
            }
            if (!P.high_accuracy) {
                // v: ((V(p) h + V(p-1)) h + ...) h + v_0;  x: ((x^[p] h + x^[p-1]) h + ...) h + x_0, x^[o] = V(o-1) / o.
#pragma unroll
                for (std::uint32_t k = 0; k < 3u; ++k) {
                    rv[k] = stored ? c[k][static_cast<std::size_t>(p - 1u) * SO] : 0.;
                    rx[k] = 0.;
                }
                // (The loads of the next order are issued before the arithmetic of the current one.)
                double wn[3], xn[3];
#pragma unroll
                for (std::uint32_t k = 0; k < 3u; ++k) {
                    wn[k] = stored ? c[k][static_cast<std::size_t>(p - 2u) * SO] : 0.; // V(p - 1)
                    xn[k] = (SX && stored) ? c[k][static_cast<std::size_t>(p - 1u) * SO + XO] : 0.; // X(p)
                }
                for (std::uint32_t o = p; o >= 2u; --o) {
                    const double od = static_cast<double>(o), ro = nbk::lds1(rcp_a + o * 8u);
                    double w[3], xw[3];
#pragma unroll
                    for (std::uint32_t k = 0; k < 3u; ++k) {
                        w[k] = wn[k];
                        xw[k] = xn[k];
                        wn[k] = (stored && o > 2u) ? c[k][static_cast<std::size_t>(o - 3u) * SO] : 0.; // V(o - 2)
                        xn[k] = (SX && stored && o > 2u) ? c[k][static_cast<std::size_t>(o - 2u) * SO + XO] : 0.; // X(o - 1)
                    }
#pragma unroll
                    for (std::uint32_t k = 0; k < 3u; ++k) {
                        // x^[o]: stored, or V(o - 1) / o (0 / o = 0 without a division)
                        const double xo = SX ? xw[k] : (stored ? nb1_div(w[k], o, od, ro) : 0.);
                        rv[k] = ::fma(rv[k], h, w[k]);
                        rx[k] = o == p ? xo : ::fma(rx[k], h, xo);
                    }
                }
#pragma unroll
                for (std::uint32_t k = 0; k < 3u; ++k) {
                    rv[k] = ::fma(rv[k], h, v0[k]);
                    rx[k] = ::fma(::fma(rx[k], h, v0[k]), h, x0[k]);
                }
            } else {
                double cpv[3], cpx[3], prev[3], cur_h = h;
#pragma unroll
                for (std::uint32_t k = 0; k < 3u; ++k) {
                    rv[k] = v0[k];
                    rx[k] = x0[k];
                    cpv[k] = cpx[k] = 0.;
                    prev[k] = v0[k];
                }
                for (std::uint32_t o = 1; o <= p; ++o) {
                    const double od = static_cast<double>(o), ro = nbk::lds1(rcp_a + o * 8u);
#pragma unroll
                    for (std::uint32_t k = 0; k < 3u; ++k) {
                        const double cv_ = stored ? c[k][static_cast<std::size_t>(o - 1u) * SO] : 0.; // V(o)
                        double cx_; // x^[o]
                        if (SX && o >= 2u) {
                            cx_ = stored ? c[k][static_cast<std::size_t>(o - 1u) * SO + XO] : 0.;
                        } else {
                            cx_ = (stored || o == 1u) ? nb1_div(prev[k], o, od, ro) : 0.;
                        }
                        prev[k] = cv_;
                        {
                            const double tmp = __dmul_rn(cv_, cur_h);
                            const double y = __dsub_rn(tmp, cpv[k]);
                            const double tt = __dadd_rn(rv[k], y);
                            cpv[k] = __dsub_rn(__dsub_rn(tt, rv[k]), y);
                            rv[k] = tt;
                        }
                        {
                            const double tmp = __dmul_rn(cx_, cur_h);
                            const double y = __dsub_rn(tmp, cpx[k]);
                            const double tt = __dadd_rn(rx[k], y);
                            cpx[k] = __dsub_rn(__dsub_rn(tt, rx[k]), y);
                            rx[k] = tt;
                        }
                    }
                    cur_h = __dmul_rn(cur_h, h);
                }
            }
            if (write) {
#pragma unroll
                for (std::uint32_t k = 0; k < 3u; ++k) {
                    const std::uint32_t s = side * 3u + k;
                    D.state[static_cast<std::size_t>(TB.v_sv[s]) * nb + glane] = rv[k];
                    D.state[static_cast<std::size_t>(TB.x_sv[s]) * nb + glane] = rx[k];
                    nf = nf || !isfinite(rv[k]) || !isfinite(rx[k]);
                }
            }
        }
        return nf;
    };

    for (std::uint32_t chunk = claim_chunk_warp(R.counter); chunk < n_chunks; chunk = claim_chunk_warp(R.counter)) {
        const std::uint32_t lane_raw = chunk * 32u + tid;
        bool valid = lane_raw < D.n;
        const std::uint32_t lane = valid ? lane_raw : D.n - 1u;

        if constexpr (!PROP) {
            // (A step with a skip mask leaves the lanes that are not running untouched, tc included.)
            const bool skipped = R.skip != nullptr && R.skip[lane] != 0u;
            valid = valid && !skipped;
            const unsigned long long m0 = jet(lane);
            const double mdt = R.max_delta_t != nullptr ? R.max_delta_t[lane] : R.default_max_delta_t;
            const double h = step_size(lane, m0, mdt);
            if (pub && valid) {
                publish(lane);
            }
            const bool state_nf = update(lane, valid, h);
            if (valid) {
                const dfl nt = dfl_add(dfl{D.t_hi[lane], D.t_lo[lane]}, dfl{h, 0.});
                D.t_hi[lane] = nt.hi;
                D.t_lo[lane] = nt.lo;
                D.last_h[lane] = h;
                const bool nf = !(isfinite(nt.hi) && isfinite(nt.lo)) || state_nf;
                D.step_outcome[lane]
                    = nf ? HY_OUTCOME_ERR_NF_STATE : (h == mdt ? HY_OUTCOME_TIME_LIMIT : HY_OUTCOME_SUCCESS);
            }
        } else {
            bool running;
            {
                lane_prop lp;
                lp.init(D, R, lane);
                *park = lp;
                running = lp.running;
            }
            while (__any_sync(0xffffffffu, running)) {
                const unsigned long long m0 = jet(lane);
                const double cur_max = park->cur_max();
                const double h = step_size(lane, m0, cur_max);
                if (pub && valid) {
                    publish(lane);
                }
                const bool state_nf = update(lane, valid && running, h);
                if (running) {
                    lane_prop lp = *park;
                    lp.advance(h, cur_max, state_nf, R, valid);
                    *park = lp;
                    running = lp.running;
                }
            }
            if (valid) {
                park->store(D, lane);
                park->report_iters(R);
            }
        }
        __syncwarp();
    }
}

} // namespace heyoka_b200::dev

#endif
