// Superinstructions of the cooperative kernels: several elementary recurrences run back to back by ONE work
// item, found by pattern matching in make_smem_plan(). Every u variable keeps its own tape row and is computed
// by exactly the same arithmetic, in the same order, as by diff_op(): the fusion removes interpreter overhead
// (one dispatch and no synchronisation for a dozen ops), it does not change a single rounding.
#ifndef HEYOKA_B200_CSRC_FUSED_CUH
#define HEYOKA_B200_CSRC_FUSED_CUH

#include <cstdint>

#include "recurrences.cuh"

namespace heyoka_b200::dev
{

constexpr std::uint32_t FOP_FIRST = 0x100u, FOP_NBODY_PAIR = 0x100u, FOP_SUM_T = 0x101u;

// The gravitational pair interaction of model::nbody (src/model/nbody.cpp:97-153) at order n:
//   d_k = x_k^j - x_k^i (src/detail/sub.cpp)            r2 = sum_sq(d_0, d_1, d_2) (src/detail/sum_sq.cpp)
//   q = pow(r2, alpha) (src/math/pow.cpp)               f = c1 q | -q | q (src/math/prod.cpp)
//   m_k = d_k f (src/math/prod.cpp, var * var)          n_k = c2_k m_k (optional)
// aux: [a_k, b_k, d_k] x 3, r2, q, alpha (constant index), order-0 pow algorithm, table j (alpha + 1) (constant index), c1 (constant index),
//      [m_k, operand order, n_k, c2_k (constant index)] x 3   (rows as packed row references; d_k, r2, q, f are
//      history rows and m_k, n_k single-slot rows by construction, so their masks are never decoded).
// A sum whose terms are all single-slot rows: args[off + k] is the slot of term k (pairwise summation of up to 8
// terms, src/math/sum.cpp:250-371).
template <int N, int CNT, typename Tape>
__device__ __forceinline__ vd<N> sum_single_slot_fixed(const Tape &t, std::uint32_t off)
{
    using Row = typename Tape::row_t;
    vd<N> v[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        v[k] = k < CNT ? Row::load(t.base + t.arg(off + k) * Row::stride) : splat<N>(0.);
    }
    return pairwise8(v, static_cast<std::uint32_t>(CNT)); // CNT is a constant: the selects fold away
}
template <int N, typename Tape>
__device__ __forceinline__ vd<N> sum_single_slot(const Tape &t, std::uint32_t off, std::uint32_t cnt)
{
    switch (cnt) {
        case 2:
            return sum_single_slot_fixed<N, 2>(t, off);
        case 3:
            return sum_single_slot_fixed<N, 3>(t, off);
        case 4:
            return sum_single_slot_fixed<N, 4>(t, off);
        case 5:
            return sum_single_slot_fixed<N, 5>(t, off);
        case 6:
            return sum_single_slot_fixed<N, 6>(t, off);
        case 7:
            return sum_single_slot_fixed<N, 7>(t, off);
        default:
            return sum_single_slot_fixed<N, 8>(t, off);
    }
}

// sv_out(offset, value, n): propagates a value that is the derivative of state variables (see coop_jet()).
// GLOBAL_RQ: the r^2 and r^alpha histories live in the overflow tape (global memory / L2) instead of shared memory.
template <int N, bool GLOBAL_RQ, typename Tape, typename SvOut>
__device__ __forceinline__ void fused_nbody_pair(const program &P, const Tape &t, const std::uint32_t *aux,
                                                 std::uint32_t fkind, bool have_n, std::uint32_t n,
                                                 const SvOut &sv_out)
{
    using V = vd<N>;
    using Row = typename Tape::row_t;
    constexpr int S = static_cast<int>(Row::stride);

    // ---- d_k^[n] as SUB_VV: row(a).at(n) - row(b).at(n) ----
    const double *d0[3]; // order-0 address of the three difference rows
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const V v = t.row(aux[3 * k]).at(n) - t.row(aux[3 * k + 1]).at(n);
        const Row D = t.hrow(aux[3 * k + 2]);
        d0[k] = D.hptr(0u);
        Row::store(const_cast<double *>(d0[k]) + n * S, v);
    }

    // ---- r2^[n]: SUM_SQ over the three differences; the three convolutions run interleaved (each keeps
    // its own accumulator and its own summation order) ----
    const Row R2 = GLOBAL_RQ ? t.grow(aux[9]) : t.hrow(aux[9]);
    {
        const bool odd = (n & 1u) != 0u;
        V acc[3] = {splat<N>(0.), splat<N>(0.), splat<N>(0.)};
        if (n > 0u) {
            const std::uint32_t j1 = odd ? (n - 1u) / 2u : (n - 2u) / 2u;
            const double *pa0 = d0[0] + n * S, *pa1 = d0[1] + n * S, *pa2 = d0[2] + n * S;
            const double *pb0 = d0[0], *pb1 = d0[1], *pb2 = d0[2];
#pragma unroll 2
            for (std::uint32_t j = 0; j <= j1; ++j) {
                acc[0] = vfma(Row::load(pa0), Row::load(pb0), acc[0]);
                acc[1] = vfma(Row::load(pa1), Row::load(pb1), acc[1]);
                acc[2] = vfma(Row::load(pa2), Row::load(pb2), acc[2]);
                pa0 -= S;
                pa1 -= S;
                pa2 -= S;
                pb0 += S;
                pb1 += S;
                pb2 += S;
            }
        }
        V v[3];
        if (odd) {
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                v[k] = acc[k];
            }
        } else {
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const V ak2 = Row::load(d0[k] + (n / 2u) * S);
                const V sq = ak2 * ak2;
                v[k] = n > 0u ? (acc[k] + acc[k]) + sq : sq;
            }
        }
        const V r = (v[0] + v[1]) + v[2]; // pairwise_sum of three terms
        R2.set(n, odd ? r + r : r);
    }

    // ---- q^[n] = pow(r2, alpha) ----
    const Row Q = GLOBAL_RQ ? t.grow(aux[10]) : t.hrow(aux[10]);
    V q;
    {
        const V alpha = splat<N>(t.cst(aux[11]));
        if (n == 0u) {
            q = pow_eval(aux[12], R2.at(0u), alpha);
        } else {
            const double nd = static_cast<double>(n);
            // fac_j = n alpha - j (alpha + 1): the products j (alpha + 1) come from a table (aux[13]).
            const double n_alpha = nd * t.cst(aux[11]);
            const double *jap1 = t.consts + aux[13];
            V acc = splat<N>(0.);
            const double *pb = R2.hptr(n), *pa = Q.hptr(0u);
#pragma unroll 4
            for (std::uint32_t j = 0; j < n; ++j) {
                const double fac = n_alpha - jap1[j];
                acc = vfma(splat<N>(fac), Row::load(pb) * Row::load(pa), acc);
                pb -= S;
                pa += S;
            }
            q = acc / (nd * R2.at(0u));
        }
        Q.set(n, q);
    }

    // ---- m_k^[n] = sum_j A^[n-j] B^[j] with (A, B) = (d_k, f) or (f, d_k). f = c1 q (fkind 1), -q (2) or q
    // (0) is not stored: f^[j] is recomputed from q^[j] (one rounding, the same value a stored row would
    // hold), which frees a history row per pair. The f values are shared by the three products. ----
    // (Multiplications by 1 and -1 are exact: one code path for the three kinds.)
    const double c1 = fkind == 1u ? t.cst(aux[14]) : (fkind == 2u ? -1. : 1.);
    const auto f_of = [&](const V &qj) { return c1 * qj; };
    const bool f_first = aux[16] != 0u;
    V acc[3] = {splat<N>(0.), splat<N>(0.), splat<N>(0.)};
    if (!f_first) {
        const double *pf = Q.hptr(0u);
        const double *pd0 = d0[0] + n * S, *pd1 = d0[1] + n * S, *pd2 = d0[2] + n * S;
#pragma unroll 4
        for (std::uint32_t j = 0; j <= n; ++j) {
            const V fj = f_of(Row::load(pf));
            acc[0] = vfma(Row::load(pd0), fj, acc[0]);
            acc[1] = vfma(Row::load(pd1), fj, acc[1]);
            acc[2] = vfma(Row::load(pd2), fj, acc[2]);
            pf += S;
            pd0 -= S;
            pd1 -= S;
            pd2 -= S;
        }
    } else {
        const double *pf = Q.hptr(n);
        const double *pd0 = d0[0], *pd1 = d0[1], *pd2 = d0[2];
#pragma unroll 4
        for (std::uint32_t j = 0; j <= n; ++j) {
            const V fj = f_of(Row::load(pf));
            acc[0] = vfma(fj, Row::load(pd0), acc[0]);
            acc[1] = vfma(fj, Row::load(pd1), acc[1]);
            acc[2] = vfma(fj, Row::load(pd2), acc[2]);
            pf -= S;
            pd0 += S;
            pd1 += S;
            pd2 += S;
        }
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        Row::store(const_cast<double *>(t.hrow(aux[15 + 4 * k]).hptr(0u)), acc[k]);
        if (aux[27 + k] != 0u) {
            sv_out(aux[27 + k], acc[k], n);
        }
        if (have_n) {
            const V nk = t.cst(aux[18 + 4 * k]) * acc[k];
            Row::store(const_cast<double *>(t.hrow(aux[17 + 4 * k]).hptr(0u)), nk);
            if (aux[30 + k] != 0u) {
                sv_out(aux[30 + k], nk, n);
            }
        }
    }
}

} // namespace heyoka_b200::dev

#endif
