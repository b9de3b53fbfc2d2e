// TEST INFRASTRUCTURE: host emulation of the N-body kernel's jet (heyoka_b200/csrc/nb_core.hpp) on plain arrays.
//
// nb_core.hpp is the arithmetic of k_nb (nb_kernel.cuh) written once for host and device; the device only supplies
// the storage policy (shared memory + tensor memory). This file supplies a storage policy on std::vector and runs a
// TEAM of `tt` threads owning `lt` lanes exactly like the kernel does: every thread its pair interaction, then the
// rounds of the pre-decoded role table (make_nb_roles()), one "thread" after the other (the threads of a team only
// communicate across synchronisation points). It returns every coefficient, so that the two-orders-at-a-time index
// arithmetic, the output-slot layout and the role records can be checked against the oracle WITHOUT a GPU
// (tests/test_nb_plan.py). It is never linked into the product library. Build: g++ -ffp-contract=off.
#include <cstdint>
#include <cstring>
#include <vector>

#include <heyoka_b200.h>

#include "nb_core.hpp"
#include "nb_plan.hpp"
#include "smem_plan.hpp"

namespace hb = heyoka_b200;
using hb::nb::d2;

namespace
{

struct emul {
    const hb::detail::nb_plan &pl;
    std::uint32_t p, npp, n_eq, lt;
    std::vector<d2> pos, out;   // [slot][lane]
    std::vector<d2> rows;       // [pair][lane][5 rows: d0 d1 d2 r2 q][npp]
    std::vector<double> coef;   // [lane][sv][p + 1]
    std::vector<double> mk;     // [pair][lane][3][2 * npp]: the products' coefficients (diagnostics)
    const double *state;        // [sv][lane]
};

struct pair_mem {
    emul &E;
    std::uint32_t pi, l;
    const hb::detail::nb_pair_desc &d;
    std::uint32_t cur_m = 0;
    d2 *row(int r)
    {
        return E.rows.data() + ((static_cast<std::size_t>(pi) * E.lt + l) * 5u + r) * E.npp;
    }
    d2 pos_a(int k)
    {
        return E.pos[d.pa[k] * E.lt + l];
    }
    d2 pos_b(int k)
    {
        return E.pos[d.pb[k] * E.lt + l];
    }
    void st_d(std::uint32_t m, const d2 (&D)[3])
    {
        for (int k = 0; k < 3; ++k) {
            row(k)[m] = D[k];
        }
    }
    void st_r2(std::uint32_t m, const d2 &r)
    {
        row(3)[m] = r;
    }
    void st_q(std::uint32_t m, const d2 &q)
    {
        row(4)[m] = q;
    }
    void ld_ss(std::uint32_t ai, std::uint32_t li, d2 (&A)[3], d2 (&Lo)[3])
    {
        for (int k = 0; k < 3; ++k) {
            A[k] = row(k)[ai];
            Lo[k] = row(k)[li];
        }
    }
    void ld_a(std::uint32_t ai, d2 (&A)[3])
    {
        for (int k = 0; k < 3; ++k) {
            A[k] = row(k)[ai];
        }
    }
    void ld_main(std::uint32_t qi, std::uint32_t li, d2 &Q, d2 &Rlo, d2 (&Dlo)[3])
    {
        Q = row(4)[qi];
        Rlo = row(3)[li];
        for (int k = 0; k < 3; ++k) {
            Dlo[k] = row(k)[li];
        }
    }
    d2 fac(std::uint32_t n, std::uint32_t j)
    {
        const double *f = E.pl.fac.data() + static_cast<std::size_t>(n) * E.pl.fac_stride + j;
        return d2{f[0], f[1]};
    }
    double fac1(std::uint32_t n, std::uint32_t j)
    {
        return E.pl.fac[static_cast<std::size_t>(n) * E.pl.fac_stride + j];
    }
    void out(int k, const d2 &v)
    {
        E.out[d.om[k] * E.lt + l] = v;
        double *dst = E.mk.data() + ((static_cast<std::size_t>(pi) * E.lt + l) * 3u + k) * 2u * E.npp + 2u * cur_m;
        dst[0] = v.x;
        dst[1] = v.y;
    }
    void out_n(int k, const d2 &v)
    {
        if (d.on[k] != 0xffffu) {
            E.out[d.on[k] * E.lt + l] = v;
        }
    }
};

// One thread of the summation phase: lanes [l0, l0 + NL).
struct role_mem {
    emul &E;
    std::uint32_t l0;
    d2 out_u(std::uint32_t unit, int l)
    {
        return E.out[unit + l];
    }
    void out_st_u(std::uint32_t unit, int l, const d2 &v)
    {
        E.out[unit + l] = v;
    }
    void pos_st_u(std::uint32_t unit, int l, const d2 &v)
    {
        E.pos[unit + l] = v;
    }
    double cst(std::uint32_t i)
    {
        return E.pl.consts[i];
    }
    double rcp(std::uint32_t n)
    {
        return 1. / static_cast<double>(n);
    }
    void coef(std::uint32_t sv, std::uint32_t order, std::uint32_t l, double v)
    {
        if (order <= E.p) {
            E.coef[(static_cast<std::size_t>(l0 + l) * E.n_eq + sv) * (E.p + 1u) + order] = v;
        }
    }
    template <std::size_t NL>
    void coef_pair(std::uint32_t sv, std::uint32_t order, const double (&a)[NL], const double (&b)[NL])
    {
        for (std::uint32_t l = 0; l < NL; ++l) {
            coef(sv, order, l, a[l]);
            coef(sv, order + 1u, l, b[l]);
        }
    }
    template <std::size_t NL>
    void coef_one(std::uint32_t sv, std::uint32_t order, const double (&a)[NL])
    {
        for (std::uint32_t l = 0; l < NL; ++l) {
            coef(sv, order, l, a[l]);
        }
    }
    double state(std::uint32_t sv, int l)
    {
        return E.state[static_cast<std::size_t>(sv) * E.lt + l0 + l];
    }
};

template <int NL>
void run_team(emul &E, std::uint32_t tt)
{
    const auto &pl = E.pl;
    const std::uint32_t lt = E.lt, gs = lt / NL;
    const auto roles = hb::detail::make_nb_roles(pl, tt, lt, NL);
    const auto rec = [&](std::uint32_t rd, std::uint32_t t, std::uint32_t (&w)[8]) {
        static_assert(sizeof(hb::detail::nb_role) == 32u);
        std::memcpy(w, &roles.table[static_cast<std::size_t>(rd) * tt + t], 32u);
    };
    for (std::uint32_t rd = 0; rd < roles.n_rounds; ++rd) {
        for (std::uint32_t t = 0; t < tt; ++t) {
            std::uint32_t w[8];
            rec(rd, t, w);
            role_mem RM{E, (t % gs) * NL};
            hb::nb::role_init<NL>(RM, w);
        }
    }
    const std::uint32_t n_pairs = static_cast<std::uint32_t>(pl.pairs.size());
    for (std::uint32_t m = 0; m < E.npp; ++m) {
        for (std::uint32_t t = 0; t < n_pairs * lt; ++t) {
            const std::uint32_t pi = t / lt, l = t % lt;
            const auto &d = pl.pairs[pi];
            pair_mem PM{E, pi, l, d};
            PM.cur_m = m;
            const hb::nb::pair_consts C{d.c1, {d.c2[0], d.c2[1], d.c2[2]}, pl.alpha, pl.pow_algo, (d.flags & 1u) != 0u};
            hb::nb::pair_block(PM, C, m);
        }
        for (std::uint32_t rd = 0; rd < roles.n_rounds; ++rd) {
            for (std::uint32_t t = 0; t < tt; ++t) {
                std::uint32_t w[8];
                rec(rd, t, w);
                role_mem RM{E, (t % gs) * NL};
                hb::nb::role_block<NL>(RM, w, m, E.p);
            }
        }
    }
}

} // namespace

extern "C" {

// Plan summary: out[0] = ok, n_pairs, n_pos, n_out, n_sums, n_levels. Returns the length of `why`.
int nb_emul_plan(const hy_program *p, std::uint32_t *out, char *why, std::size_t why_len)
{
    const auto pl = hb::detail::make_nb_plan(*p);
    out[0] = pl.ok ? 1u : 0u;
    out[1] = static_cast<std::uint32_t>(pl.pairs.size());
    out[2] = pl.n_pos;
    out[3] = pl.n_out;
    out[4] = static_cast<std::uint32_t>(pl.sums.size());
    out[5] = pl.ok ? static_cast<std::uint32_t>(pl.level_offsets.size()) - 1u : 0u;
    if (why != nullptr && why_len != 0u) {
        std::strncpy(why, pl.why.c_str(), why_len - 1u);
        why[why_len - 1u] = '\0';
    }
    return static_cast<int>(pl.why.size());
}

// Sizes that setup_nb() (batch.cu) lays out shared memory with, for a team of `tt` threads owning `lt` lanes, `nl` per
// thread in the summation phase: out[0] = rounds of the role table, out[1] = its records, out[2] = constants,
// out[3] = row stride of the fac table. Returns 0, -1 if the program does not qualify.
int nb_emul_roles(const hy_program *p, std::uint32_t tt, std::uint32_t lt, std::uint32_t nl, std::uint32_t *out)
{
    const auto pl = hb::detail::make_nb_plan(*p);
    if (!pl.ok) {
        return -1;
    }
    const auto roles = hb::detail::make_nb_roles(pl, tt, lt, nl);
    out[0] = roles.n_rounds;
    out[1] = static_cast<std::uint32_t>(roles.table.size());
    out[2] = static_cast<std::uint32_t>(pl.consts.size());
    out[3] = pl.fac_stride;
    return 0;
}

// The cooperative plan (make_smem_plan(), smem_plan.hpp) that hy_batch builds with the given options: out[0] = n_slots,
// out[1] = n_gslots, out[2] = work items, out[3] = segments, out[4] = 1 if an item is an elementary op (kernel mode 1)
// and 0 if all are superinstructions (mode 0), out[5] = bytes of the table blob, restating make_plan_blob() (batch.cu)
// word by word.
int coop_emul_plan(const hy_program *p, int fuse, int fuse_sv, int spill, std::uint32_t *out)
{
    const auto pl = hb::detail::make_smem_plan(*p, fuse != 0, fuse_sv != 0, spill != 0);
    std::size_t w = 20u; // dev::coop_header
    const auto align = [&](std::size_t a) { w = (w + a - 1u) / a * a; };
    align(4);
    w += 8u * pl.ops.size() + pl.seg_offsets.size() + pl.args.size() + pl.aux.size();
    align(2);
    w += 2u * (p->consts.size() + pl.extra_consts.size());
    align(2);
    w += 2u * (p->order + 3u); // reciprocals 1 / k, k = 0..order + 2
    align(4);
    w += 4u * p->n_eq + pl.svout.size() + pl.sv_phase.size();
    align(4);
    bool elementary = false;
    for (const auto &op : pl.ops) {
        elementary = elementary || op.opcode < hb::detail::HY_FOP_FIRST;
    }
    out[0] = pl.n_slots;
    out[1] = pl.n_gslots;
    out[2] = static_cast<std::uint32_t>(pl.ops.size());
    out[3] = pl.n_segments;
    out[4] = elementary ? 1u : 0u;
    out[5] = static_cast<std::uint32_t>((w + 3u) / 4u * 16u);
    return 0;
}

// Jets of the `lt` lanes of ONE team of `tt` threads. state[n_eq][lt] -> coef[lt][n_eq][order + 1] (state variables),
// and, per pair interaction i and lane l: u_idx[i * 8 + {0..2: d_k, 3: r2, 4: q, 5..7: m_k}] = u variable index,
// u_rows[((i * lt + l) * 8 + r) * n_ord + o] = coefficient of order o (n_ord = 2 * ceil(order / 2)).
// Returns 0, -1 if the program does not qualify, -2 for an unsupported team shape.
int nb_emul_jet(const hy_program *p, std::uint32_t tt, std::uint32_t lt, const double *state, double *coef,
                std::uint32_t *u_idx, double *u_rows)
{
    const auto pl = hb::detail::make_nb_plan(*p);
    if (!pl.ok) {
        return -1;
    }
    const std::uint32_t n_pairs = static_cast<std::uint32_t>(pl.pairs.size());
    if (lt == 0u || n_pairs * lt > tt || (lt > 1u && lt % 2u != 0u)) {
        return -2;
    }
    emul E{pl, p->order, (p->order + 1u) / 2u, p->n_eq, lt, {}, {}, {}, {}, {}, state};
    E.pos.assign(static_cast<std::size_t>(pl.n_pos) * lt, d2{0., 0.});
    E.out.assign(static_cast<std::size_t>(pl.n_out) * lt, d2{0., 0.});
    E.rows.assign(static_cast<std::size_t>(n_pairs) * lt * 5u * E.npp, d2{0., 0.});
    E.coef.assign(static_cast<std::size_t>(lt) * p->n_eq * (p->order + 1u), 0.);
    E.mk.assign(static_cast<std::size_t>(n_pairs) * lt * 3u * 2u * E.npp, 0.);
    if (lt >= 2u) {
        run_team<2>(E, tt);
    } else {
        run_team<1>(E, tt);
    }
    std::memcpy(coef, E.coef.data(), E.coef.size() * sizeof(double));
    const std::uint32_t n_ord = 2u * E.npp;
    for (std::uint32_t pi = 0; pi < n_pairs; ++pi) {
        for (std::uint32_t r = 0; r < 8u; ++r) {
            u_idx[pi * 8u + r] = pl.pair_uvars[pi * 8u + r];
        }
        for (std::uint32_t l = 0; l < lt; ++l) {
            for (std::uint32_t r = 0; r < 8u; ++r) {
                double *dst = u_rows + ((static_cast<std::size_t>(pi) * lt + l) * 8u + r) * n_ord;
                if (r < 5u) {
                    const d2 *src = E.rows.data() + ((static_cast<std::size_t>(pi) * lt + l) * 5u + r) * E.npp;
                    for (std::uint32_t m = 0; m < E.npp; ++m) {
                        dst[2u * m] = src[m].x;
                        dst[2u * m + 1u] = src[m].y;
                    }
                } else {
                    std::memcpy(dst, E.mk.data() + ((static_cast<std::size_t>(pi) * lt + l) * 3u + (r - 5u)) * n_ord,
                                n_ord * sizeof(double));
                }
            }
        }
    }
    return 0;
}

} // extern "C"
