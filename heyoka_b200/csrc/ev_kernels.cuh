// Event detection in batch mode on the device (include/heyoka_b200.h, section E).
//
// What the reference does on the host for every step of an integrator with events
// (src/taylor_adaptive_batch.cpp:728-1035, src/detail/event_detection.cpp:1733-2173) is split here into small kernels
// on the batch's stream, all data staying in HBM:
//   k_ev_jet     one thread per lane: the jet of the state variables AND of the event equations (order p included:
//                src/taylor_02.cpp:1211-1330 "max_svf_idx"), the step size from both (src/taylor_00.cpp:102-273), the
//                error bound g_eps (:746-773 of the batch integrator), the Taylor coefficients of n_eq + n_ev rows
//                written to the public tc array (:776). The state is NOT propagated (src/taylor_00.cpp:587-590).
//   k_ev_fex     one thread per (event, lane), lanes innermost = coalesced: the fast exclusion check (enclosure of the
//                event polynomial over the step by Horner's scheme in interval arithmetic, :704-816); what survives
//                is appended to a compact candidate list - typically a tiny fraction of the batch.
//   k_ev_detect  one thread per candidate: real-root isolation by the reverse / translate / count-sign-changes
//                bisection of :1980-2087 (the working list is a LIFO stack, kept in a global arena, candidate
//                innermost), then a bracketed root finder per isolating interval (Algorithm 748 of Alefeld, Potra and
//                Shi, the algorithm behind the reference's boost::math::tools::toms748_solve call at :375), direction
//                and cooldown filtering; detected events are appended to a record list, and the earliest terminal
//                event of every lane is found with a 64-bit atomicMin on |t|.
//   k_ev_first   one thread per record: which record is that earliest terminal event (ties: smallest event index).
//   k_ev_apply   one thread per lane: the step is cut at the first terminal event, the state is propagated by
//                evaluating the Taylor polynomials (the reference's m_d_out_f call at :800), time, last_h, outcome,
//                cooldown bookkeeping (:848-865, :903-917).
//   k_ev_filter  one thread per record: which records the host must see (non-terminal events before the first
//                terminal one, :871-876; nothing for lanes that went non-finite, :838-843).
// Callbacks are host code by nature: the host reads the (usually empty) record list back once per step.
#ifndef HEYOKA_B200_CSRC_EV_KERNELS_CUH
#define HEYOKA_B200_CSRC_EV_KERNELS_CUH

#include <cfloat>

#include "kernels.cuh"

namespace heyoka_b200::dev
{

constexpr int EV_MAXP1 = 48;     // maximum Taylor order + 1 of an integrator with events
constexpr int EV_STACK = 48;     // depth of the bisection stack (the reference gives up at 250, :2062)

struct ev_rec {
    std::uint32_t lane, idx;
    std::int32_t terminal, d_sgn;
    double t, abs_der;
    std::uint32_t live, pad;
};

struct ev_args {
    std::uint32_t n_ev, n_te, max_svf;
    double tol;
    const std::uint32_t *ev_defs; // [n_ev]
    const int *dirs;              // [n_ev]
    const double *cooldowns;      // [n_te], < 0: automatic
    const double *bc;             // binomial coefficients [(p + 1)^2]
    double *h;                    // [B] step size: deduced by k_ev_jet, cut by k_ev_apply
    double *mdt;                  // [B] the limit the step was taken with
    double *g_eps;                // [B]
    double *cd;                   // [n_te][2][B]: time spent in cooldown, cooldown
    unsigned char *cd_on;         // [n_te][B]
    std::uint32_t *cand;          // [n_ev * B] candidate = ev * B + lane
    unsigned *counters;           // [0] candidates, [1] records (may exceed rec_cap: overflow), [2] isolation failures
    ev_rec *rec;
    std::uint32_t rec_cap;
    unsigned long long *te_key;   // [B] bits of |t| of the earliest terminal event, ~0 if none
    unsigned long long *te_sel;   // [B] (event index << 32 | record index) of the selected terminal event
    double *arena;                // bisection stacks, [EV_STACK][p + 3][arena_threads]
    std::uint32_t arena_threads;
};

namespace evk
{

__device__ __forceinline__ int sgn(double x)
{
    return (0. < x) - (x < 0.);
}

// Polynomial evaluation and first derivative (src/detail/event_detection.cpp:249-280), no contraction: the host
// compiler of the reference does not fuse these either.
__device__ __forceinline__ double poly_eval(const double *a, double x, std::uint32_t n)
{
    double ret = a[n];
    for (std::uint32_t i = 1; i <= n; ++i) {
        ret = __dadd_rn(a[n - i], __dmul_rn(ret, x));
    }
    return ret;
}
__device__ __forceinline__ double poly_eval_1(const double *a, double x, std::uint32_t n)
{
    double ret = __dmul_rn(a[n], static_cast<double>(n));
    for (std::uint32_t i = 1; i < n; ++i) {
        ret = __dadd_rn(__dmul_rn(a[n - i], static_cast<double>(n - i)), __dmul_rn(ret, x));
    }
    return ret;
}
// a(x) -> a(x * scal) (:171-192).
__device__ __forceinline__ void poly_rescale(double *ret, const double *a, double scal, std::uint32_t n)
{
    double cur_f = 1.;
    for (std::uint32_t i = 0; i <= n; ++i) {
        ret[i] = __dmul_rn(a[i], cur_f);
        cur_f = __dmul_rn(cur_f, scal);
    }
}
// a(x) -> 2^n a(x / 2) (:197-221).
__device__ __forceinline__ void poly_rescale_p2(double *ret, const double *a, std::uint32_t n)
{
    double cur_f = 1.;
    for (std::uint32_t i = 0; i <= n; ++i) {
        ret[n - i] = __dmul_rn(cur_f, a[n - i]);
        cur_f = __dmul_rn(cur_f, 2.);
    }
}
// a(x) -> a(x + 1) with the table of binomial coefficients (:413-507).
__device__ __forceinline__ void poly_translate_1(double *out, const double *a, std::uint32_t n, const double *bc)
{
    for (std::uint32_t i = 0; i <= n; ++i) {
        out[i] = 0.;
    }
    for (std::uint32_t i = 0; i <= n; ++i) {
        const double ai = a[i];
        const double *row = bc + i * (n + 1u);
        for (std::uint32_t k = 0; k <= i; ++k) {
            out[k] = __dadd_rn(out[k], __dmul_rn(ai, __ldg(row + k)));
        }
    }
}
// Sign changes in the coefficient list, zeros skipped (src/detail/llvm_helpers_ed.cpp:58-190).
__device__ __forceinline__ std::uint32_t count_sign_changes(const double *a, std::uint32_t n)
{
    std::uint32_t ret = 0;
    int last = sgn(a[0]);
    for (std::uint32_t i = 1; i <= n; ++i) {
        const int cur = sgn(a[i]);
        ret += (last != 0 && cur + last == 0) ? 1u : 0u;
        last = cur != 0 ? cur : last;
    }
    return ret;
}

// ---- Algorithm 748 (Alefeld, Potra, Shi 1995) in the arrangement of boost::math::tools::toms748_solve ----
struct root_finder {
    const double *poly;
    std::uint32_t order;
    double a, b, fa, fb, d, fd, e, fe;

    __device__ __forceinline__ double f(double x) const
    {
        return poly_eval(poly, x, order);
    }
    __device__ __forceinline__ static int sign(double z)
    {
        return z == 0. ? 0 : (signbit(z) ? -1 : 1);
    }
    __device__ __forceinline__ bool converged() const
    {
        return fabs(a - b) <= 4. * DBL_EPSILON * fmin(fabs(a), fabs(b));
    }
    __device__ __forceinline__ static double safe_div(double num, double denom, double r)
    {
        if (fabs(denom) < 1. && fabs(denom * DBL_MAX) <= fabs(num)) {
            return r;
        }
        return num / denom;
    }
    // New enclosing interval around c; the point dropped from the bracket goes to (d, fd).
    __device__ void bracket(double c)
    {
        const double tol = DBL_EPSILON * 2.;
        if ((b - a) < 2. * tol * a) {
            c = a + (b - a) / 2.;
        } else if (c <= a + fabs(a) * tol) {
            c = a + fabs(a) * tol;
        } else if (c >= b - fabs(b) * tol) {
            c = b - fabs(b) * tol;
        }
        const double fc = f(c);
        if (fc == 0.) {
            a = c;
            fa = 0.;
            d = 0.;
            fd = 0.;
        } else if (sign(fa) * sign(fc) < 0) {
            d = b;
            fd = fb;
            b = c;
            fb = fc;
        } else {
            d = a;
            fd = fa;
            a = c;
            fa = fc;
        }
    }
    __device__ double secant() const
    {
        const double tol = DBL_EPSILON * 5.;
        const double c = a - (fa / (fb - fa)) * (b - a);
        if (c <= a + fabs(a) * tol || c >= b - fabs(b) * tol) {
            return (a + b) / 2.;
        }
        return c;
    }
    __device__ double quadratic(unsigned count) const
    {
        const double B = safe_div(fb - fa, b - a, DBL_MAX);
        double A = safe_div(fd - fb, d - b, DBL_MAX);
        A = safe_div(A - B, d - a, 0.);
        if (A == 0.) {
            return secant();
        }
        double c = (sign(A) * sign(fa) > 0) ? a : b;
        for (unsigned i = 1; i <= count; ++i) {
            c -= safe_div(fa + (B + A * (c - b)) * (c - a), B + A * (2. * c - a - b), 1. + c - a);
        }
        if (c <= a || c >= b) {
            c = secant();
        }
        return c;
    }
    __device__ double cubic() const
    {
        const double q11 = (d - e) * fd / (fe - fd);
        const double q21 = (b - d) * fb / (fd - fb);
        const double q31 = (a - b) * fa / (fb - fa);
        const double d21 = (b - d) * fd / (fd - fb);
        const double d31 = (a - b) * fb / (fb - fa);
        const double q22 = (d21 - q11) * fb / (fe - fb);
        const double q32 = (d31 - q21) * fa / (fd - fa);
        const double d32 = (d31 - q21) * fd / (fd - fa);
        const double q33 = (d32 - q22) * fa / (fe - fa);
        double c = q31 + q32 + q33 + a;
        if (c <= a || c >= b) {
            c = quadratic(3);
        }
        return c;
    }
    // Interpolation step: cubic if the four function values are distinct, else quadratic.
    __device__ double interpolate(unsigned q_count) const
    {
        const double m = DBL_MIN * 32.;
        const bool prof = fabs(fa - fb) < m || fabs(fa - fd) < m || fabs(fa - fe) < m || fabs(fb - fd) < m
                          || fabs(fb - fe) < m || fabs(fd - fe) < m;
        return prof ? quadratic(q_count) : cubic();
    }
    // Returns 0 (ok), -1 (iteration limit) or 1 (no bracket); root = midpoint of the final bracket.
    __device__ int solve(double ax, double bx, double &root)
    {
        // Iteration budget of :321-341: the number of digits of the significand, two of which go to f(ax), f(bx).
        unsigned count = DBL_MANT_DIG - 2;
        const unsigned budget = count;
        a = ax;
        b = bx;
        fa = f(ax);
        fb = f(bx);
        if (!(a < b)) {
            root = 0.;
            return 1;
        }
        bool trivial = false;
        if (converged() || fa == 0. || fb == 0.) {
            trivial = true;
        } else if (sign(fa) * sign(fb) > 0) {
            root = 0.;
            return 1;
        }
        if (!trivial) {
            fe = e = fd = 1e5;
            d = 0.;
            bracket(secant());
            --count;
            if (count != 0u && fa != 0. && !converged()) {
                const double c = quadratic(2);
                e = d;
                fe = fd;
                bracket(c);
                --count;
            }
            while (count != 0u && fa != 0. && !converged()) {
                const double a0 = a, b0 = b;
                double c = interpolate(2);
                e = d;
                fe = fd;
                bracket(c);
                if (--count == 0u || fa == 0. || converged()) {
                    break;
                }
                c = interpolate(3);
                bracket(c);
                if (--count == 0u || fa == 0. || converged()) {
                    break;
                }
                // Double-length secant step.
                const bool a_small = fabs(fa) < fabs(fb);
                const double u = a_small ? a : b, fu = a_small ? fa : fb;
                c = u - 2. * (fu / (fb - fa)) * (b - a);
                if (fabs(c - u) > (b - a) / 2.) {
                    c = a + (b - a) / 2.;
                }
                e = d;
                fe = fd;
                bracket(c);
                if (--count == 0u || fa == 0. || converged()) {
                    break;
                }
                if ((b - a) < 0.5 * (b0 - a0)) {
                    continue;
                }
                // Not converging fast enough: bisect.
                e = d;
                fe = fd;
                bracket(a + (b - a) / 2.);
                --count;
            }
        }
        if (fa == 0.) {
            b = a;
        } else if (fb == 0.) {
            a = b;
        }
        root = a / 2. + b / 2.;
        const unsigned used = trivial ? 0u : budget - count;
        return (used + 2u < static_cast<unsigned>(DBL_MANT_DIG)) ? 0 : -1;
    }
};

} // namespace evk

// ------------------------------------------------------------------------------------------------
// The jet with events: one thread per lane, tape in HBM (the layout of k_hbm).
// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_ev_jet(program P, batch D, run_args R, ev_args E, double *scratch,
                                                std::size_t slab_doubles)
{
    const std::uint32_t lane_in_warp = threadIdx.x & 31u;
    const std::size_t warp_global = (static_cast<std::size_t>(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
    double *slab = scratch + warp_global * slab_doubles + lane_in_warp;
    const std::uint32_t n_chunks = (D.n + 31u) / 32u, p = P.order, pp1 = p + 1u;

    for (std::uint32_t chunk = claim_chunk_warp(R.counter); chunk < n_chunks; chunk = claim_chunk_warp(R.counter)) {
        const std::uint32_t lane_raw = chunk * 32u + lane_in_warp;
        const bool valid = lane_raw < D.n;
        const std::uint32_t lane = valid ? lane_raw : D.n - 1u;
        hbm_tape tape{slab, pp1, D.pars, D.n, lane, D.t_hi[lane], P.args, P.consts};
        const double mdt = R.max_delta_t != nullptr ? R.max_delta_t[lane] : R.default_max_delta_t;

        hbm_jet(P, tape, D.state);
        // Order p of the u variables up to the last one an event equation refers to.
        if (E.max_svf >= P.n_eq) {
            for (std::uint32_t k = 0; k <= E.max_svf - P.n_eq; ++k) {
                const uint4 op = __ldg(P.ops + k);
                const auto self = tape.row(P.n_eq + k);
                self.set(p, diff_op<1>(P, tape, op, self, p));
            }
        }
        // Norms over the state variables, then the event equations (src/taylor_00.cpp:139-197).
        double m0 = 0., mp = 0., mp1 = 0.;
        for (std::uint32_t i = 0; i < P.n_eq + E.n_ev; ++i) {
            const auto r = tape.row(i < P.n_eq ? i : __ldg(E.ev_defs + (i - P.n_eq)));
            const double a0 = fabs(r.at(0).v[0]), ap = fabs(r.at(p).v[0]), ap1 = fabs(r.at(p - 1u).v[0]);
            m0 = i == 0u ? a0 : std_max(m0, a0);
            mp = i == 0u ? ap : std_max(mp, ap);
            mp1 = i == 0u ? ap1 : std_max(mp1, ap1);
        }
        const double h = h_from_norms(P, m0, mp, mp1, mdt);
        // Bound on the remainder of the Taylor series of the event equations (automatic cooldown).
        double g_eps;
        if (isfinite(m0)) {
            const double max_r_size = m0 < 1. ? E.tol : E.tol * m0;
            g_eps = max_r_size < DBL_EPSILON * m0 ? DBL_EPSILON * m0 : max_r_size;
        } else {
            g_eps = CUDART_INF;
        }
        if (valid) {
            E.h[lane] = h;
            E.mdt[lane] = mdt;
            E.g_eps[lane] = g_eps;
            E.te_key[lane] = ~0ull;
            E.te_sel[lane] = ~0ull;
            for (std::uint32_t i = 0; i < P.n_eq + E.n_ev; ++i) {
                const auto r = tape.row(i < P.n_eq ? i : __ldg(E.ev_defs + (i - P.n_eq)));
                for (std::uint32_t o = 0; o < pp1; ++o) {
                    D.tc[(static_cast<std::size_t>(i) * pp1 + o) * D.n + lane] = r.at(o).v[0];
                }
            }
        }
    }
}

// lb_offset of :1917-1934: the part of the step (rescaled to [0, 1)) still in the cooldown of terminal event ev.
__device__ __forceinline__ double ev_lb_offset(const ev_args &E, std::uint32_t n, std::uint32_t ev, std::uint32_t lane,
                                               double h)
{
    if (ev < E.n_te && E.cd_on[static_cast<std::size_t>(ev) * n + lane] != 0u) {
        const double first = E.cd[(static_cast<std::size_t>(ev) * 2u) * n + lane];
        const double second = E.cd[(static_cast<std::size_t>(ev) * 2u + 1u) * n + lane];
        return h >= 0. ? (second - first) / fabs(h) : (second + first) / fabs(h);
    }
    return 0.;
}

// Fast exclusion check, one thread per (event, lane).
__global__ void k_ev_fex(program P, batch D, ev_args E)
{
    const std::size_t idx = static_cast<std::size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (idx >= static_cast<std::size_t>(E.n_ev) * D.n) {
        return;
    }
    const std::uint32_t ev = static_cast<std::uint32_t>(idx / D.n), lane = static_cast<std::uint32_t>(idx % D.n);
    const std::uint32_t p = P.order;
    const double h = E.h[lane];
    const double *c = D.tc + static_cast<std::size_t>(P.n_eq + ev) * (p + 1u) * D.n + lane;
    const bool back = h < 0.;
    const double h_lo = back ? h : 0., h_hi = back ? 0. : h;
    double acc_lo = c[static_cast<std::size_t>(p) * D.n], acc_hi = acc_lo;
    for (std::uint32_t i = 1; i <= p; ++i) {
        const double cf = c[static_cast<std::size_t>(p - i) * D.n];
        const double t1 = __dmul_rn(acc_lo, h_lo), t2 = __dmul_rn(acc_lo, h_hi), t3 = __dmul_rn(acc_hi, h_lo),
                     t4 = __dmul_rn(acc_hi, h_hi);
        const double lo = std_min(std_min(t1, t2), std_min(t3, t4)), hi = std_max(std_max(t1, t2), std_max(t3, t4));
        acc_lo = __dadd_rn(cf, lo);
        acc_hi = __dadd_rn(cf, hi);
    }
    const int s_lo = evk::sgn(acc_lo), s_hi = evk::sgn(acc_hi);
    if (s_lo == s_hi && s_lo != 0) {
        return; // no root in the step
    }
    // The entry checks of the per-element detection (:1803-1825, :1936-1946).
    if (!isfinite(h) || !isfinite(E.g_eps[lane]) || h == 0. || ev_lb_offset(E, D.n, ev, lane, h) >= 1.) {
        return;
    }
    E.cand[atomicAdd(E.counters + 0, 1u)] = static_cast<std::uint32_t>(idx);
}

// Root isolation + root finding, one thread per candidate.
__global__ void __launch_bounds__(64) k_ev_detect(program P, batch D, ev_args E)
{
    const std::uint32_t p = P.order, np1 = p + 1u, T = E.arena_threads;
    const std::uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned n_cand = E.counters[0];
    double ptr[EV_MAXP1], tmp[EV_MAXP1], tmp1[EV_MAXP1], tmp2[EV_MAXP1];
    double isol_lb[EV_MAXP1], isol_ub[EV_MAXP1];
    // Stack entry s of this thread: arena[(s * (np1 + 2) + k) * T + tid], k < np1 coefficients, then lb, ub.
    double *const st = E.arena + tid;
    const std::size_t ent = static_cast<std::size_t>(np1 + 2u) * T;

    for (unsigned ci = tid; ci < n_cand; ci += T) {
        const std::uint32_t cidx = E.cand[ci], ev = cidx / D.n, lane = cidx % D.n;
        const bool terminal = ev < E.n_te;
        const double h = E.h[lane];
        const int dir = __ldg(E.dirs + ev);
        const double lb_offset = ev_lb_offset(E, D.n, ev, lane, h);
        const bool on_cd = terminal && E.cd_on[static_cast<std::size_t>(ev) * D.n + lane] != 0u;
        {
            const double *c = D.tc + static_cast<std::size_t>(P.n_eq + ev) * np1 * D.n + lane;
            for (std::uint32_t o = 0; o <= p; ++o) {
                ptr[o] = c[static_cast<std::size_t>(o) * D.n];
            }
        }
        // add_d_event (:1841-1912).
        const auto add_event = [&](double root) {
            if (!isfinite(root)) {
                return;
            }
            if (fabs(root) >= fabs(h)) {
                root = nextafter(h, 0.);
            }
            const double der = evk::poly_eval_1(ptr, root, p);
            if (!isfinite(der)) {
                return;
            }
            const int d_sgn = evk::sgn(der);
            if (dir != 0 && d_sgn != dir) {
                return;
            }
            const unsigned slot = atomicAdd(E.counters + 1, 1u);
            if (slot < E.rec_cap) {
                E.rec[slot] = ev_rec{lane, terminal ? ev : ev - E.n_te, terminal ? 1 : 0, d_sgn, root, fabs(der), 0u, 0u};
            }
            if (terminal) {
                atomicMin(E.te_key + lane, static_cast<unsigned long long>(__double_as_longlong(fabs(root))));
            }
        };

        evk::poly_rescale(tmp, ptr, h, p);
        std::uint32_t n_wl = 1, n_isol = 0;
        for (std::uint32_t k = 0; k <= p; ++k) {
            st[static_cast<std::size_t>(k) * T] = tmp[k];
        }
        st[static_cast<std::size_t>(np1) * T] = 0.;
        st[static_cast<std::size_t>(np1 + 1u) * T] = 1.;
        bool failed = false;
        do {
            --n_wl;
            const double *top = st + static_cast<std::size_t>(n_wl) * ent;
            bool all_fin = true;
            for (std::uint32_t k = 0; k <= p; ++k) {
                tmp[k] = top[static_cast<std::size_t>(k) * T];
                all_fin = all_fin && (k == 0u || isfinite(tmp[k]));
            }
            const double lb = top[static_cast<std::size_t>(np1) * T], ub = top[static_cast<std::size_t>(np1 + 1u) * T];
            // An event exactly at the lower bound of the interval (:2000-2025).
            if (tmp[0] == 0. && all_fin && !(on_cd && lb < lb_offset)) {
                add_event(__dmul_rn(lb, h));
            }
            // Reverse, translate by 1, count the sign changes (:598-697).
            for (std::uint32_t k = 0; k <= p; ++k) {
                tmp1[k] = tmp[p - k];
            }
            evk::poly_translate_1(tmp2, tmp1, p, E.bc);
            const std::uint32_t n_sc = evk::count_sign_changes(tmp2, p);
            if (n_sc == 1u) {
                isol_lb[n_isol] = lb;
                isol_ub[n_isol] = ub;
                ++n_isol;
            } else if (n_sc > 1u) {
                // Bisect: q -> 2^n q(x / 2) and 2^n q((x + 1) / 2) (:2036-2060).
                evk::poly_rescale_p2(tmp1, tmp, p);
                evk::poly_translate_1(tmp2, tmp1, p, E.bc);
                const double mid = lb / 2. + ub / 2.;
                const bool lower = lb_offset < mid;
                if (n_wl + (lower ? 2u : 1u) > static_cast<std::uint32_t>(EV_STACK)) {
                    failed = true;
                    break;
                }
                if (lower) {
                    double *e0 = st + static_cast<std::size_t>(n_wl) * ent;
                    for (std::uint32_t k = 0; k <= p; ++k) {
                        e0[static_cast<std::size_t>(k) * T] = tmp1[k];
                    }
                    e0[static_cast<std::size_t>(np1) * T] = lb;
                    e0[static_cast<std::size_t>(np1 + 1u) * T] = mid;
                    ++n_wl;
                }
                double *e1 = st + static_cast<std::size_t>(n_wl) * ent;
                for (std::uint32_t k = 0; k <= p; ++k) {
                    e1[static_cast<std::size_t>(k) * T] = tmp2[k];
                }
                e1[static_cast<std::size_t>(np1) * T] = mid;
                e1[static_cast<std::size_t>(np1 + 1u) * T] = ub;
                ++n_wl;
            }
            if (n_isol > p) {
                failed = true;
                break;
            }
        } while (n_wl != 0u);
        if (failed) {
            atomicAdd(E.counters + 2, 1u);
            continue;
        }
        if (n_isol == 0u) {
            continue;
        }
        // Root finding on the polynomial rescaled to [0, 1) (:2100-2160).
        evk::poly_rescale(tmp1, ptr, h, p);
        for (std::uint32_t k = 0; k < n_isol; ++k) {
            double lb = isol_lb[k];
            double ub = isol_ub[k];
            if (on_cd && lb < lb_offset) {
                lb = lb_offset;
                const double f_lb = evk::poly_eval(tmp1, lb, p), f_ub = evk::poly_eval(tmp1, ub, p);
                if (!(f_lb * f_ub < 0.)) {
                    continue;
                }
            }
            // The root is searched in [lb, ub) (:315-320).
            if (isfinite(lb) && isfinite(ub) && ub > lb) {
                ub = nextafter(ub, lb);
            }
            evk::root_finder rf{tmp1, p, 0., 0., 0., 0., 0., 0., 0., 0.};
            double root;
            if (rf.solve(lb, ub, root) == 0) {
                add_event(__dmul_rn(root, h));
            }
        }
    }
}

// Which record is the earliest terminal event of its lane (ties: smallest event index).
__global__ void k_ev_first(batch D, ev_args E)
{
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned n_rec = min(E.counters[1], E.rec_cap);
    if (i >= n_rec) {
        return;
    }
    const ev_rec r = E.rec[i];
    if (r.terminal != 0
        && static_cast<unsigned long long>(__double_as_longlong(fabs(r.t))) == E.te_key[r.lane]) {
        atomicMin(E.te_sel + r.lane, (static_cast<unsigned long long>(r.idx) << 32) | i);
    }
}

// The step itself, one thread per lane.
__global__ void k_ev_apply(program P, batch D, ev_args E)
{
    const std::uint32_t lane = blockIdx.x * blockDim.x + threadIdx.x;
    if (lane >= D.n) {
        return;
    }
    const unsigned long long sel = E.te_sel[lane];
    const bool has_te = sel != ~0ull;
    double h = E.h[lane], te_abs_der = 0.;
    std::uint32_t te_idx = 0;
    if (has_te) {
        const ev_rec r = E.rec[static_cast<std::uint32_t>(sel & 0xffffffffull)];
        h = r.t;
        te_idx = r.idx;
        te_abs_der = r.abs_der;
        E.h[lane] = h;
    }
    // State update by the dense-output function (src/taylor_adaptive_batch.cpp:800).
    const std::size_t nn = D.n;
    bool nf = false;
    for (std::uint32_t i = 0; i < P.n_eq; ++i) {
        const double *c = D.tc + static_cast<std::size_t>(i) * (P.order + 1u) * nn + lane;
        const double res = eval_poly(P, [c, nn](std::uint32_t o) { return c[static_cast<std::size_t>(o) * nn]; }, h);
        D.state[static_cast<std::size_t>(i) * nn + lane] = res;
        nf = nf || !isfinite(res);
    }
    const dfl nt = dfl_add(dfl{D.t_hi[lane], D.t_lo[lane]}, dfl{h, 0.});
    D.t_hi[lane] = nt.hi;
    D.t_lo[lane] = nt.lo;
    D.last_h[lane] = h;
    if (!(isfinite(nt.hi) && isfinite(nt.lo)) || nf) {
        D.step_outcome[lane] = HY_OUTCOME_ERR_NF_STATE;
        return;
    }
    // Cooldowns: time goes by (:848-865) ...
    for (std::uint32_t k = 0; k < E.n_te; ++k) {
        const std::size_t ci = static_cast<std::size_t>(k) * nn + lane;
        if (E.cd_on[ci] != 0u) {
            double *first = E.cd + (static_cast<std::size_t>(k) * 2u) * nn + lane;
            const double tmp = __dadd_rn(*first, h);
            if (fabs(tmp) >= first[nn]) {
                E.cd_on[ci] = 0u;
            } else {
                *first = tmp;
            }
        }
    }
    if (has_te) {
        // ... and the terminal event that fired enters its cooldown (:903-917, :519-550).
        double cdv = __ldg(E.cooldowns + te_idx);
        if (!(cdv >= 0.)) {
            cdv = E.g_eps[lane] / te_abs_der * 10.;
            cdv = isfinite(cdv) ? cdv : 0.;
        }
        E.cd_on[static_cast<std::size_t>(te_idx) * nn + lane] = 1u;
        E.cd[(static_cast<std::size_t>(te_idx) * 2u) * nn + lane] = 0.;
        E.cd[(static_cast<std::size_t>(te_idx) * 2u + 1u) * nn + lane] = cdv;
        // A terminal event without callback (or whose callback returns false) stops the integration: -idx - 1; the
        // host turns it into idx if the callback asks to continue (:958-969).
        D.step_outcome[lane] = -static_cast<long long>(te_idx) - 1;
    } else {
        D.step_outcome[lane] = h == E.mdt[lane] ? HY_OUTCOME_TIME_LIMIT : HY_OUTCOME_SUCCESS;
    }
}

// Which records the host must see.
__global__ void k_ev_filter(batch D, ev_args E)
{
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    const unsigned n_rec = min(E.counters[1], E.rec_cap);
    if (i >= n_rec) {
        return;
    }
    const ev_rec r = E.rec[i];
    bool live = D.step_outcome[r.lane] != HY_OUTCOME_ERR_NF_STATE;
    const unsigned long long sel = E.te_sel[r.lane];
    if (r.terminal != 0) {
        live = live && static_cast<unsigned>(sel & 0xffffffffull) == i;
    } else if (sel != ~0ull) {
        live = live && fabs(r.t) < fabs(D.last_h[r.lane]);
    }
    E.rec[i].live = live ? 1u : 0u;
}

// The absolute times of the records a device propagation calls back for (hy_batch_propagate_until_ev()): new time -
// last_h + t in double-length arithmetic, as the front ends compute the time of a non-terminal event
// (src/taylor_adaptive_batch.cpp:889). recs: the shard's live records, lanes local to the shard.
__global__ void k_ev_times(batch D, const hy_event_rec *recs, std::uint32_t n_rec, double *t_hi, double *t_lo)
{
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_rec) {
        return;
    }
    const hy_event_rec r = recs[i];
    dfl t = dfl_add(dfl{D.t_hi[r.lane], D.t_lo[r.lane]}, dfl{-D.last_h[r.lane], 0.});
    t = dfl_add(t, dfl{r.t, 0.});
    t_hi[i] = t.hi;
    t_lo[i] = t.lo;
}

// The lanes whose terminal-event callback asks to continue: outcome -idx - 1 -> idx (:958-969).
__global__ void k_ev_continue(batch D, const std::uint32_t *lanes, std::uint32_t n)
{
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        D.step_outcome[lanes[i]] = -D.step_outcome[lanes[i]] - 1;
    }
}

// reset_cooldowns() for one lane or all of them (src/taylor_adaptive_batch.cpp:2300-2330).
__global__ void k_ev_reset_cd(ev_args E, std::uint32_t n, std::uint32_t lane_or_all)
{
    const std::size_t i = static_cast<std::size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= static_cast<std::size_t>(E.n_te) * n) {
        return;
    }
    if (lane_or_all == 0xffffffffu || i % n == lane_or_all) {
        E.cd_on[i] = 0u;
    }
}

} // namespace heyoka_b200::dev

#endif
