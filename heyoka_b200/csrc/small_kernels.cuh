// Small non-template kernels (included by batch.cu only).
#ifndef HEYOKA_B200_CSRC_SMALL_KERNELS_CUH
#define HEYOKA_B200_CSRC_SMALL_KERNELS_CUH

#include "kernels.cuh"
#include "nb_core.hpp"

namespace heyoka_b200::dev
{

__global__ void k_fill_outcome(long long *out, std::uint32_t n, long long value)
{
    const std::uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        out[i] = value;
    }
}

// After propagate_until(): the lanes that were done before the last iteration (loop_len) of the reference's lock-step
// loop took zero-length steps there (src/taylor_adaptive_batch.cpp:1372-1397): last_h = 0. Also prepares the masked
// zero-length step that re-expands their Taylor coefficients (skip = 1 for the lanes to leave alone, limits = 0).
__global__ void k_prop_early(const unsigned long long *iters, unsigned long long loop_len, std::uint32_t n,
                             double *last_h, unsigned char *skip, double *zero_limits, unsigned *any_early)
{
    const std::uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        const bool early = iters[i] < loop_len;
        if (early) {
            last_h[i] = 0.;
            atomicOr(any_early, 1u);
        }
        skip[i] = early ? 0u : 1u;
        zero_limits[i] = 0.;
    }
}

// Dense output (src/taylor_01.cpp:1015-1185): Horner, or compensated summation in high-accuracy mode.
__global__ void k_d_output(program P, std::uint32_t n, const double *tc, const double *tau, double *out)
{
    const std::uint32_t lane = blockIdx.x * blockDim.x + threadIdx.x;
    if (lane >= n) {
        return;
    }
    const double h = tau[lane];
    const std::size_t nn = n;
    for (std::uint32_t i = 0; i < P.n_eq; ++i) {
        const double *c = tc + static_cast<std::size_t>(i) * (P.order + 1u) * n + lane;
        out[static_cast<std::size_t>(i) * n + lane]
            = eval_poly(P, [c, nn](std::uint32_t o) { return c[static_cast<std::size_t>(o) * nn]; }, h);
    }
}

// ---- The reference's lock-step loop (src/taylor_adaptive_batch.cpp:1372-1527, and :1696-2053 for propagate_grid()):
// per-lane bookkeeping on the device between the steps. One thread per lane. ----
struct lockstep_state {
    const double *tf_hi, *tf_lo; // target times (tf_lo may be nullptr; a grid's target is its last row)
    const double *max_delta_t;   // positive per-lane limits or nullptr (+inf)
    double *rem_hi, *rem_lo;     // remaining time to the target (double-length)
    unsigned char *t_dir;        // 1: forward
    double *dt_limit;            // signed limit of the next step
    unsigned *flags; // [0] number of lanes at their target in this iteration, [1] non-finite state, [2] overflow of rem
};

// Before the first step: remaining times, directions, counters, limit of the first step (for a grid, :1728-1760).
__global__ void k_lockstep_init(batch D, lockstep_state L, double *min_h, double *max_h, unsigned long long *ts_count)
{
    const std::uint32_t lane = blockIdx.x * blockDim.x + threadIdx.x;
    if (lane >= D.n) {
        return;
    }
    const dfl rem = dfl_sub(dfl{L.tf_hi[lane], L.tf_lo != nullptr ? L.tf_lo[lane] : 0.}, dfl{D.t_hi[lane], D.t_lo[lane]});
    if (!(isfinite(rem.hi) && isfinite(rem.lo))) {
        atomicOr(L.flags + 2, 1u);
    }
    L.rem_hi[lane] = rem.hi;
    L.rem_lo[lane] = rem.lo;
    const bool dir = dfl_ge0(rem);
    L.t_dir[lane] = dir ? 1 : 0;
    min_h[lane] = CUDART_INF;
    max_h[lane] = 0.;
    ts_count[lane] = 0ull;
    L.dt_limit[lane] = step_limit(dir, rem, L.max_delta_t != nullptr ? L.max_delta_t[lane] : CUDART_INF);
}

// After a lock-step step (:1402-1460, :1915-1971): counters, min/max |h|, remaining time, outcome, limit of the next
// step.
__global__ void k_lockstep_book(batch D, lockstep_state L, long long *outcome, double *min_h, double *max_h,
                                unsigned long long *ts_count)
{
    const std::uint32_t lane = blockIdx.x * blockDim.x + threadIdx.x;
    if (lane >= D.n) {
        return;
    }
    const long long oc = D.step_outcome[lane];
    const double h = D.last_h[lane];
    if (oc == HY_OUTCOME_ERR_NF_STATE) {
        atomicOr(L.flags + 1, 1u);
    } else {
        ts_count[lane] += (h != 0.) ? 1ull : 0ull;
        if (oc == HY_OUTCOME_SUCCESS) {
            const double ah = fabs(h);
            min_h[lane] = fmin(min_h[lane], ah);
            max_h[lane] = fmax(max_h[lane], ah);
        }
        dfl rem{0., 0.};
        if (h == L.rem_hi[lane]) {
            atomicAdd(L.flags, 1u);
        } else {
            rem = dfl_sub(dfl{L.tf_hi[lane], L.tf_lo != nullptr ? L.tf_lo[lane] : 0.}, dfl{D.t_hi[lane], D.t_lo[lane]});
        }
        L.rem_hi[lane] = rem.hi;
        L.rem_lo[lane] = rem.lo;
        L.dt_limit[lane]
            = step_limit(L.t_dir[lane] != 0, rem, L.max_delta_t != nullptr ? L.max_delta_t[lane] : CUDART_INF);
    }
    outcome[lane] = oc;
}

// ---- propagate_grid() (src/taylor_adaptive_batch.cpp:1545-2055): dense-output sampling between the lock-step steps,
// whose target is the last grid point. ----
struct grid_state {
    const double *grid; // [n_pts][batch]
    std::uint32_t n_pts;
    double *out;            // [n_pts][n_eq][batch], NaN-filled
    std::uint32_t *cur_idx; // first grid point not yet written, per lane
    unsigned *left;         // set when some lane has grid points left
};

// The grid points covered by the last step of a lane (:1811-1886): [first, last) from the lane's cursor, and the start
// of the step (the Taylor coefficients are centred there).
struct grid_window {
    std::uint32_t first, last;
    dfl start;
};
__device__ __forceinline__ grid_window grid_covered(const batch &D, const grid_state &G, const lockstep_state &L,
                                                    std::uint32_t lane)
{
    const std::size_t n = D.n;
    const dfl t{D.t_hi[lane], D.t_lo[lane]};
    const dfl cmp = dfl_sub(t, dfl{D.last_h[lane], 0.}); // start of the last step
    const dfl t0 = dfl_lt(cmp, t) ? cmp : t, t1 = dfl_lt(t, cmp) ? cmp : t;
    const bool rem0 = L.rem_hi[lane] == 0. && L.rem_lo[lane] == 0.;
    const std::uint32_t first = G.cur_idx[lane];
    std::uint32_t idx = first;
    while (idx < G.n_pts) {
        const dfl g{G.grid[static_cast<std::size_t>(idx) * n + lane], 0.};
        if (!((!dfl_lt(g, t0) && !dfl_lt(t1, g)) || rem0)) {
            break;
        }
        ++idx;
    }
    return grid_window{first, idx, cmp};
}

// Dense output at every grid point covered by the last step: one thread per (lane, state variable) - blockIdx.y is the
// state variable - so that the [n_pts][n_eq][batch] output is written by n_eq times as many threads as there are lanes
// (a lane covers tens of grid points per step when the grid is dense: 36 x 21 coefficients x points per lane are too
// much serial work for one thread). Reads the cursors only: k_grid_advance() moves them afterwards. Does nothing if a
// non-finite state was detected in this iteration.
__global__ void k_grid_sample(program P, batch D, grid_state G, lockstep_state L)
{
    const std::uint32_t lane = blockIdx.x * blockDim.x + threadIdx.x, i = blockIdx.y;
    if (lane >= D.n || L.flags[1] != 0u) {
        return;
    }
    const std::size_t n = D.n;
    const grid_window w = grid_covered(D, G, L, lane);
    const double *c = D.tc + static_cast<std::size_t>(i) * (P.order + 1u) * n + lane;
    for (std::uint32_t idx = w.first; idx < w.last; ++idx) {
        const dfl g{G.grid[static_cast<std::size_t>(idx) * n + lane], 0.};
        const double tau = dfl_sub(g, w.start).hi;
        G.out[(static_cast<std::size_t>(idx) * P.n_eq + i) * n + lane]
            = eval_poly(P, [c, n](std::uint32_t o) { return c[static_cast<std::size_t>(o) * n]; }, tau);
    }
}

// The cursors past the grid points k_grid_sample() has written (:1899-1912).
__global__ void k_grid_advance(batch D, grid_state G, lockstep_state L)
{
    const std::uint32_t lane = blockIdx.x * blockDim.x + threadIdx.x;
    if (lane >= D.n || L.flags[1] != 0u) {
        return;
    }
    const grid_window w = grid_covered(D, G, L, lane);
    G.cur_idx[lane] = w.last;
    if (w.last < G.n_pts) {
        atomicOr(G.left, 1u);
    }
}

// Evaluation of a continuous output (src/continuous_output.cpp:640-960): per lane, upper_bound of the time in the
// lane's column of the (padded) times, the Taylor coefficients of the step that contains it, Horner / compensated
// summation at h = t - start of that step. times: [n_rows][batch] with n_rows = n_steps + 2 (padding included);
// tcs: [n_steps][n_eq][order + 1][batch], in slabs of slab_iters iterations (slabs[k] = iterations k * slab_iters ...).
__global__ void k_cout_eval(program P, std::uint32_t n, std::uint32_t n_rows, const double *const *slabs,
                            std::uint32_t slab_iters, const double *t_hi, const double *t_lo, const double *tm,
                            double *out)
{
    const std::uint32_t lane = blockIdx.x * blockDim.x + threadIdx.x;
    if (lane >= n) {
        return;
    }
    const std::size_t nn = n;
    const auto time_at = [&](std::uint32_t row) { return dfl{t_hi[row * nn + lane], t_lo[row * nn + lane]}; };
    // Direction: start < padding row (+-inf by direction), src/continuous_output.cpp:684-694.
    const bool dir = dfl_lt(time_at(0u), time_at(n_rows - 1u));
    const dfl t{tm[lane], 0.};
    std::uint32_t first = 0, count = n_rows;
    while (count != 0u) {
        const std::uint32_t step = count / 2u;
        std::uint32_t idx = first + step;
        const dfl v = time_at(idx);
        // !(t < v) forward, !(t > v) backward.
        const bool cond = dir ? !dfl_lt(t, v) : !dfl_lt(v, t);
        if (cond) {
            first = idx + 1u;
            count -= step + 1u;
        } else {
            count = step;
        }
    }
    std::uint32_t tc_idx = first;
    tc_idx -= (tc_idx != 0u) ? 1u : 0u;
    tc_idx -= (first == n_rows - 1u) ? 1u : 0u;
    const double h = dfl_sub(t, time_at(tc_idx)).hi;
    const double *base
        = slabs[tc_idx / slab_iters] + static_cast<std::size_t>(tc_idx % slab_iters) * P.n_eq * (P.order + 1u) * nn + lane;
    for (std::uint32_t i = 0; i < P.n_eq; ++i) {
        const double *c = base + static_cast<std::size_t>(i) * (P.order + 1u) * nn;
        out[static_cast<std::size_t>(i) * nn + lane]
            = eval_poly(P, [c, nn](std::uint32_t o) { return c[static_cast<std::size_t>(o) * nn]; }, h);
    }
}

// Self-test of the lean correctly-rounded division of the N-body kernel (nb::div_rn, nb_core.hpp) against the
// compiler's IEEE division: n pseudo-random pairs (splitmix64), three quarters with exponents within 2^+-300 (the
// fast path), one quarter over the whole range incl. zeros, denormals and infinities (the out-of-line division).
__global__ void k_selftest_div(unsigned long long n, unsigned long long seed, unsigned long long *mismatches)
{
    const auto mix = [](unsigned long long z) {
        z += 0x9e3779b97f4a7c15ull;
        z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
        z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
        return z ^ (z >> 31);
    };
    unsigned long long bad = 0;
    for (unsigned long long i = static_cast<unsigned long long>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
         i += static_cast<unsigned long long>(gridDim.x) * blockDim.x) {
        const unsigned long long r0 = mix(seed + 3ull * i), r1 = mix(seed + 3ull * i + 1ull), r2 = mix(seed + 3ull * i + 2ull);
        const auto make = [&](unsigned long long r, unsigned long long e) {
            const bool wide = (r2 & 3ull) == 0ull;
            const unsigned long long ex = wide ? (e % 2047ull) : (1023ull - 300ull + e % 601ull);
            return __longlong_as_double(static_cast<long long>((r & 0x800fffffffffffffull) | (ex << 52)));
        };
        const double a = make(r0, r2 >> 8), b = make(r1, r2 >> 24);
        const double q0 = nb::div_rn(a, b), q1 = __ddiv_rn(a, b);
        const bool same = __double_as_longlong(q0) == __double_as_longlong(q1) || (isnan(q0) && isnan(q1));
        bad += same ? 0ull : 1ull;
    }
    if (bad != 0ull) {
        atomicAdd(mismatches, bad);
    }
}

// Taylor map of a variational batch of order 1 (hy_batch_eval_taylor_map()): out_i = x_i + sum_j Phi_ij dx_j, with
// x = state rows [0, n_orig) and Phi_ij = state row n_orig + i * m + j. One thread per lane, lanes the coalesced axis.
// Fixed arithmetic, so that a sequential restatement gives the same bits: acc = x_i, then for j = 0 .. m - 1
// acc = acc + Phi_ij * dx_j with the product and the sum each rounded to nearest (__dmul_rn / __dadd_rn: no
// contraction). The kernel streams Phi once: dx is loaded once per lane into shared memory (a per-thread column, so no
// barrier is needed) in chunks of at most TMAP_CHUNK arguments and reused across the n_orig rows; with more arguments
// than one chunk the partial sums go through `out` between chunks, which keeps the order of the additions.
constexpr std::uint32_t TMAP_THREADS = 128, TMAP_CHUNK = 40;

__global__ void __launch_bounds__(TMAP_THREADS) k_taylor_map(const double *__restrict__ state, std::uint32_t n,
                                                             std::uint32_t n_orig, std::uint32_t m,
                                                             const double *__restrict__ dx, double *__restrict__ out)
{
    extern __shared__ double s_dx[]; // [chunk][TMAP_THREADS]
    const std::uint32_t lane = blockIdx.x * TMAP_THREADS + threadIdx.x;
    if (lane >= n) {
        return;
    }
    const std::size_t N = n;
    double *my_dx = s_dx + threadIdx.x;
    for (std::uint32_t j0 = 0; j0 < m; j0 += TMAP_CHUNK) {
        const std::uint32_t jn = min(TMAP_CHUNK, m - j0);
        for (std::uint32_t j = 0; j < jn; ++j) {
            my_dx[j * TMAP_THREADS] = dx[(j0 + j) * N + lane];
        }
        for (std::uint32_t i = 0; i < n_orig; ++i) {
            const double *phi = state + (n_orig + static_cast<std::size_t>(i) * m + j0) * N + lane;
            double acc = j0 == 0u ? state[i * N + lane] : out[i * N + lane];
#pragma unroll 8
            for (std::uint32_t j = 0; j < jn; ++j) {
                acc = __dadd_rn(acc, __dmul_rn(__ldcs(phi + j * N), my_dx[j * TMAP_THREADS]));
            }
            out[i * N + lane] = acc;
        }
    }
}

__global__ void k_fill_double(double *out, std::size_t n, double value)
{
    const std::size_t i = static_cast<std::size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < n) {
        out[i] = value;
    }
}

} // namespace heyoka_b200::dev

#endif
