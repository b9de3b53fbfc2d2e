// TEST INFRASTRUCTURE: the arithmetic of the device's dense-output paths restated on the host, without the device
// headers, so that tests/test_gpu_cout_eval.py can hold k_cout_eval, k_grid_sample and k_d_output (small_kernels.cuh)
// to it bit for bit. Compiled with -ffp-contract=off: every + - * below is rounded on its own, and the fused
// multiply-add of the Horner loop is std::fma (correctly rounded, like the device's fma). It is never linked into the
// product library.
#include <cmath>
#include <cstddef>
#include <cstdint>

namespace
{

struct dfl {
    double hi, lo;
};

// Double-length arithmetic (include/heyoka/detail/dfloat.hpp): Knuth's and Dekker's error-free sums.
dfl two_sum(double a, double b)
{
    const double x = a + b, z = x - a;
    return {x, (a - (x - z)) + (b - z)};
}
dfl fast_two_sum(double a, double b)
{
    const double x = a + b;
    return {x, (a - x) + b};
}
dfl add(dfl a, dfl b)
{
    const dfl h = two_sum(a.hi, b.hi), l = two_sum(a.lo, b.lo);
    dfl r = fast_two_sum(h.hi, h.lo + l.hi);
    return fast_two_sum(r.hi, r.lo + l.lo);
}
dfl sub(dfl a, dfl b)
{
    return add(a, dfl{-b.hi, -b.lo});
}
bool lt(dfl a, dfl b)
{
    return a.hi < b.hi || (a.hi == b.hi && a.lo < b.lo);
}

// One Taylor polynomial at h; c[o * stride] is the order-o coefficient. mode 0: Horner with fma; 1: compensated
// summation of the monomials (high-accuracy mode); 2: Horner with the product and the sum rounded apart (the CPU
// oracle's dense output, not a device form).
double poly(const double *c, std::size_t stride, unsigned p, int mode, double h)
{
    if (mode == 1) {
        double res = c[0], comp = 0., cur = h;
        for (unsigned o = 1; o <= p; ++o) {
            const double y = c[o * stride] * cur - comp;
            const double t = res + y;
            comp = (t - res) - y;
            res = t;
            cur = cur * h;
        }
        return res;
    }
    double res = c[p * stride];
    for (unsigned o = 1; o <= p; ++o) {
        res = mode == 0 ? std::fma(res, h, c[(p - o) * stride]) : res * h + c[(p - o) * stride];
    }
    return res;
}

} // namespace

extern "C" {

// out[i][lane] = P_{step[lane]} of state variable i at h[lane], from the coefficients of lane src[lane] (src may be
// null: the lane itself). tcs: [n_steps][n_eq][p + 1][n].
void ce_eval(unsigned n_eq, unsigned p, std::uint64_t n, int mode, const double *tcs, const std::int64_t *step,
             const std::uint64_t *src, const double *h, double *out)
{
    for (std::uint64_t lane = 0; lane < n; ++lane) {
        const std::uint64_t l = src != nullptr ? src[lane] : lane;
        const double *base = tcs + static_cast<std::size_t>(step[lane]) * n_eq * (p + 1u) * n + l;
        for (unsigned i = 0; i < n_eq; ++i) {
            out[i * n + lane] = poly(base + static_cast<std::size_t>(i) * (p + 1u) * n, n, p, mode, h[lane]);
        }
    }
}

// The step k_cout_eval() evaluates at tm[lane]: upper_bound over the lane's column of the n_rows padded times (forward
// if row 0 < the padding row, then t < v decides; backward v < t), the row before it, and one row less when the time
// is past the last recorded one.
void ce_select(std::uint64_t n, std::uint64_t n_rows, const double *t_hi, const double *t_lo, const double *tm,
               std::int64_t *step)
{
    for (std::uint64_t lane = 0; lane < n; ++lane) {
        const auto at = [&](std::uint64_t r) { return dfl{t_hi[r * n + lane], t_lo[r * n + lane]}; };
        const bool fwd = lt(at(0), at(n_rows - 1u));
        const dfl t{tm[lane], 0.};
        std::uint64_t first = 0, count = n_rows;
        while (count != 0u) {
            const std::uint64_t half = count / 2u, idx = first + half;
            if (fwd ? !lt(t, at(idx)) : !lt(at(idx), t)) {
                first = idx + 1u;
                count -= half + 1u;
            } else {
                count = half;
            }
        }
        std::uint64_t k = first;
        k -= k != 0u ? 1u : 0u;
        k -= first == n_rows - 1u ? 1u : 0u;
        step[lane] = static_cast<std::int64_t>(k);
    }
}

// h[lane] = (tm - times[step]).hi in double-length arithmetic; hi_only != 0 drops the low word of the time.
void ce_h(std::uint64_t n, const double *t_hi, const double *t_lo, const std::int64_t *step, const double *tm,
          int hi_only, double *h)
{
    for (std::uint64_t lane = 0; lane < n; ++lane) {
        const std::size_t r = static_cast<std::size_t>(step[lane]) * n + lane;
        h[lane] = sub(dfl{tm[lane], 0.}, dfl{t_hi[r], hi_only != 0 ? 0. : t_lo[r]}).hi;
    }
}

// propagate_grid()'s sampling after one step (grid_covered() and k_grid_sample()): the step spans [t - last_h, t],
// closed at both ends; from the cursor cur[lane], the grid points inside it are taken, or every remaining point once
// the lane is at its target (rem0). Writes the dense output of those points into out [n_pts][n_eq][n] with
// tau = (g - (t - last_h)).hi, evaluated on tc [n_eq][p + 1][n] in the given mode, and moves the cursors.
void ce_grid_sample(unsigned n_eq, unsigned p, std::uint64_t n, int mode, std::uint64_t n_pts, const double *grid,
                    const double *t_hi, const double *t_lo, const double *last_h, const unsigned char *rem0,
                    const double *tc, std::uint64_t *cur, double *out)
{
    for (std::uint64_t lane = 0; lane < n; ++lane) {
        const dfl t{t_hi[lane], t_lo[lane]}, start = sub(t, dfl{last_h[lane], 0.});
        const dfl t0 = lt(start, t) ? start : t, t1 = lt(t, start) ? start : t;
        for (; cur[lane] < n_pts; ++cur[lane]) {
            const dfl g{grid[cur[lane] * n + lane], 0.};
            if (!((!lt(g, t0) && !lt(t1, g)) || rem0[lane] != 0)) {
                break;
            }
            const double tau = sub(g, start).hi;
            for (unsigned i = 0; i < n_eq; ++i) {
                out[(cur[lane] * n_eq + i) * n + lane]
                    = poly(tc + static_cast<std::size_t>(i) * (p + 1u) * n + lane, n, p, mode, tau);
            }
        }
    }
}

// update_d_output()'s tau: rel_time: last_h + t; absolute: (t - (time - last_h)).hi in double-length arithmetic.
void ce_tau(std::uint64_t n, int rel_time, const double *t, const double *t_hi, const double *t_lo, const double *last_h,
            double *tau)
{
    for (std::uint64_t lane = 0; lane < n; ++lane) {
        tau[lane] = rel_time != 0 ? last_h[lane] + t[lane]
                                  : sub(dfl{t[lane], 0.}, sub(dfl{t_hi[lane], t_lo[lane]}, dfl{last_h[lane], 0.})).hi;
    }
}

} // extern "C"
