// The arithmetic of the angle reducer (callback::angle_reducer, include/heyoka_b200/callback.hpp), shared by the
// kernels and by the host library (hy_reduce_angles()) so that the device path and the host loops produce the same
// bits. Every operation is rounded on its own: __dmul_rn / __dsub_rn / __dadd_rn / __ddiv_rn on the device; on the
// host the library is compiled with -ffp-contract=off (build.py), so no FMA can contract a product into a sum. This
// function must not move to a public header, where a user's compiler flags could contract it.
#ifndef HEYOKA_B200_CSRC_ANGLE_REDUCE_HPP
#define HEYOKA_B200_CSRC_ANGLE_REDUCE_HPP

#include <cmath>

#if defined(__CUDACC__)
#define HY_AR_HD __host__ __device__ __forceinline__
#else
#define HY_AR_HD inline
#endif

namespace heyoka_b200::detail
{

// 2 pi rounded to the nearest double (0x1.921fb54442d18p+2).
constexpr double angle_two_pi = 6.283185307179586;

HY_AR_HD double ar_mul(double a, double b)
{
#if defined(__CUDA_ARCH__)
    return __dmul_rn(a, b);
#else
    return a * b;
#endif
}
HY_AR_HD double ar_sub(double a, double b)
{
#if defined(__CUDA_ARCH__)
    return __dsub_rn(a, b);
#else
    return a - b;
#endif
}
HY_AR_HD double ar_add(double a, double b)
{
#if defined(__CUDA_ARCH__)
    return __dadd_rn(a, b);
#else
    return a + b;
#endif
}
HY_AR_HD bool ar_finite(double a)
{
#if defined(__CUDA_ARCH__)
    return ::isfinite(a);
#else
    return std::isfinite(a);
#endif
}
HY_AR_HD double ar_floor(double a)
{
#if defined(__CUDA_ARCH__)
    return ::floor(a);
#else
    return std::floor(a);
#endif
}
HY_AR_HD double ar_div(double a, double b)
{
#if defined(__CUDA_ARCH__)
    return __ddiv_rn(a, b);
#else
    return a / b;
#endif
}

// x reduced into [0, 2pi): a finite x outside that range becomes r = x - 2pi * floor(x / 2pi), with 2pi the double
// above, then the fix-ups that the rounding of the product makes necessary: a slightly negative r gets 2pi added, an r
// at or above 2pi (also the 2pi that a tiny negative r rounds to) gets 2pi subtracted. One pass suffices while the
// product's rounding error is below 2pi, i.e. for |x| below about 2^53; for larger |x| the residue of a pass is a few
// units in the last place of x, and the passes repeat on it (about 20 passes at 1e300). Near the top of the range the
// product may overflow: the multiple of 2pi is then taken off in two halves (q is even there). Non-finite values and
// values already in [0, 2pi) (-0. included) are returned as they are.
HY_AR_HD double reduce_angle(double x)
{
    if (!ar_finite(x)) {
        return x;
    }
    double r = x;
    while (!(r >= 0. && r < angle_two_pi)) {
        double q = ar_floor(ar_div(r, angle_two_pi));
        const double m = ar_mul(angle_two_pi, q);
        if (ar_finite(m)) {
            r = ar_sub(r, m);
        } else {
            q = ar_mul(q, 0.5);
            const double m2 = ar_mul(angle_two_pi, q);
            r = ar_sub(ar_sub(r, m2), m2);
        }
        if (r < 0.) {
            r = ar_add(r, angle_two_pi);
        }
        if (r >= angle_two_pi) {
            r = ar_sub(r, angle_two_pi);
        }
    }
    return r;
}

} // namespace heyoka_b200::detail

#undef HY_AR_HD

#endif
