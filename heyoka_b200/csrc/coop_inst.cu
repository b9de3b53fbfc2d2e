// One family of instantiations of the cooperative kernel (see coop_variants.hpp). Compiled several times with
// different -DHY_COOP_N / -DHY_COOP_MAXT.
#include "coop_variants.hpp"
#include "kernels.cuh"

#if !defined(HY_COOP_N) || !defined(HY_COOP_MAXT) || !defined(HY_COOP_MODE)
#error "HY_COOP_N, HY_COOP_MAXT and HY_COOP_MODE must be defined"
#endif

#define HY_CAT_(a, b, c, d, e, f) a##b##c##d##e##f
#define HY_CAT(a, b, c, d, e, f) HY_CAT_(a, b, c, d, e, f)

namespace heyoka_b200::detail
{

namespace
{

#define HY_COOP(L)                                                                                                     \
    coop_variant                                                                                                       \
    {                                                                                                                  \
        L, HY_COOP_N, HY_COOP_MAXT, HY_COOP_MODE, dev::k_coop<L, HY_COOP_N, false, HY_COOP_MAXT, HY_COOP_MODE>,           \
            dev::k_coop<L, HY_COOP_N, true, HY_COOP_MAXT, HY_COOP_MODE>                                                 \
    }

const coop_variant family[] = {
#if HY_COOP_MODE == 5 && HY_COOP_N == 1
    // Tape in global memory, one CTA per chunk of lanes.
    HY_COOP(1), HY_COOP(2)
#elif HY_COOP_MODE == 5 && HY_COOP_N == 2
    HY_COOP(2), HY_COOP(4)
#elif HY_COOP_MODE == 4 && HY_COOP_N == 1
    // Tape in global memory: a few lanes per warp.
    HY_COOP(1), HY_COOP(2), HY_COOP(4)
#elif HY_COOP_MODE == 4 && HY_COOP_N == 2
    HY_COOP(2), HY_COOP(4), HY_COOP(8)
#elif HY_COOP_N == 1
    HY_COOP(1),  HY_COOP(2), HY_COOP(4), HY_COOP(8), HY_COOP(16), HY_COOP(32)
#elif HY_COOP_N == 2
    HY_COOP(2), HY_COOP(4), HY_COOP(8), HY_COOP(16), HY_COOP(32)
#elif HY_COOP_N == 4
    HY_COOP(4), HY_COOP(8), HY_COOP(16), HY_COOP(32)
#else
#error "unsupported HY_COOP_N"
#endif
};

} // namespace

coop_family HY_CAT(coop_family_n, HY_COOP_N, _, HY_COOP_MAXT, _m, HY_COOP_MODE)()
{
    return {family, sizeof(family) / sizeof(family[0])};
}

} // namespace heyoka_b200::detail
