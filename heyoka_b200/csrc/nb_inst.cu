// One family of instantiations of the N-body kernel (see nb_variants.hpp). Compiled several times with different
// -DHY_NB_LT / -DHY_NB_CTA.
#include "nb_variants.hpp"
#include "nb_kernel.cuh"

#if !defined(HY_NB_LT) || !defined(HY_NB_CTA)
#error "HY_NB_LT and HY_NB_CTA must be defined"
#endif

#define HY_NB_CAT_(a, b, c, d) a##b##c##d
#define HY_NB_CAT(a, b, c, d) HY_NB_CAT_(a, b, c, d)

namespace heyoka_b200::detail
{

namespace
{

#define HY_NB(OFF, MAXT)                                                                                               \
    nb_variant                                                                                                         \
    {                                                                                                                  \
        HY_NB_LT, HY_NB_CTA != 0, OFF, MAXT, dev::k_nb<HY_NB_LT, HY_NB_CTA != 0, OFF, false, MAXT>,                    \
            dev::k_nb<HY_NB_LT, HY_NB_CTA != 0, OFF, true, MAXT>                                                       \
    }

const nb_variant family[] = {
#if HY_NB_CTA != 0
    HY_NB(false, 512), HY_NB(true, 512)
#else
    HY_NB(false, 512), HY_NB(false, 384), HY_NB(false, 256)
#endif
};

} // namespace

nb_family HY_NB_CAT(nb_family_lt, HY_NB_LT, _cta, HY_NB_CTA)()
{
    return {family, sizeof(family) / sizeof(family[0])};
}

} // namespace heyoka_b200::detail

#if defined(HY_NB_PHASE_CLOCK)
// The phase counters of this family's kernels (nb_kernel.cuh): copies the first n / NB_PH_SLOTS teams' counters to out
// and resets them all; with out == nullptr only resets them. Returns the number of teams the counters have room for,
// or -1 on a CUDA error.
extern "C" int HY_NB_CAT(hy_nb_phase_clock_lt, HY_NB_LT, _cta, HY_NB_CTA)(unsigned long long *out, std::size_t n)
{
    namespace hd = heyoka_b200::dev;
    constexpr std::size_t total = static_cast<std::size_t>(hd::nb_phase_teams) * hd::NB_PH_SLOTS;
    n = n < total ? n : total;
    if (out != nullptr && cudaMemcpyFromSymbol(out, hd::nb_phase_cycles, n * sizeof(unsigned long long)) != cudaSuccess) {
        return -1;
    }
    static const unsigned long long zero[total] = {};
    if (cudaMemcpyToSymbol(hd::nb_phase_cycles, zero, sizeof(zero)) != cudaSuccess) {
        return -1;
    }
    return static_cast<int>(hd::nb_phase_teams);
}
#endif
