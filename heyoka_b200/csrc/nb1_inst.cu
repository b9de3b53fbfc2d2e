// The instantiations of the one-thread-per-lane N-body kernel (nb1_kernel.cuh), see nb_variants.hpp.
#include "nb_variants.hpp"
#include "nb1_kernel.cuh"

namespace heyoka_b200::detail
{

namespace
{

#define HY_NB1(MAXT)                                                                                                   \
    nb_variant                                                                                                         \
    {                                                                                                                  \
        32, false, false, MAXT, dev::k_nb1<false, false, MAXT>, dev::k_nb1<false, true, MAXT>, true                    \
    }

const nb_variant family[] = {HY_NB1(512), HY_NB1(384), HY_NB1(256)};

} // namespace

nb_family nb_family_lane()
{
    return {family, sizeof(family) / sizeof(family[0])};
}

} // namespace heyoka_b200::detail
