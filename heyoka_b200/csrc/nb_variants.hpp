// Table of the compiled instantiations of the N-body kernel dev::k_nb<LT, CTA, OFFCHIP, PROP, MAXT> (nb_kernel.cuh). Each
// (LT, CTA) family is instantiated in its own translation unit (nb_inst.cu compiled with -DHY_NB_LT=... -DHY_NB_CTA=...),
// so that the families build in parallel.
#ifndef HEYOKA_B200_CSRC_NB_VARIANTS_HPP
#define HEYOKA_B200_CSRC_NB_VARIANTS_HPP

#include <cstddef>

#include "device_program.cuh"

namespace heyoka_b200::dev
{
struct run_args;    // kernels.cuh
struct nb_dev_plan; // nb_kernel.cuh
} // namespace heyoka_b200::dev

namespace heyoka_b200::detail
{

using nb_fn = void (*)(dev::program, dev::nb_dev_plan, dev::batch, dev::run_args);

struct nb_variant {
    int LT;    // lanes per team
    bool cta;  // a team is a whole CTA (of exactly maxt threads), else a warp
    bool offchip; // r^2, d_2, r^alpha rows in an L2-resident slab of global memory (CTA teams)
    int maxt;  // maximum threads per CTA (256: up to 255 registers per thread, 384: 168, 512: 128)
    nb_fn step, prop;
    bool lane = false; // one thread per lane, systems with one pair interaction (k_nb1, nb1_kernel.cuh)
};

struct nb_family {
    const nb_variant *v;
    std::size_t n;
};

nb_family nb_family_lt1_cta0();
nb_family nb_family_lt2_cta0();
nb_family nb_family_lt4_cta0();
nb_family nb_family_lt8_cta0();
nb_family nb_family_lt16_cta0();
nb_family nb_family_lt32_cta0();
nb_family nb_family_lt1_cta1();
nb_family nb_family_lane();

} // namespace heyoka_b200::detail

#endif
