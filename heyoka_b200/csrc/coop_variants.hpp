// Table of the compiled instantiations of the cooperative kernel dev::k_coop<L, N, PROP, MAXT>. Each (N, MAXT)
// family is explicitly instantiated in its own translation unit (coop_inst.cu compiled with -DHY_COOP_N=...
// -DHY_COOP_MAXT=... -DHY_COOP_MODE=...), so that the families build in parallel.
#ifndef HEYOKA_B200_CSRC_COOP_VARIANTS_HPP
#define HEYOKA_B200_CSRC_COOP_VARIANTS_HPP

#include <cstddef>
#include <cstdint>

#include "device_program.cuh"

namespace heyoka_b200::dev
{
struct run_args; // kernels.cuh
}

namespace heyoka_b200::detail
{

using coop_fn = void (*)(dev::program, const std::uint32_t *, dev::batch, dev::run_args, double *);

struct coop_variant {
    int L, N, maxt; // lanes per warp, lanes per thread, maximum threads per CTA
    int mode;       // HY_COOP_MODE (not hy_kernel_info::tape_mode): 1: handles elementary ops, 0: superinstruction-only
                    // programs, 4: tape in global memory, 5: idem, CTA-wide teams
    coop_fn step, prop;
};

struct coop_family {
    const coop_variant *v;
    std::size_t n;
};

coop_family coop_family_n1_512_m1();
coop_family coop_family_n1_512_m0();
coop_family coop_family_n1_256_m1();
coop_family coop_family_n1_256_m0();
coop_family coop_family_n2_512_m1();
coop_family coop_family_n2_512_m0();
coop_family coop_family_n2_256_m1();
coop_family coop_family_n2_256_m0();
coop_family coop_family_n4_512_m1();
coop_family coop_family_n4_512_m0();
coop_family coop_family_n4_256_m1();
coop_family coop_family_n4_256_m0();
coop_family coop_family_n1_512_m4();
coop_family coop_family_n2_512_m4();
coop_family coop_family_n1_512_m5();
coop_family coop_family_n2_512_m5();

} // namespace heyoka_b200::detail

#endif
