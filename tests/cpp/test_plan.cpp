// Host-side checks of the shared-memory planner (csrc/smem_plan.cpp) on the 6-body outer Solar System program:
// tape sizes of the three residency modes, superinstructions found, level structure, bank-conflict-free layout.
#include <heyoka_b200/heyoka_b200.hpp>

#include <cstdio>
#include <set>
#include <vector>

#include "program.hpp"
#include "smem_plan.hpp"

using namespace heyoka_b200;

static int n_fail = 0;
#define REQUIRE(cond)                                                                                                  \
    do {                                                                                                               \
        if (!(cond)) {                                                                                                 \
            std::printf("REQUIRE failed at %s:%d: %s\n", __FILE__, __LINE__, #cond);                                   \
            ++n_fail;                                                                                                  \
        }                                                                                                              \
    } while (0)

int main()
{
    const std::vector<double> masses{1.00000597682, 1 / 1047.355, 1 / 3501.6, 1 / 22869., 1 / 19314., 7.4074074e-09};
    auto sys = model::nbody(6, kw::masses = masses, kw::Gconst = 0.01720209895 * 0.01720209895 * 365 * 365);
    auto [dc, sv] = taylor_decompose_sys(sys, {});
    const auto P = detail::lower_decomposition(dc, 36, 0, 20, true);
    REQUIRE(P.n_uvars == 234u);

    // Reference tape: n_uvars * order + n_eq (src/taylor_02.cpp:1227-1233) = 234 * 20 + 36 = 4716 doubles per lane.
    const auto plain = detail::make_smem_plan(P, false, false, false);
    const auto fused = detail::make_smem_plan(P, true, true, false);
    std::printf("slots per lane: unfused %u, fused %u\n", plain.n_slots, fused.n_slots);
    REQUIRE(plain.n_slots < 234u * 21u / 2u);
    REQUIRE(fused.n_fused == 15u && fused.n_segments == 2u);
    REQUIRE(fused.n_slots == 1761u);            // 16 warps x 2 lanes would need 2 x 8 x 1761 x 16 = 450 KB: 8 warps fit
    // Level 0 = the 15 pair interactions, level 1 = the 18 sums.
    REQUIRE(fused.seg_offsets.size() == 3u && fused.seg_offsets[1] - fused.seg_offsets[0] == 15u
            && fused.seg_offsets[2] - fused.seg_offsets[1] == 18u);
    for (std::size_t i = 0; i < fused.ops.size(); ++i) {
        REQUIRE(fused.ops[i].opcode == (i < 15u ? detail::HY_FOP_NBODY_PAIR : detail::HY_FOP_SUM_T));
    }
    // Bank-conflict-free layout: for every role of the pair superinstruction (the three differences, r^2, r^alpha),
    // the first slots of 8 consecutive pairs are distinct modulo 8 (a slot is 16 bytes with 2 lanes per warp).
    for (const std::uint32_t role : {2u, 5u, 8u, 9u, 10u}) {
        for (std::size_t first = 0; first + 8u <= 15u; ++first) {
            std::set<std::uint32_t> banks;
            for (std::size_t i = first; i < first + 8u; ++i) {
                const auto ref = fused.aux[fused.ops[i].a + role];
                banks.insert((ref & ((1u << detail::ROW_SLOT_BITS) - 1u)) % 8u);
            }
            REQUIRE(banks.size() == 8u);
        }
    }
    // model::nbody with 32 bodies: 496 pair interactions in level 0, sums of up to 31 terms split at 8 (src/taylor_01.cpp split_sums), a tape far beyond shared memory.
    {
        std::vector<double> m32(32, 1e-4);
        m32[0] = 1.;
        auto sys32 = model::nbody(32, kw::masses = m32);
        auto [dc32, sv32] = taylor_decompose_sys(sys32, {});
        const auto P32 = detail::lower_decomposition(dc32, 192, 0, 20, false);
        const auto pl = detail::make_smem_plan(P32, true, true, false);
        std::printf("N = 32: %u u variables, %u superinstructions, %u levels, %u slots per lane\n", P32.n_uvars,
                    pl.n_fused, pl.n_segments, pl.n_slots);
        REQUIRE(pl.n_fused == 496u);
        REQUIRE(pl.seg_offsets[1] - pl.seg_offsets[0] == 496u);
        REQUIRE(pl.n_slots * 8u > 227u * 1024u); // one lane alone does not fit in an SM's shared memory
    }
    if (n_fail == 0) {
        std::printf("ALL PASSED\n");
        return 0;
    }
    return 1;
}
