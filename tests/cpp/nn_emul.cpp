// TEST INFRASTRUCTURE: the dense-network planner (heyoka_b200/csrc/nn_plan.cpp) called on a program, its result copied
// to plain arrays, so that tests/test_gpu_nn_shapes.py can check WITHOUT a GPU that the matrices the planner rebuilds
// from the decomposition are the weights the network was built with, and restate setup_nn() (batch.cu) from them. It is
// never linked into the product library.
#include <cstdint>
#include <cstring>

#include <heyoka_b200.h>

#include "nn_plan.hpp"

namespace hb = heyoka_b200;

extern "C" {

// info[0] = ok, info[1] = number of layers, info[2 + 3 l ..] = n_in, n_out, act of layer l (at most 8 layers: the
// planner refuses deeper networks). out_of_sv[n_eq]. w: every layer's row-major [n_out][n_in] block, one after the
// other (w_cap doubles); bias: every layer's [n_out] (b_cap doubles). Either may be null. Returns 0, -2 if w or bias
// is too small.
int nn_emul_plan(const hy_program *p, std::uint32_t *info, char *why, std::size_t why_len, std::uint32_t *out_of_sv,
                 double *w, std::size_t w_cap, double *bias, std::size_t b_cap)
{
    const auto pl = hb::detail::make_nn_plan(*p);
    info[0] = pl.ok ? 1u : 0u;
    info[1] = static_cast<std::uint32_t>(pl.layers.size());
    if (why != nullptr && why_len != 0u) {
        std::strncpy(why, pl.why.c_str(), why_len - 1u);
        why[why_len - 1u] = '\0';
    }
    if (!pl.ok) {
        return 0;
    }
    std::size_t nw = 0, nb = 0;
    for (std::size_t l = 0; l < pl.layers.size() && l < 8u; ++l) {
        const auto &L = pl.layers[l];
        info[2u + 3u * l] = L.n_in;
        info[3u + 3u * l] = L.n_out;
        info[4u + 3u * l] = static_cast<std::uint32_t>(L.act);
        nw += L.w.size();
        nb += L.bias.size();
    }
    for (std::size_t s = 0; s < pl.out_of_sv.size(); ++s) {
        out_of_sv[s] = pl.out_of_sv[s];
    }
    if ((w != nullptr && nw > w_cap) || (bias != nullptr && nb > b_cap)) {
        return -2;
    }
    for (const auto &L : pl.layers) {
        if (w != nullptr) {
            std::memcpy(w, L.w.data(), L.w.size() * sizeof(double));
            w += L.w.size();
        }
        if (bias != nullptr) {
            std::memcpy(bias, L.bias.data(), L.bias.size() * sizeof(double));
            bias += L.bias.size();
        }
    }
    return 0;
}

} // extern "C"
