// Host-side planning for the dense-network kernel (nn_kernel.cuh).
//
// A program qualifies when its right-hand side is a feed-forward network of dense layers, x' = ffnn(x)
// (src/model/ffnn.cpp:36-142): after decomposition every neuron is a (nested, <= 8 terms per node: src/math/sum.cpp)
// sum of products w_ij * in_j plus a bias (weights of +-1 folded into plain inputs, negations and differences),
// followed by tanh (with its hidden dependency tanh^2, src/math/tanh.cpp) or,
// for the output layer, by nothing. The planner walks those sums back into what they are - one weight matrix and one
// bias vector per layer - so that the device can evaluate a layer of every Taylor order as ONE matrix product
// [n_out x n_in] . [n_in x lanes] on the FP64 tensor cores (mma.sync.m8n8k4.f64) instead of interpreting ~10^4 products
// and sums one at a time. The tanh / square recurrences keep the reference's arithmetic; the matrix product sums the
// same products in a different association (and fused): that is the one place where the Taylor coefficients differ
// from the generic path, by a few units of rounding (bound stated and tested in tests/test_gpu_parity.py).
#ifndef HEYOKA_B200_CSRC_NN_PLAN_HPP
#define HEYOKA_B200_CSRC_NN_PLAN_HPP

#include <cstdint>
#include <string>
#include <vector>

#include "program.hpp"

namespace heyoka_b200::detail
{

struct nn_layer {
    std::uint32_t n_in = 0, n_out = 0;
    int act = 0;               // 0: none (output layer), 1: tanh
    std::vector<double> w;     // row-major [n_out][n_in]
    std::vector<double> bias;  // [n_out]
    std::vector<std::uint32_t> u_out; // u variable of every neuron's pre-activation (diagnostics)
};

struct nn_plan {
    bool ok = false;
    std::string why;
    std::vector<nn_layer> layers;         // layers[0] reads the state variables (n_in = n_eq)
    std::vector<std::uint32_t> out_of_sv; // state variable i derives from output neuron out_of_sv[i] of the last layer
};

nn_plan make_nn_plan(const hy_program &);

} // namespace heyoka_b200::detail

#endif
