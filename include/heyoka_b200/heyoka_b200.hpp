// heyoka_b200 — umbrella header of the C++ API (the part of heyoka's <heyoka/heyoka.hpp> that the batch Taylor
// hot path needs: expressions, models, kw::, taylor_adaptive_batch<double>, ensemble propagation).
// A reference user can switch with `namespace heyoka = heyoka_b200;`.
#ifndef HEYOKA_B200_HEYOKA_B200_HPP
#define HEYOKA_B200_HEYOKA_B200_HPP

#include <heyoka_b200/callback.hpp>
#include <heyoka_b200/expression.hpp>
#include <heyoka_b200/kw.hpp>
#include <heyoka_b200/model.hpp>
#include <heyoka_b200/taylor.hpp>
#include <heyoka_b200/taylor_decompose.hpp>
#include <heyoka_b200/var_ode_sys.hpp>

#endif
