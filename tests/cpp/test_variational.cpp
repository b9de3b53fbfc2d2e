// C++ API tests for variational integrators: diff(), var_ode_sys, and taylor_adaptive_batch<double> built from a
// var_ode_sys (getters, IC fill, eval_taylor_map() / get_tstate(), refusals). Run by tests/test_variational_cpp.py.
//
//   test_variational cpu   -> symbolic layer and refusals (no CUDA device needed)
//   test_variational gpu   -> everything
#include <cmath>
#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include <heyoka_b200/heyoka_b200.hpp>

using namespace heyoka_b200;

static int n_fail = 0;
#define REQUIRE(cond)                                                                                                  \
    do {                                                                                                               \
        if (!(cond)) {                                                                                                 \
            std::printf("REQUIRE failed at %s:%d: %s\n", __FILE__, __LINE__, #cond);                                   \
            ++n_fail;                                                                                                  \
        }                                                                                                              \
    } while (0)
#define REQUIRE_THROWS(expr, exc)                                                                                      \
    do {                                                                                                               \
        bool ok_ = false;                                                                                              \
        try {                                                                                                          \
            expr;                                                                                                      \
        } catch (const exc &) {                                                                                        \
            ok_ = true;                                                                                                \
        } catch (...) {                                                                                                \
        }                                                                                                              \
        if (!ok_) {                                                                                                    \
            std::printf("REQUIRE_THROWS failed at %s:%d: %s\n", __FILE__, __LINE__, #expr);                            \
            ++n_fail;                                                                                                  \
        }                                                                                                              \
    } while (0)

using sys_t = std::vector<std::pair<expression, expression>>;

static sys_t osc()
{
    auto [x, v] = make_vars("x", "v");
    return {prime(x) = v, prime(v) = -par[0] * par[0] * x};
}

static void test_symbolic()
{
    auto [x, y] = make_vars("x", "y");
    REQUIRE(diff(x, x) == expression{1.});
    REQUIRE(diff(x, y) == expression{0.});
    REQUIRE(diff(par[0], par[0]) == expression{1.});
    REQUIRE(diff(heyoka_b200::time, x) == expression{0.});
    REQUIRE(diff(x * y, y) == x);
    REQUIRE_THROWS(diff(x, expression{2.}), std::invalid_argument);
    // The functions the decomposition creates are refused rather than guessed.
    REQUIRE_THROWS(diff(expression{func_kind::sub, {x, y}}, x), std::invalid_argument);
    REQUIRE_THROWS(diff(expression{func_kind::div, {x, y}}, x), std::invalid_argument);
    REQUIRE_THROWS(diff(expression{func_kind::sum_sq, {x, y}}, x), std::invalid_argument);

    const auto sys = osc();
    const var_ode_sys vs(sys, var_args::vars | var_args::params);
    REQUIRE(vs.get_n_orig_sv() == 2u && vs.get_order() == 1u);
    REQUIRE(vs.get_vargs().size() == 3u && vs.get_vargs()[2] == par[0]);
    REQUIRE(vs.get_sys().size() == 8u);
    REQUIRE(to_string(vs.get_sys()[2].first) == "∂[(0, 1)]x");
    REQUIRE(to_string(vs.get_sys()[7].first) == "∂[(2, 1)]v");
    const var_ode_sys vl(sys, std::vector<expression>{par[0], sys[1].first});
    REQUIRE(vl.get_vargs()[0] == par[0] && vl.get_vargs()[1] == sys[1].first);

    REQUIRE_THROWS(var_ode_sys(sys, var_args::vars, 0u), std::invalid_argument);
    REQUIRE_THROWS(var_ode_sys(sys, var_args::vars, 2u), not_implemented_error);
    REQUIRE_THROWS(var_ode_sys(sys, var_args::time), not_implemented_error);
    REQUIRE_THROWS(var_ode_sys(sys, std::vector<expression>{}), std::invalid_argument);
    REQUIRE_THROWS(var_ode_sys(sys, std::vector<expression>{x, x}), std::invalid_argument);
    REQUIRE_THROWS(var_ode_sys(sys, std::vector<expression>{y}), std::invalid_argument);
}

static void test_integrator()
{
    const auto sys = osc();
    const var_ode_sys vs(sys, std::vector<expression>{sys[0].first, sys[1].first, par[0]});
    const std::uint32_t batch = 3;
    const std::vector<double> w{0.9, 1.1, 1.4};
    taylor_adaptive_batch<double> ta(vs, {0.5, 0.6, 0.7, -0.1, 0.0, 0.1}, batch, kw::pars = w);
    REQUIRE(ta.is_variational() && ta.get_n_orig_sv() == 2u && ta.get_dim() == 8u && ta.get_vorder() == 1u);
    REQUIRE(ta.get_vargs().size() == 3u && ta.get_sys().size() == 8u);
    REQUIRE(ta.get_vslice(0) == std::make_pair(0u, 2u) && ta.get_vslice(1) == std::make_pair(2u, 8u));
    REQUIRE(ta.get_vslice(1u, 1u) == std::make_pair(5u, 8u));
    REQUIRE((ta.get_mindex(0) == std::vector<std::uint32_t>{0, 0, 0, 0}));
    REQUIRE((ta.get_mindex(7) == std::vector<std::uint32_t>{1, 0, 0, 1}));
    REQUIRE_THROWS((void)ta.get_vslice(2), std::invalid_argument);
    REQUIRE_THROWS((void)ta.get_vslice(2u, 1u), std::invalid_argument);
    REQUIRE_THROWS((void)ta.get_mindex(8), std::invalid_argument);
    // IC fill: STM rows 2.. = [[1, 0, 0], [0, 1, 0]] per lane.
    const auto &st = ta.get_state();
    for (std::uint32_t lane = 0; lane < batch; ++lane) {
        const double want[6] = {1, 0, 0, 0, 1, 0};
        for (int r = 0; r < 6; ++r) {
            REQUIRE(st[(2 + r) * batch + lane] == want[r]);
        }
    }
    ta.propagate_until(2.0);
    const double t = 2.0;
    std::vector<double> dx(3 * batch, 0.);
    for (std::uint32_t lane = 0; lane < batch; ++lane) {
        dx[lane] = 1e-4; // dx0 only
    }
    const auto &tm = ta.eval_taylor_map(dx);
    REQUIRE(&tm == &ta.get_tstate() && tm.size() == 2u * batch);
    const auto &s = ta.get_state();
    for (std::uint32_t lane = 0; lane < batch; ++lane) {
        // x + Phi[:, 0] * 1e-4, with Phi[0][0] = cos(w t), Phi[1][0] = -w sin(w t).
        REQUIRE(std::abs(s[2 * batch + lane] - std::cos(w[lane] * t)) < 1e-12);
        REQUIRE(tm[lane] == s[lane] + s[2 * batch + lane] * 1e-4);
        REQUIRE(tm[batch + lane] == s[batch + lane] + s[5 * batch + lane] * 1e-4);
    }
    REQUIRE_THROWS(ta.eval_taylor_map(std::vector<double>(2 * batch)), std::invalid_argument);
    // A copy keeps the variational structure.
    const auto cp = ta;
    REQUIRE(cp.is_variational() && cp.get_vargs().size() == 3u && cp.get_tstate() == ta.get_tstate());

    // A full-size state is taken as given.
    std::vector<double> full(8 * batch, 0.5);
    taylor_adaptive_batch<double> tf(vs, full, batch, kw::pars = w);
    REQUIRE(tf.get_state() == full);

    // A non-variational integrator.
    taylor_adaptive_batch<double> plain(sys, {0.5, 0.6, 0.7, -0.1, 0.0, 0.1}, batch, kw::pars = w);
    REQUIRE(!plain.is_variational() && plain.get_n_orig_sv() == 2u && plain.get_vorder() == 0u);
    REQUIRE_THROWS(plain.eval_taylor_map(dx), std::invalid_argument);
    REQUIRE_THROWS((void)plain.get_vslice(0), std::invalid_argument);
}

int main(int argc, char **argv)
{
    const bool gpu = argc > 1 && std::strcmp(argv[1], "gpu") == 0;
    test_symbolic();
    if (gpu) {
        test_integrator();
    }
    if (n_fail != 0) {
        std::printf("%d FAILED\n", n_fail);
        return 1;
    }
    std::printf("ALL PASSED (%s)\n", gpu ? "gpu" : "cpu");
    return 0;
}
