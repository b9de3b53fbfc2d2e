// C++ API tests of propagate_grid() on a batch sharded over several devices (kw::devices): the grid loop runs on the
// device over every shard and gives the bits of the single-device batch. Run by tests/test_gpu_sharded_grid.py.
//
//   test_sharded_grid gpu   -> a plain grid, events in strict and lazy host_sync, the angle reducer; three shards on
//                              device 0 against device 0 alone
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <string>
#include <tuple>
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

using ta_t = taylor_adaptive_batch<double>;
using log_t = std::vector<std::tuple<int, std::uint32_t, double, double, int>>;

constexpr std::uint32_t B = 37;
const std::vector<int> three{0, 0, 0};

static bool same_bits(const std::vector<double> &a, const std::vector<double> &b)
{
    return a.size() == b.size() && std::memcmp(a.data(), b.data(), sizeof(double) * a.size()) == 0;
}

static bool same_results(ta_t &a, ta_t &b)
{
    return same_bits(a.get_state(), b.get_state()) && same_bits(a.get_dtime().first, b.get_dtime().first)
           && same_bits(a.get_dtime().second, b.get_dtime().second) && same_bits(a.get_last_h(), b.get_last_h())
           && same_bits(a.get_tc(), b.get_tc()) && a.get_propagate_res() == b.get_propagate_res();
}

// n_pts points from the current times over `span`, scaled per lane.
static std::vector<double> make_grid(ta_t &ta, double span, int n_pts)
{
    std::vector<double> grid;
    for (int k = 0; k < n_pts; ++k) {
        for (std::uint32_t i = 0; i < B; ++i) {
            grid.push_back(ta.get_time()[i] + span * k / (n_pts - 1) * (1. + 0.01 * i));
        }
    }
    return grid;
}

// The pendulum x' = v, v' = -9.8 sin(x) - p0 v, rotating (|v| > 2 sqrt(9.8)) in every third lane.
static std::vector<double> pendulum_state()
{
    std::vector<double> st(2u * B);
    for (std::uint32_t i = 0; i < B; ++i) {
        st[i] = 0.05 + 0.13 * i;
        st[B + i] = (i % 3 == 0 ? 7. : 0.5) * (i % 2 == 0 ? 1. : -1.);
    }
    return st;
}

// With events: an nt-event at every zero of x, a terminal event at every zero of v whose callback flips p0.
static ta_t make_ev(log_t &log, const std::vector<int> &devices)
{
    auto [x, v] = make_vars("x", "v");
    nt_event_batch<double> nte(x, [&log](ta_t &, double t, int d_sgn, std::uint32_t i) {
        log.emplace_back(0, i, t, 0., d_sgn);
    });
    t_event_batch<double> te(v, kw::callback = [&log](ta_t &ta, int d_sgn, std::uint32_t i) {
        const auto &[hi, lo] = ta.get_dtime();
        log.emplace_back(1, i, hi[i], lo[i], d_sgn);
        ta.get_pars_data()[i] = ta.get_pars()[i] == 0. ? 0.5 : 0.;
        return true;
    });
    return ta_t{{{x, v}, {v, -9.8 * sin(x) - par[0] * v}}, pendulum_state(), B, kw::pars = std::vector<double>(B, 0.),
                kw::t_events = {te}, kw::nt_events = {nte}, kw::devices = devices};
}

static void gpu_tests()
{
    auto [x, v] = make_vars("x", "v");
    const std::vector<std::pair<expression, expression>> sys{{x, v}, {v, -9.8 * sin(x) - par[0] * v}};
    const std::vector<double> pars(B, 0.05);

    // A plain grid, forward and backward.
    for (const double span : {6., -6.}) {
        ta_t t1{sys, pendulum_state(), B, kw::pars = pars};
        ta_t t3{sys, pendulum_state(), B, kw::pars = pars, kw::devices = three};
        const auto grid = make_grid(t1, span, 25);
        const auto o1 = std::get<1>(t1.propagate_grid(grid)), o3 = std::get<1>(t3.propagate_grid(grid));
        REQUIRE(same_bits(o1, o3));
        REQUIRE(same_results(t1, t3));
        REQUIRE(!std::isnan(o1.back()));
    }

    // Events, strict and lazy host_sync: the same callback log and bits.
    for (const bool lazy : {false, true}) {
        log_t l1, l3;
        auto t1 = make_ev(l1, {}), t3 = make_ev(l3, three);
        if (lazy) {
            t1.set_host_sync(host_sync::lazy);
            t3.set_host_sync(host_sync::lazy);
        }
        const auto grid = make_grid(t1, 6., 25);
        const auto o1 = std::get<1>(t1.propagate_grid(grid)), o3 = std::get<1>(t3.propagate_grid(grid));
        REQUIRE(!l1.empty());
        REQUIRE(l1 == l3);
        REQUIRE(same_bits(o1, o3));
        REQUIRE(same_results(t1, t3));
        REQUIRE(t3.get_host_sync() == (lazy ? host_sync::lazy : host_sync::strict));
    }

    // The angle reducer.
    {
        const callback::angle_reducer ar({x});
        ta_t t1{sys, pendulum_state(), B, kw::pars = pars};
        ta_t t3{sys, pendulum_state(), B, kw::pars = pars, kw::devices = three};
        const auto grid = make_grid(t1, 4., 13);
        auto r1 = t1.propagate_grid(grid, kw::callback = step_callback_batch<double>(ar));
        auto r3 = t3.propagate_grid(grid, kw::callback = step_callback_batch<double>(ar));
        REQUIRE(std::get<0>(r3).target<callback::angle_reducer>() != nullptr);
        REQUIRE(same_bits(std::get<1>(r1), std::get<1>(r3)));
        REQUIRE(same_results(t1, t3));
        for (std::uint32_t i = 0; i < B; ++i) {
            REQUIRE(t3.get_state()[i] >= 0. && t3.get_state()[i] < 6.283185307179586);
        }
    }
}

int main(int argc, char **argv)
{
    const std::string md = argc > 1 ? argv[1] : "cpu";
    try {
        if (md == "gpu") {
            gpu_tests();
        }
    } catch (const std::exception &e) {
        std::printf("exception: %s\n", e.what());
        ++n_fail;
    }
    if (n_fail != 0) {
        std::printf("%d FAILED\n", n_fail);
        return 1;
    }
    std::printf("ALL PASSED (%s)\n", md.c_str());
    return 0;
}
