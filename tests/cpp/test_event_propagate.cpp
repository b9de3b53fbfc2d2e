// C++ API tests of the device event propagations (hy_batch_propagate_until_ev() / hy_batch_propagate_grid_ev() under
// taylor_adaptive_batch<double>). Run by tests/test_gpu_event_propagate.py.
//
//   test_event_propagate gpu   -> the device path (no step callback) against the host loop (a step callback that
//                                 returns true), bit for bit, in strict and lazy host_sync, sharded, and through
//                                 ensemble_propagate_until_batch
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

static bool same_bits(const std::vector<double> &a, const std::vector<double> &b)
{
    return a.size() == b.size() && std::memcmp(a.data(), b.data(), sizeof(double) * a.size()) == 0;
}

constexpr std::uint32_t B = 37;

// x' = v, v' = -9.8 sin(x) - p0 v: an nt-event at every zero of x, a terminal event at every zero of v whose callback
// flips p0 and (with stop) stops lane 3 at its third call; lane 2's nt-callback raises at its second call when `raise` is set.
static ta_t make(log_t &log, bool raise, bool stop = true)
{
    auto [x, v] = make_vars("x", "v");
    std::vector<double> st(2u * B), pars(B, 0.);
    for (std::uint32_t i = 0; i < B; ++i) {
        st[i] = 0.05 + 0.013 * i;
        st[B + i] = 0.002 * i - 0.03;
    }
    auto counts = std::make_shared<std::vector<int>>(2u * B, 0);
    nt_event_batch<double> nte(x, [&log, raise, counts](ta_t &, double t, int d_sgn, std::uint32_t i) {
        log.emplace_back(0, i, t, 0., d_sgn);
        if (raise && i == 2u && ++(*counts)[i] == 2) {
            throw std::invalid_argument("lane 2 refuses");
        }
    });
    t_event_batch<double> te(v, kw::callback = [&log, counts, stop](ta_t &ta, int d_sgn, std::uint32_t i) {
        const auto &[hi, lo] = ta.get_dtime();
        log.emplace_back(1, i, hi[i], lo[i], d_sgn);
        ta.get_pars_data()[i] = ta.get_pars()[i] == 0. ? 0.5 : 0.;
        return !(stop && i == 3u && ++(*counts)[B + i] == 3);
    });
    return ta_t{{{x, v}, {v, -9.8 * sin(x) - par[0] * v}}, st, B, kw::pars = pars, kw::t_events = {te},
                kw::nt_events = {nte}};
}

static bool same_results(ta_t &a, ta_t &b)
{
    bool ok = same_bits(a.get_state(), b.get_state()) && same_bits(a.get_dtime().first, b.get_dtime().first)
              && same_bits(a.get_dtime().second, b.get_dtime().second) && same_bits(a.get_last_h(), b.get_last_h())
              && same_bits(a.get_tc(), b.get_tc()) && same_bits(a.get_pars(), b.get_pars());
    for (std::uint32_t i = 0; i < B; ++i) {
        ok = ok && a.get_step_res()[i] == b.get_step_res()[i] && a.get_propagate_res()[i] == b.get_propagate_res()[i];
    }
    return ok && a.get_te_cooldowns() == b.get_te_cooldowns();
}

enum class mode { until, for_, grid, cout };

// One call on a fresh integrator, device path (host = false) or host loop; returns the exception message ("" if none).
static std::string run(ta_t &ta, mode md, bool host, std::vector<double> &out)
{
    const step_callback_batch<double> cb = [](ta_t &) { return true; };
    try {
        if (md == mode::until) {
            host ? (void)ta.propagate_until(6., kw::callback = cb) : (void)ta.propagate_until(6.);
        } else if (md == mode::for_) {
            host ? (void)ta.propagate_for(-6., kw::max_delta_t = 0.05, kw::callback = cb)
                 : (void)ta.propagate_for(-6., kw::max_delta_t = 0.05);
        } else if (md == mode::cout) {
            auto res = host ? ta.propagate_until(6., kw::c_output = true, kw::callback = cb)
                            : ta.propagate_until(6., kw::c_output = true);
            if (std::get<0>(res)) {
                out = std::get<0>(res)->get_tcs();
                const auto &tm = std::get<0>(res)->get_times();
                out.insert(out.end(), tm.begin(), tm.end());
            }
        } else {
            std::vector<double> grid;
            for (int k = 0; k < 25; ++k) {
                grid.insert(grid.end(), B, 6. * k / 24.);
            }
            auto res = host ? ta.propagate_grid(grid, kw::callback = cb) : ta.propagate_grid(grid);
            out = std::get<1>(res);
        }
    } catch (const std::exception &e) {
        return e.what();
    }
    return "";
}

static void gpu_tests()
{
    for (const bool lazy : {false, true}) {
        for (const bool raise : {false, true}) {
            for (const auto md : {mode::until, mode::for_, mode::grid, mode::cout}) {
                log_t ld, lh;
                auto d = make(ld, raise), h = make(lh, raise);
                if (lazy) {
                    d.set_host_sync(host_sync::lazy);
                    h.set_host_sync(host_sync::lazy);
                }
                std::vector<double> od, oh;
                const auto ed = run(d, md, false, od), eh = run(h, md, true, oh);
                REQUIRE(ed == eh);
                REQUIRE(raise == !ed.empty());
                REQUIRE(ld == lh);
                REQUIRE(!ld.empty());
                REQUIRE(same_bits(od, oh));
                REQUIRE(same_results(d, h));
                REQUIRE(d.get_host_sync() == (lazy ? host_sync::lazy : host_sync::strict));
            }
        }
    }

    // Sharded over the same device three times: the same bits as one device.
    {
        log_t l1, l3;
        auto t1 = make(l1, false), t3 = make(l3, false);
        t3.set_devices({0, 0, 0});
        t1.propagate_until(6.);
        t3.propagate_until(6.);
        REQUIRE(l1 == l3);
        REQUIRE(same_results(t1, t3));
    }

    // ensemble_propagate_until_batch with events: every member takes the device path, the same bits as the host loop.
    {
        log_t l0;
        auto ta = make(l0, false, false);
        const auto gen = [](ta_t t, std::size_t i) {
            for (std::uint32_t l = 0; l < t.get_batch_size(); ++l) {
                t.get_state_data()[l] += 0.01 * static_cast<double>(i);
            }
            return t;
        };
        auto ens = ensemble_propagate_until_batch(ta, 4., 3, gen);
        for (std::size_t i = 0; i < 3; ++i) {
            auto tl = gen(ta, i);
            tl.propagate_until(4., kw::callback = [](ta_t &) { return true; });
            REQUIRE(same_bits(std::get<0>(ens[i]).get_state(), tl.get_state()));
            REQUIRE(std::get<0>(ens[i]).get_propagate_res() == tl.get_propagate_res());
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
