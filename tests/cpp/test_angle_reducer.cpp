// C++ API tests of callback::angle_reducer. Run by tests/test_gpu_angle_reducer.py.
//
//   test_angle_reducer cpu   -> construction errors (no CUDA device needed)
//   test_angle_reducer gpu   -> the device path against the host loop (the reducer wrapped in a lambda), bit for bit
#include <cmath>
#include <cstdio>
#include <cstdint>
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
constexpr double two_pi = 6.283185307179586;

static bool same_bits(const std::vector<double> &a, const std::vector<double> &b)
{
    return a.size() == b.size() && std::memcmp(a.data(), b.data(), sizeof(double) * a.size()) == 0;
}

static std::uint64_t launches(taylor_adaptive_batch<double> &ta)
{
    std::uint64_t n = 0;
    hy_batch_launch_count(ta.get_device_batch(), &n);
    return n;
}

static void cpu_tests()
{
    auto [x, v] = make_vars("x", "v");
    REQUIRE_THROWS(callback::angle_reducer(std::vector<expression>{}), std::invalid_argument);
    REQUIRE_THROWS(callback::angle_reducer({x + v}), std::invalid_argument);
    REQUIRE_THROWS(callback::angle_reducer({par[0]}), std::invalid_argument);
    REQUIRE(callback::angle_reducer({x, v, x}).get_vars().size() == 2u);
}

static void gpu_tests()
{
    auto [x, v] = make_vars("x", "v");
    const sys_t sys{prime(x) = v, prime(v) = -9.8 * sin(x)};
    // Rotating pendulum above the separatrix: the angle grows without bound.
    const std::uint32_t B = 5;
    std::vector<double> st{0.1, -0.3, 2., 5., -4., 7., -6.5, 8., 9., -7.5};
    const callback::angle_reducer ar({x});

    for (const int tape : {0, 1, 4}) {
        for (const double tf : {4., -4.}) {
            auto run = [&](bool device, std::size_t max_steps) {
                taylor_adaptive_batch<double> ta{sys, st, B};
                ta.set_kernel(tape);
                const auto l0 = launches(ta);
                step_callback_batch<double> cb = ar;
                if (!device) {
                    cb = [ar](taylor_adaptive_batch<double> &t) { return ar(t); };
                }
                auto res = ta.propagate_until(tf, kw::callback = cb, kw::write_tc = true, kw::max_steps = max_steps);
                REQUIRE(std::get<1>(res).target<callback::angle_reducer>() != nullptr || !device);
                return std::tuple{ta, launches(ta) - l0};
            };
            for (const std::size_t ms : {std::size_t(0), std::size_t(7)}) {
                auto [td, ld] = run(true, ms);
                auto [th, lh] = run(false, ms);
                REQUIRE(same_bits(td.get_state(), th.get_state()));
                REQUIRE(same_bits(td.get_time(), th.get_time()));
                REQUIRE(same_bits(td.get_last_h(), th.get_last_h()));
                REQUIRE(same_bits(td.get_tc(), th.get_tc()));
                REQUIRE(td.get_propagate_res() == th.get_propagate_res());
                std::size_t steps = 0;
                for (const auto &r : th.get_propagate_res()) {
                    steps = std::max(steps, std::get<3>(r));
                }
                REQUIRE(ld < 16u);
                REQUIRE(lh >= steps);
                for (std::uint32_t i = 0; i < B; ++i) {
                    const double a = td.get_state()[i];
                    REQUIRE(a >= 0. && a < two_pi);
                }
            }
        }
    }

    // An unknown variable: invalid_argument before any step.
    {
        taylor_adaptive_batch<double> ta{sys, st, B};
        auto [z] = make_vars("z");
        REQUIRE_THROWS(ta.propagate_until(1., kw::callback = step_callback_batch<double>(callback::angle_reducer({z}))),
                       std::invalid_argument);
        REQUIRE(ta.get_time()[0] == 0.);
    }

    // ensemble_propagate_until_batch takes the reducer through kw::callback.
    {
        taylor_adaptive_batch<double> ta{sys, st, B};
        const auto gen = [](taylor_adaptive_batch<double> t, std::size_t i) {
            for (std::uint32_t l = 0; l < t.get_batch_size(); ++l) {
                t.get_state_data()[t.get_batch_size() + l] += 0.25 * static_cast<double>(i);
            }
            return t;
        };
        const auto ens = ensemble_propagate_until_batch(ta, 3., 3, gen,
                                                        kw::callback = step_callback_batch<double>(ar));
        for (std::size_t i = 0; i < 3; ++i) {
            auto tl = gen(ta, i);
            const auto h = [ar](taylor_adaptive_batch<double> &t) { return ar(t); };
            tl.propagate_until(3., kw::callback = step_callback_batch<double>(h));
            REQUIRE(same_bits(std::get<0>(ens[i]).get_state(), tl.get_state()));
        }
    }

    // Sharded over the same device three times: the device path on every shard, same bits as one device.
    {
        std::vector<double> st2(2u * 7u);
        for (std::size_t i = 0; i < 7u; ++i) {
            st2[i] = 0.3 * static_cast<double>(i);
            st2[7u + i] = 6.5 + 0.5 * static_cast<double>(i);
        }
        taylor_adaptive_batch<double> t1{sys, st2, 7u};
        taylor_adaptive_batch<double> t3{sys, st2, 7u, kw::devices = std::vector<int>{0, 0, 0}};
        t1.propagate_until(5., kw::callback = step_callback_batch<double>(ar));
        t3.propagate_until(5., kw::callback = step_callback_batch<double>(ar));
        REQUIRE(same_bits(t1.get_state(), t3.get_state()));
        REQUIRE(same_bits(t1.get_time(), t3.get_time()));
    }
}

int main(int argc, char **argv)
{
    const std::string mode = argc > 1 ? argv[1] : "cpu";
    try {
        cpu_tests();
        if (mode == "gpu") {
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
    std::printf("ALL PASSED (%s)\n", mode.c_str());
    return 0;
}
