// heyoka_b200 — taylor_adaptive_batch<double>: the reference's batch integrator class, backed by the H100
// kernels through the C ABI (include/heyoka_b200.h).
//
// Mirrors include/heyoka/taylor.hpp:780-1121 (bluescarni/heyoka @ 9c91f71) for T = double: same constructor
// (system, state, batch size, kw::time / tol / high_accuracy / compact_mode / pars), same getters, step() /
// step_backward() / step(max_delta_ts), propagate_for() / propagate_until() with kw::max_steps / max_delta_t /
// callback / write_tc, get_step_res() / get_propagate_res(), update_d_output(), and ensemble_propagate_*_batch()
// incl. the grid variant (include/heyoka/ensemble_propagate.hpp:220-269). Errors are the reference's exceptions with the reference's
// messages (std::invalid_argument, not_implemented_error); numerical failure is taylor_outcome::err_nf_state.
//
// Ownership / raw-pointer contract (include/heyoka/taylor.hpp:974-977): the integrator owns host std::vector
// mirrors of state, pars and time that the user may modify through get_state_data() / get_pars_data() between
// calls; they are uploaded at every step()/propagate_*() entry and refreshed on exit. The device-resident
// batch (hy_batch) is shared between copies only in its program: a copy gets its own device buffers.
//
// Event detection (kw::t_events / kw::nt_events with t_event_batch<double> / nt_event_batch<double>,
// include/heyoka/events.hpp): the jet of the event equations, the root finding and the cooldown bookkeeping run on the
// device (include/heyoka_b200.h section E), the callbacks on the host, in the reference's order.
//
// Variational systems (var_ode_sys, order 1; include/heyoka_b200/var_ode_sys.hpp): the augmented system is an
// ordinary ODE system for the kernels; the Taylor map x + Phi dx is evaluated on the device (eval_taylor_map()).
//
// Not supported (see DESIGN.md): variational orders > 1, serialisation. kw::compact_mode, kw::parallel_mode,
// kw::parjit and the llvm_state options are accepted and ignored (there is no JIT).
#ifndef HEYOKA_B200_TAYLOR_HPP
#define HEYOKA_B200_TAYLOR_HPP

#include <cstddef>
#include <cstdint>
#include <functional>
#include <memory>
#include <optional>
#include <stdexcept>
#include <tuple>
#include <type_traits>
#include <utility>
#include <vector>

#include <heyoka_b200.h>
#include <heyoka_b200/exceptions.hpp>
#include <heyoka_b200/expression.hpp>
#include <heyoka_b200/kw.hpp>
#include <heyoka_b200/taylor_decompose.hpp>
#include <heyoka_b200/var_ode_sys.hpp>

namespace heyoka_b200
{

// include/heyoka/taylor.hpp:142-155.
enum class taylor_outcome : std::int64_t {
    success = HY_OUTCOME_SUCCESS,
    step_limit = HY_OUTCOME_STEP_LIMIT,
    time_limit = HY_OUTCOME_TIME_LIMIT,
    err_nf_state = HY_OUTCOME_ERR_NF_STATE,
    cb_stop = HY_OUTCOME_CB_STOP
};

template <typename T>
class taylor_adaptive_batch;

// continuous_output_batch<T> (include/heyoka/continuous_output.hpp:157-237): the result of
// propagate_*(kw::c_output = true). Device-resident (hy_cout); copies share the device data.
template <typename T>
class continuous_output_batch;

template <>
class continuous_output_batch<double>
{
    std::shared_ptr<hy_cout> m_h;
    std::uint32_t m_batch_size = 0, m_dim = 0, m_order = 0;
    std::vector<double> m_output;
    mutable std::vector<double> m_times_hi, m_tcs; // host copies, fetched on first use (get_times() / get_tcs())

    void check_valid() const;

public:
    continuous_output_batch() = default;
    continuous_output_batch(hy_cout *, std::uint32_t batch_size, std::uint32_t dim, std::uint32_t order);

    // State at one time per lane (batch_size values) / at the same time for every lane, [dim][batch].
    const std::vector<double> &operator()(const double *tm);
    const std::vector<double> &operator()(const std::vector<double> &tm);
    const std::vector<double> &operator()(double tm);
    [[nodiscard]] const std::vector<double> &get_output() const
    {
        return m_output;
    }
    [[nodiscard]] std::pair<std::vector<double>, std::vector<double>> get_bounds() const;
    [[nodiscard]] std::size_t get_n_steps() const;
    [[nodiscard]] std::uint32_t get_batch_size() const
    {
        return m_batch_size;
    }
    // The recorded data (include/heyoka/continuous_output.hpp:198-199), copied from the device on first use:
    // times[(n_steps + 2) * batch] (row 0 = starting times, last row = the +-infinity padding),
    // tcs[n_steps][dim][order + 1][batch].
    [[nodiscard]] const std::vector<double> &get_times() const;
    [[nodiscard]] const std::vector<double> &get_tcs() const;
};

// Host <-> device synchronisation of the integrator's host mirrors (extension; default strict).
//   strict  the reference's raw-pointer contract (include/heyoka/taylor.hpp:974-977): whatever the user wrote through
//           get_state_data() / get_pars_data() / references obtained earlier is picked up at the entry of every call,
//           and every mirror is up to date at its exit: state, parameters and times are uploaded and downloaded on
//           every step() / propagate_*() (from / to page-locked memory: the storage of the std::vectors is pinned).
//   lazy    an array is uploaded only after a call that lets the user write it (the non-const get_state_data() /
//           get_pars_data(), set_time() / set_dtime()) - call the getter again before writing again - and a mirror is
//           refreshed from the device when a getter asks for it (references obtained BEFORE a step are not refreshed
//           by the step: call the getter again). Sequences of steps / propagations then move no state over PCIe.
//           Integrators with events, step callbacks and propagate_grid() always run strict.
enum class host_sync { strict, lazy };

// ---- events (include/heyoka/events.hpp) ----
enum class event_direction { negative = -1, any = 0, positive = 1 };

template <typename T>
class t_event_batch;
template <typename T>
class nt_event_batch;

// Terminal event (include/heyoka/events.hpp:52-118, src/t_event.cpp): callback(ta, d_sgn, batch_idx) -> true if the
// integration may continue; kw::cooldown < 0 (default) = automatic; kw::direction.
template <>
class t_event_batch<double>
{
public:
    using callback_t = std::function<bool(taylor_adaptive_batch<double> &, int, std::uint32_t)>;

private:
    expression eq;
    callback_t callback;
    double cooldown = -1.;
    event_direction dir = event_direction::any;

    void finalise_ctor(callback_t, double, event_direction);

public:
    t_event_batch();
    template <typename... KwArgs>
    explicit t_event_batch(expression e, const KwArgs &...kw_args) : eq(std::move(e))
    {
        static_assert(kw::allowed_tags<kw::callback_tag, kw::cooldown_tag, kw::direction_tag>::template all<KwArgs...>(),
                      "Invalid named argument(s) in the construction of a terminal event");
        callback_t cb;
        double cd = -1.;
        event_direction d = event_direction::any;
        kw::visit(kw::callback, [&cb](const auto &v) { cb = v; }, kw_args...);
        kw::visit(kw::cooldown, [&cd](const auto &v) { cd = static_cast<double>(v); }, kw_args...);
        kw::visit(kw::direction, [&d](const auto &v) { d = v; }, kw_args...);
        finalise_ctor(std::move(cb), cd, d);
    }
    [[nodiscard]] const expression &get_expression() const
    {
        return eq;
    }
    [[nodiscard]] const callback_t &get_callback() const
    {
        return callback;
    }
    [[nodiscard]] callback_t &get_callback()
    {
        return callback;
    }
    [[nodiscard]] event_direction get_direction() const
    {
        return dir;
    }
    [[nodiscard]] double get_cooldown() const
    {
        return cooldown;
    }
};

// Non-terminal event (include/heyoka/events.hpp:142-196, src/nt_event.cpp): callback(ta, t, d_sgn, batch_idx).
template <>
class nt_event_batch<double>
{
public:
    using callback_t = std::function<void(taylor_adaptive_batch<double> &, double, int, std::uint32_t)>;

private:
    expression eq;
    callback_t callback;
    event_direction dir = event_direction::any;

    void finalise_ctor(event_direction);

public:
    nt_event_batch();
    template <typename... KwArgs>
    explicit nt_event_batch(expression e, callback_t cb, const KwArgs &...kw_args)
        : eq(std::move(e)), callback(std::move(cb))
    {
        static_assert(kw::allowed_tags<kw::direction_tag>::template all<KwArgs...>(),
                      "Invalid named argument(s) in the construction of a non-terminal event");
        event_direction d = event_direction::any;
        kw::visit(kw::direction, [&d](const auto &v) { d = v; }, kw_args...);
        finalise_ctor(d);
    }
    [[nodiscard]] const expression &get_expression() const
    {
        return eq;
    }
    [[nodiscard]] const callback_t &get_callback() const
    {
        return callback;
    }
    [[nodiscard]] callback_t &get_callback()
    {
        return callback;
    }
    [[nodiscard]] event_direction get_direction() const
    {
        return dir;
    }
};

// include/heyoka/step_callback.hpp:57-139 reduced to the call operator: bool(taylor_adaptive_batch<T> &).
template <typename T>
using step_callback_batch = std::function<bool(taylor_adaptive_batch<T> &)>;

template <>
class taylor_adaptive_batch<double>
{
public:
    using value_type = double;
    using t_event_t = t_event_batch<double>;
    using nt_event_t = nt_event_batch<double>;

private:
    struct impl;
    std::unique_ptr<impl> m_impl;

    struct ctor_opts {
        std::vector<double> time;
        bool time_is_scalar = true;
        double time_scalar = 0.;
        std::optional<double> tol;
        bool high_accuracy = false;
        bool compact_mode = false;
        std::vector<double> pars;
        std::vector<t_event_t> tes;
        std::vector<nt_event_t> ntes;
        int device = -1;
        std::vector<int> devices; // non-empty: the batch is sharded over these GPUs
    };
    struct prop_opts {
        std::size_t max_steps = 0;
        std::vector<double> max_delta_t; // empty = +inf
        step_callback_batch<double> cb;
        bool write_tc = false;
        bool c_output = false;
    };

    void finalise_ctor(std::vector<std::pair<expression, expression>>, std::vector<double>, std::uint32_t, ctor_opts);
    void finalise_ctor(const var_ode_sys &, std::vector<double>, std::uint32_t, ctor_opts);
    void step_impl(const std::vector<double> *, bool backward, bool wtc);
    void run_event_callbacks();
    void call_event_callbacks(const hy_event_rec *, std::size_t, const std::function<double(std::size_t)> &,
                              const std::function<void(std::size_t, bool)> &);
    // The hy_event_callback of the device event propagations; user: a device_ev_hook (taylor_adaptive_batch.cpp).
    static int device_event_callbacks(void *user, const hy_event_rec *, const double *t_hi, const double *t_lo,
                                      std::uint32_t n_rec, unsigned char *cont);
    void end_device_event_call(bool ok);
    std::tuple<std::optional<continuous_output_batch<double>>, step_callback_batch<double>>
    propagate_until_impl(const std::vector<double> &hi, const std::vector<double> &lo, prop_opts);
    std::tuple<step_callback_batch<double>, std::vector<double>> propagate_grid_impl(const std::vector<double> &,
                                                                                     prop_opts);
    std::tuple<step_callback_batch<double>, std::vector<double>> propagate_grid_events(const std::vector<double> &,
                                                                                       prop_opts);

    template <typename... KwArgs>
    static ctor_opts parse_ctor(const KwArgs &...kw_args)
    {
        static_assert(kw::allowed_tags<kw::time_tag, kw::tol_tag, kw::high_accuracy_tag, kw::compact_mode_tag,
                                       kw::pars_tag, kw::parallel_mode_tag, kw::parjit_tag, kw::t_events_tag,
                                       kw::nt_events_tag, kw::opt_level_tag, kw::fast_math_tag, kw::force_avx512_tag,
                                       kw::slp_vectorize_tag, kw::mname_tag, kw::code_model_tag,
                                       kw::device_tag, kw::devices_tag>::template all<KwArgs...>(),
                      "Invalid named argument(s) in the construction of a taylor_adaptive_batch");
        ctor_opts o;
        kw::visit(
            kw::time,
            [&o](const auto &v) {
                if constexpr (std::is_arithmetic_v<std::decay_t<decltype(v)>>) {
                    o.time_scalar = static_cast<double>(v);
                } else {
                    o.time_is_scalar = false;
                    o.time.assign(std::begin(v), std::end(v));
                }
            },
            kw_args...);
        kw::visit(kw::tol, [&o](const auto &v) { o.tol = static_cast<double>(v); }, kw_args...);
        kw::visit(kw::high_accuracy, [&o](const auto &v) { o.high_accuracy = static_cast<bool>(v); }, kw_args...);
        kw::visit(kw::compact_mode, [&o](const auto &v) { o.compact_mode = static_cast<bool>(v); }, kw_args...);
        kw::visit(kw::pars, [&o](const auto &v) { o.pars.assign(std::begin(v), std::end(v)); }, kw_args...);
        kw::visit(kw::device, [&o](const auto &v) { o.device = static_cast<int>(v); }, kw_args...);
        kw::visit(kw::devices, [&o](const auto &v) { o.devices.assign(std::begin(v), std::end(v)); }, kw_args...);
        kw::visit(kw::t_events, [&o](const auto &v) { o.tes.assign(std::begin(v), std::end(v)); }, kw_args...);
        kw::visit(kw::nt_events, [&o](const auto &v) { o.ntes.assign(std::begin(v), std::end(v)); }, kw_args...);
        return o;
    }

    template <typename... KwArgs>
    prop_opts parse_prop(const KwArgs &...kw_args) const
    {
        static_assert(kw::allowed_tags<kw::max_steps_tag, kw::max_delta_t_tag, kw::callback_tag, kw::write_tc_tag,
                                       kw::c_output_tag>::template all<KwArgs...>(),
                      "Invalid named argument(s) in a propagate_*() call");
        prop_opts o;
        kw::visit(kw::max_steps, [&o](const auto &v) { o.max_steps = static_cast<std::size_t>(v); }, kw_args...);
        kw::visit(
            kw::max_delta_t,
            [&o, this](const auto &v) {
                if constexpr (std::is_arithmetic_v<std::decay_t<decltype(v)>>) {
                    o.max_delta_t.assign(get_batch_size(), static_cast<double>(v));
                } else {
                    o.max_delta_t.assign(std::begin(v), std::end(v));
                    if (o.max_delta_t.empty()) {
                        // An empty vector means "no limit" (include/heyoka/taylor.hpp:733-776).
                        return;
                    }
                    check_max_delta_t_size(o.max_delta_t.size());
                }
            },
            kw_args...);
        kw::visit(kw::callback, [&o](const auto &v) { o.cb = v; }, kw_args...);
        kw::visit(kw::write_tc, [&o](const auto &v) { o.write_tc = static_cast<bool>(v); }, kw_args...);
        kw::visit(kw::c_output, [&o](const auto &v) { o.c_output = static_cast<bool>(v); }, kw_args...);
        return o;
    }
    void check_max_delta_t_size(std::size_t) const;

public:
    taylor_adaptive_batch();
    template <typename... KwArgs>
    explicit taylor_adaptive_batch(std::vector<std::pair<expression, expression>> sys, std::vector<double> state,
                                   std::uint32_t batch_size, const KwArgs &...kw_args)
        : taylor_adaptive_batch()
    {
        finalise_ctor(std::move(sys), std::move(state), batch_size, parse_ctor(kw_args...));
    }
    // Without initial conditions: a zeroed state vector (include/heyoka/taylor.hpp:914-921). Taken only when everything
    // after the batch size is a named argument, like the reference's igor::validate constraint, so that
    // {sys, {0.}, 1u} keeps meaning (state, batch size).
    template <typename... KwArgs,
              std::enable_if_t<(kw::detail::is_tagged<std::decay_t<KwArgs>>::value && ... && true), int> = 0>
    explicit taylor_adaptive_batch(std::vector<std::pair<expression, expression>> sys, std::uint32_t batch_size,
                                   const KwArgs &...kw_args)
        : taylor_adaptive_batch(std::move(sys), std::vector<double>{}, batch_size, kw_args...)
    {
    }
    // A variational system, with the same named arguments. A state of n_orig_sv rows (or an empty one: zeros) gets
    // its variational rows filled per lane: the column of an argument that is the state variable x_k holds 1 in row k
    // and 0 elsewhere (the identity block of the STM), the column of a parameter holds 0. A full-size state
    // (get_dim() rows) is taken as given. Later writes through get_state_data() do not reset the variational rows.
    template <typename... KwArgs>
    explicit taylor_adaptive_batch(const var_ode_sys &vsys, std::vector<double> state, std::uint32_t batch_size,
                                   const KwArgs &...kw_args)
        : taylor_adaptive_batch()
    {
        finalise_ctor(vsys, std::move(state), batch_size, parse_ctor(kw_args...));
    }
    taylor_adaptive_batch(const taylor_adaptive_batch &);
    taylor_adaptive_batch(taylor_adaptive_batch &&) noexcept;
    taylor_adaptive_batch &operator=(const taylor_adaptive_batch &);
    taylor_adaptive_batch &operator=(taylor_adaptive_batch &&) noexcept;
    ~taylor_adaptive_batch();

    [[nodiscard]] const taylor_dc_t &get_decomposition() const;
    [[nodiscard]] std::uint32_t get_batch_size() const;
    [[nodiscard]] std::uint32_t get_order() const;
    [[nodiscard]] double get_tol() const;
    [[nodiscard]] bool get_high_accuracy() const;
    [[nodiscard]] bool get_compact_mode() const;
    [[nodiscard]] std::uint32_t get_dim() const;
    // Variational integrators (constructed from a var_ode_sys). For the others: is_variational() == false,
    // get_n_orig_sv() == get_dim(), get_vorder() == 0, no arguments, and the members below that need the variational
    // structure throw std::invalid_argument.
    [[nodiscard]] bool is_variational() const noexcept;
    [[nodiscard]] std::uint32_t get_n_orig_sv() const noexcept;
    // The system integrated: for a variational integrator, the augmented system.
    [[nodiscard]] const std::vector<std::pair<expression, expression>> &get_sys() const noexcept;
    [[nodiscard]] std::uint32_t get_vorder() const noexcept;
    [[nodiscard]] const std::vector<expression> &get_vargs() const noexcept;
    // Rows [first, second) of the state holding the derivatives of the given order (0: the original state
    // variables), of all components / of one component.
    [[nodiscard]] std::pair<std::uint32_t, std::uint32_t> get_vslice(std::uint32_t order) const;
    [[nodiscard]] std::pair<std::uint32_t, std::uint32_t> get_vslice(std::uint32_t component, std::uint32_t order) const;
    // Dense multi-index of state row i: [component, n_0, ..., n_{m-1}] with n_j the order of differentiation with
    // respect to argument j (all zeros for the original state variables).
    [[nodiscard]] std::vector<std::uint32_t> get_mindex(std::uint32_t i) const;
    // Taylor map x + Phi dx of the current state, evaluated on the device: dx[j * batch + lane] for the m arguments;
    // returns get_tstate(), [n_orig_sv][batch].
    const std::vector<double> &eval_taylor_map(const std::vector<double> &dx);
    [[nodiscard]] const std::vector<double> &get_tstate() const noexcept;

    [[nodiscard]] const std::vector<double> &get_time() const;
    [[nodiscard]] const double *get_time_data() const;
    void set_time(const std::vector<double> &);
    void set_time(double);
    [[nodiscard]] std::pair<const std::vector<double> &, const std::vector<double> &> get_dtime() const;
    [[nodiscard]] std::pair<const double *, const double *> get_dtime_data() const;
    void set_dtime(const std::vector<double> &, const std::vector<double> &);
    void set_dtime(double, double);

    [[nodiscard]] const std::vector<double> &get_state() const;
    [[nodiscard]] const double *get_state_data() const;
    [[nodiscard]] double *get_state_data();
    [[nodiscard]] const std::vector<double> &get_pars() const;
    [[nodiscard]] const double *get_pars_data() const;
    [[nodiscard]] double *get_pars_data();
    // get_state_range() / get_pars_range() (src/taylor_adaptive_batch.cpp:2142-2175): the reference returns
    // std::ranges::subrange<std::vector<T>::iterator> (C++20); this header is C++17, so a minimal range with the same
    // begin() / end() / size() / operator[] stands in. Writable like the non-const get_*_data().
    struct range_t {
        std::vector<double>::iterator first, last;
        [[nodiscard]] std::vector<double>::iterator begin() const
        {
            return first;
        }
        [[nodiscard]] std::vector<double>::iterator end() const
        {
            return last;
        }
        [[nodiscard]] std::size_t size() const
        {
            return static_cast<std::size_t>(last - first);
        }
        [[nodiscard]] bool empty() const
        {
            return first == last;
        }
        double &operator[](std::size_t i) const
        {
            return first[static_cast<std::ptrdiff_t>(i)];
        }
    };
    [[nodiscard]] range_t get_state_range();
    [[nodiscard]] range_t get_pars_range();

    [[nodiscard]] const std::vector<double> &get_tc() const;
    [[nodiscard]] const std::vector<double> &get_last_h() const;
    [[nodiscard]] const std::vector<double> &get_d_output() const;
    const std::vector<double> &update_d_output(const std::vector<double> &, bool rel_time = false);
    const std::vector<double> &update_d_output(double, bool rel_time = false);
    [[nodiscard]] bool with_events() const;
    [[nodiscard]] const std::vector<t_event_t> &get_t_events() const;
    [[nodiscard]] const std::vector<nt_event_t> &get_nt_events() const;
    // Cooldown state of the terminal events, [batch index][event index]: empty = not in cooldown, else
    // (time spent in cooldown, cooldown) (src/taylor_adaptive_batch.cpp:2212-2219). Read back from the device on request.
    [[nodiscard]] const std::vector<std::vector<std::optional<std::pair<double, double>>>> &get_te_cooldowns() const;
    // Clears the cooldowns of the terminal events, for every batch element / for one
    // (src/taylor_adaptive_batch.cpp:2300-2330).
    void reset_cooldowns();
    void reset_cooldowns(std::uint32_t);

    void step(bool wtc = false);
    void step_backward(bool wtc = false);
    void step(const std::vector<double> &max_delta_ts, bool wtc = false);
    [[nodiscard]] const std::vector<std::tuple<taylor_outcome, double>> &get_step_res() const;

    template <typename... KwArgs>
    std::tuple<std::optional<continuous_output_batch<double>>, step_callback_batch<double>>
    propagate_until(const std::vector<double> &ts, const KwArgs &...kw_args)
    {
        return propagate_until_vec(ts, parse_prop(kw_args...));
    }
    template <typename... KwArgs>
    std::tuple<std::optional<continuous_output_batch<double>>, step_callback_batch<double>>
    propagate_until(double t, const KwArgs &...kw_args)
    {
        return propagate_until_vec(std::vector<double>(get_batch_size(), t), parse_prop(kw_args...));
    }
    template <typename... KwArgs>
    std::tuple<std::optional<continuous_output_batch<double>>, step_callback_batch<double>>
    propagate_for(const std::vector<double> &delta_ts, const KwArgs &...kw_args)
    {
        return propagate_for_vec(delta_ts, parse_prop(kw_args...));
    }
    template <typename... KwArgs>
    std::tuple<std::optional<continuous_output_batch<double>>, step_callback_batch<double>>
    propagate_for(double delta_t, const KwArgs &...kw_args)
    {
        return propagate_for_vec(std::vector<double>(get_batch_size(), delta_t), parse_prop(kw_args...));
    }
    // propagate_grid() (include/heyoka/taylor.hpp, src/taylor_adaptive_batch.cpp:1545-2055): grid[k * batch + lane];
    // returns the callback and the states at the grid points, [n_pts][dim][batch], NaN where not reached.
    // kw::max_steps, kw::max_delta_t, kw::callback (a step callback, like events, runs the reference's loop on the host:
    // one device step per iteration).
    template <typename... KwArgs>
    std::tuple<step_callback_batch<double>, std::vector<double>> propagate_grid(const std::vector<double> &grid,
                                                                                const KwArgs &...kw_args)
    {
        return propagate_grid_impl(grid, parse_prop(kw_args...));
    }
    [[nodiscard]] const std::vector<std::tuple<taylor_outcome, double, double, std::size_t>> &
    get_propagate_res() const;

    // Extension: see host_sync above.
    [[nodiscard]] host_sync get_host_sync() const;
    void set_host_sync(host_sync);

    // Extensions: the device-resident batch behind this integrator, device placement and kernel selection.
    [[nodiscard]] hy_batch *get_device_batch();
    // Moves the integrator to another GPU / shards it over several GPUs (the device buffers are re-created there).
    void set_device(int device);
    void set_devices(const std::vector<int> &devices);
    [[nodiscard]] int get_device() const;
    void set_kernel(int tape_mode, std::uint32_t lanes_per_warp = 0, std::uint32_t lanes_per_thread = 0,
                    std::uint32_t block_threads = 0, std::uint32_t blocks_per_sm = 0);

private:
    std::tuple<std::optional<continuous_output_batch<double>>, step_callback_batch<double>>
    propagate_until_vec(const std::vector<double> &, prop_opts);
    std::tuple<std::optional<continuous_output_batch<double>>, step_callback_batch<double>>
    propagate_for_vec(const std::vector<double> &, prop_opts);
};

// ------------------------------------------------------------------------------------------------
// Ensemble propagation (include/heyoka/ensemble_propagate.hpp:220-269, src/ensemble_propagate.cpp:192-311):
// n_iter independent copies of an integrator, each customised by gen(ta, i), propagated and returned. The
// reference runs the members under TBB; here the members are dealt out round-robin to the visible GPUs and every GPU
// is driven by its own host thread (member i lives on device i mod n_devices), so the members of different devices
// run concurrently. Like in the reference, gen() may be called concurrently and the results do not depend on the
// partitioning (test/ensemble_propagate.cpp:413-431).
// ------------------------------------------------------------------------------------------------
namespace detail
{

// Number of usable CUDA devices (hy_device_count()).
int ensemble_device_count();

// Runs fn(i, device) for i in [0, n_iter), one worker thread per device; rethrows the first exception.
void ensemble_for_each(std::size_t n_iter, const std::function<void(std::size_t, int)> &fn);

} // namespace detail

template <typename... KwArgs>
std::vector<std::tuple<taylor_adaptive_batch<double>, std::optional<continuous_output_batch<double>>,
                       step_callback_batch<double>>>
ensemble_propagate_until_batch(
    const taylor_adaptive_batch<double> &ta, double t, std::size_t n_iter,
    const std::function<taylor_adaptive_batch<double>(taylor_adaptive_batch<double>, std::size_t)> &gen,
    const KwArgs &...kw_args)
{
    using member_t = std::tuple<taylor_adaptive_batch<double>, std::optional<continuous_output_batch<double>>,
                                step_callback_batch<double>>;
    std::vector<std::optional<member_t>> tmp(n_iter);
    detail::ensemble_for_each(n_iter, [&](std::size_t i, int device) {
        auto local_ta = gen(ta, i);
        local_ta.set_device(device);
        auto res = local_ta.propagate_until(t, kw_args...);
        tmp[i].emplace(std::move(local_ta), std::move(std::get<0>(res)), std::move(std::get<1>(res)));
    });
    std::vector<member_t> retval;
    retval.reserve(n_iter);
    for (auto &m : tmp) {
        retval.push_back(std::move(*m));
    }
    return retval;
}

template <typename... KwArgs>
std::vector<std::tuple<taylor_adaptive_batch<double>, std::optional<continuous_output_batch<double>>,
                       step_callback_batch<double>>>
ensemble_propagate_for_batch(
    const taylor_adaptive_batch<double> &ta, double delta_t, std::size_t n_iter,
    const std::function<taylor_adaptive_batch<double>(taylor_adaptive_batch<double>, std::size_t)> &gen,
    const KwArgs &...kw_args)
{
    using member_t = std::tuple<taylor_adaptive_batch<double>, std::optional<continuous_output_batch<double>>,
                                step_callback_batch<double>>;
    std::vector<std::optional<member_t>> tmp(n_iter);
    detail::ensemble_for_each(n_iter, [&](std::size_t i, int device) {
        auto local_ta = gen(ta, i);
        local_ta.set_device(device);
        auto res = local_ta.propagate_for(delta_t, kw_args...);
        tmp[i].emplace(std::move(local_ta), std::move(std::get<0>(res)), std::move(std::get<1>(res)));
    });
    std::vector<member_t> retval;
    retval.reserve(n_iter);
    for (auto &m : tmp) {
        retval.push_back(std::move(*m));
    }
    return retval;
}

// ensemble_propagate_grid_batch() (include/heyoka/ensemble_propagate.hpp:257-269, src/ensemble_propagate.cpp:258-
// 297): the scalar time grid is splatted over the batch, every member runs propagate_grid().
template <typename... KwArgs>
std::vector<std::tuple<taylor_adaptive_batch<double>, step_callback_batch<double>, std::vector<double>>>
ensemble_propagate_grid_batch(
    const taylor_adaptive_batch<double> &ta, const std::vector<double> &grid_, std::size_t n_iter,
    const std::function<taylor_adaptive_batch<double>(taylor_adaptive_batch<double>, std::size_t)> &gen,
    const KwArgs &...kw_args)
{
    const auto batch_size = ta.get_batch_size();
    std::vector<double> grid;
    grid.reserve(grid_.size() * batch_size);
    for (const auto gval : grid_) {
        grid.insert(grid.end(), batch_size, gval);
    }
    using member_t = std::tuple<taylor_adaptive_batch<double>, step_callback_batch<double>, std::vector<double>>;
    std::vector<std::optional<member_t>> tmp(n_iter);
    detail::ensemble_for_each(n_iter, [&](std::size_t i, int device) {
        auto local_ta = gen(ta, i);
        local_ta.set_device(device);
        auto res = local_ta.propagate_grid(grid, kw_args...);
        tmp[i].emplace(std::move(local_ta), std::move(std::get<0>(res)), std::move(std::get<1>(res)));
    });
    std::vector<member_t> retval;
    retval.reserve(n_iter);
    for (auto &m : tmp) {
        retval.push_back(std::move(*m));
    }
    return retval;
}

} // namespace heyoka_b200

#endif
