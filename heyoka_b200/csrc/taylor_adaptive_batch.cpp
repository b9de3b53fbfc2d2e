// taylor_adaptive_batch<double>: host-side mirror of the reference class on top of the C ABI.
// Reference: src/taylor_adaptive_batch.cpp (ctor :78-427, step :1039-1078, propagate :1081-1534,
// dense output :2251-2327, getters), include/heyoka/detail/dfloat.hpp.
#include <heyoka_b200/taylor.hpp>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <exception>
#include <limits>
#include <string>
#include <thread>

#include "capi_common.hpp"
#include "program.hpp"

namespace heyoka_b200
{

namespace
{

// Double-length arithmetic (include/heyoka/detail/dfloat.hpp:104-169). volatile: no contraction / reassociation.
struct dfl {
    double hi, lo;
};
inline dfl eft_knuth(double a, double b)
{
    volatile double x = a + b;
    volatile double z = x - a;
    volatile double y = (a - (x - z)) + (b - z);
    return {x, y};
}
inline dfl eft_dekker(double a, double b)
{
    volatile double x = a + b;
    volatile double y = (a - x) + b;
    return {x, y};
}
inline dfl dfl_add(dfl a, dfl b)
{
    const dfl h = eft_knuth(a.hi, b.hi), l = eft_knuth(a.lo, b.lo);
    dfl uv = eft_dekker(h.hi, h.lo + l.hi);
    uv = eft_dekker(uv.hi, uv.lo + l.lo);
    return uv;
}
inline dfl dfl_sub(dfl a, dfl b)
{
    return dfl_add(a, dfl{-b.hi, -b.lo});
}
inline bool dfl_lt(dfl x, dfl y)
{
    return (x.hi < y.hi) || (x.hi == y.hi && x.lo < y.lo);
}
inline bool dfl_ge0(dfl x)
{
    return (x.hi > 0.) || (x.hi == 0. && x.lo >= 0.);
}

std::string fp_to_string(double x)
{
    char buf[64];
    std::snprintf(buf, sizeof(buf), "%.17g", x);
    return buf;
}

[[noreturn]] void throw_from_status(int st)
{
    const std::string msg = hy_last_error();
    switch (st) {
        case HY_ERR_NOT_IMPLEMENTED:
            throw not_implemented_error(msg);
        case HY_ERR_OVERFLOW:
            throw std::overflow_error(msg);
        case HY_ERR_CUDA:
            throw std::runtime_error(msg);
        default:
            throw std::invalid_argument(msg);
    }
}

inline void check(int st)
{
    if (st != HY_OK) {
        throw_from_status(st);
    }
}

} // namespace

struct taylor_adaptive_batch<double>::impl {
    std::vector<std::pair<expression, expression>> sys;
    taylor_dc_t dc;
    // The lowered program is shared between copies, like the JIT-compiled code of the reference
    // (src/detail/i_data.cpp:335-352); every copy owns its device buffers.
    std::shared_ptr<hy_program> prog;
    hy_batch *batch = nullptr;
    std::uint32_t batch_size = 0, dim = 0, order = 0, n_pars = 0;
    double tol = 0;
    bool high_accuracy = false, compact_mode = false;
    int device = -1;
    std::vector<int> devices; // non-empty: sharded over these GPUs (hy_batch_create_multi())
    int tape_mode = 0;
    std::uint32_t k_lpw = 0, k_lpt = 0, k_threads = 0, k_bpsm = 0;

    std::vector<double> state, pars, time_hi, time_lo, tc, last_h, d_out;
    std::vector<std::tuple<taylor_outcome, double>> step_res;
    std::vector<std::tuple<taylor_outcome, double, double, std::size_t>> prop_res;
    // scratch
    std::vector<std::int64_t> oc;
    std::vector<double> tmp_a, tmp_b;
    std::vector<std::uint64_t> tmp_n;
    bool tc_valid = false; // the device holds the Taylor coefficients mirrored in `tc`
    std::vector<t_event_batch<double>> tes;
    std::vector<nt_event_batch<double>> ntes;
    std::vector<std::vector<std::optional<std::pair<double, double>>>> te_cooldowns; // filled by get_te_cooldowns()
    // Variational integrators (var_ode_sys): order (0 = not variational), arguments, original state variables, and
    // the last Taylor map [n_orig_sv][batch].
    std::uint32_t vorder = 0, n_orig_sv = 0;
    std::vector<expression> vargs;
    std::vector<double> tstate;
    // Host <-> device synchronisation (see host_sync in taylor.hpp). strict: everything is uploaded at the entry of
    // every call and refreshed at its exit (the reference's raw-pointer contract). lazy: an array is uploaded only
    // after the user could have written it (non-const getters, setters), and the mirrors are refreshed when a getter
    // asks for them.
    bool lazy = false;
    bool host_new_state = true, host_new_pars = true, host_new_time = true;
    bool dev_new_state = false, dev_new_time = false, dev_new_tc = false, dev_new_step = false, dev_new_prop = false;
    // The storage of the mirrors is page-locked in place (hy_host_pin()).
    std::vector<void *> pinned;
    void pin(void *ptr, std::size_t bytes)
    {
        if (ptr != nullptr && bytes != 0u && std::find(pinned.begin(), pinned.end(), ptr) == pinned.end()
            && hy_host_pin(ptr, bytes) == HY_OK) {
            pinned.push_back(ptr);
        }
    }
    void pin_mirrors()
    {
        pin(state.data(), state.size() * sizeof(double));
        pin(pars.data(), pars.size() * sizeof(double));
        pin(time_hi.data(), time_hi.size() * sizeof(double));
        pin(time_lo.data(), time_lo.size() * sizeof(double));
        pin(last_h.data(), last_h.size() * sizeof(double));
        pin(d_out.data(), d_out.size() * sizeof(double));
        pin(oc.data(), oc.size() * sizeof(std::int64_t));
        pin(tmp_a.data(), tmp_a.size() * sizeof(double));
        pin(tmp_b.data(), tmp_b.size() * sizeof(double));
        pin(tmp_n.data(), tmp_n.size() * sizeof(std::uint64_t));
    }
    void unpin_all()
    {
        for (void *p : pinned) {
            hy_host_unpin(p);
        }
        pinned.clear();
    }

    impl() = default;
    impl(const impl &o)
        : sys(o.sys), dc(o.dc), prog(o.prog), batch_size(o.batch_size), dim(o.dim), order(o.order), n_pars(o.n_pars),
          tol(o.tol), high_accuracy(o.high_accuracy), compact_mode(o.compact_mode), device(o.device), devices(o.devices),
          tape_mode(o.tape_mode), k_lpw(o.k_lpw), k_lpt(o.k_lpt), k_threads(o.k_threads), k_bpsm(o.k_bpsm),
          state(o.state), pars(o.pars), time_hi(o.time_hi), time_lo(o.time_lo), tc(o.tc), last_h(o.last_h),
          d_out(o.d_out), step_res(o.step_res), prop_res(o.prop_res), oc(o.oc), tmp_a(o.tmp_a), tmp_b(o.tmp_b),
          tmp_n(o.tmp_n), tc_valid(o.tc_valid), tes(o.tes), ntes(o.ntes), vorder(o.vorder), n_orig_sv(o.n_orig_sv),
          vargs(o.vargs), tstate(o.tstate), lazy(o.lazy)
    {
        if (prog) {
            make_batch();
            pin_mirrors();
            if (o.batch != nullptr && tc_valid) {
                // The copy can serve update_d_output() right away (src/detail/i_data.cpp:335-352 copies m_tc).
                check(hy_batch_upload_tc(batch, tc.data()));
            }
            if (o.batch != nullptr) {
                copy_cooldowns(o.batch, batch);
            }
        }
    }
    ~impl()
    {
        unpin_all();
        hy_batch_destroy(batch);
    }
    // The cooldowns of the terminal events travel with copies and device changes (src/detail/event_detection.cpp:1622-1645).
    void copy_cooldowns(hy_batch *from, hy_batch *to) const
    {
        if (tes.empty()) {
            return;
        }
        const std::size_t m = tes.size() * batch_size;
        std::vector<std::uint8_t> act(m);
        std::vector<double> spent(m), cd(m);
        check(hy_batch_get_cooldowns(from, act.data(), spent.data(), cd.data()));
        check(hy_batch_set_cooldowns(to, act.data(), spent.data(), cd.data()));
    }
    void make_batch()
    {
        if (devices.empty()) {
            check(hy_batch_create(prog.get(), batch_size, device, &batch));
        } else {
            check(hy_batch_create_multi(prog.get(), batch_size, devices.data(), static_cast<std::uint32_t>(devices.size()),
                                        &batch));
        }
        if (tape_mode != 0 || k_lpw != 0 || k_lpt != 0 || k_threads != 0 || k_bpsm != 0) {
            check(hy_batch_set_kernel(batch, tape_mode, k_lpw, k_lpt, k_threads, k_bpsm));
        }
        if (!tes.empty() || !ntes.empty()) {
            std::vector<std::int32_t> dirs;
            std::vector<double> cds;
            for (const auto &e : tes) {
                dirs.push_back(static_cast<std::int32_t>(e.get_direction()));
                cds.push_back(e.get_cooldown());
            }
            for (const auto &e : ntes) {
                dirs.push_back(static_cast<std::int32_t>(e.get_direction()));
            }
            check(hy_batch_set_events(batch, static_cast<std::uint32_t>(tes.size()), dirs.data(), cds.data(), tol));
        }
    }
    void push()
    {
        const bool st = !lazy || host_new_state, pr = n_pars != 0u && (!lazy || host_new_pars), tm = !lazy || host_new_time;
        if (st || pr || tm) {
            check(hy_batch_upload(batch, st ? state.data() : nullptr, pr ? pars.data() : nullptr,
                                  tm ? time_hi.data() : nullptr, tm ? time_lo.data() : nullptr));
        }
        host_new_state = host_new_pars = host_new_time = false;
    }
    // The mirrors the user can see, refreshed from the device if it holds something newer.
    void refresh_state()
    {
        if (dev_new_state) {
            check(hy_batch_download(batch, state.data(), nullptr, nullptr, nullptr));
            dev_new_state = false;
        }
    }
    void refresh_time()
    {
        if (dev_new_time) {
            check(hy_batch_download(batch, nullptr, time_hi.data(), time_lo.data(), last_h.data()));
            dev_new_time = false;
        }
    }
    void refresh_tc()
    {
        if (dev_new_tc) {
            pin(tc.data(), tc.size() * sizeof(double));
            check(hy_batch_download_tc(batch, tc.data()));
            dev_new_tc = false;
        }
    }
    void refresh_step_res()
    {
        if (dev_new_step) {
            check(hy_batch_download_step_res(batch, oc.data(), tmp_a.data()));
            for (std::uint32_t i = 0; i < batch_size; ++i) {
                step_res[i] = std::tuple{static_cast<taylor_outcome>(oc[i]), tmp_a[i]};
            }
            dev_new_step = false;
        }
    }
    void refresh_prop_res()
    {
        if (dev_new_prop) {
            check(hy_batch_download_prop_res(batch, oc.data(), tmp_a.data(), tmp_b.data(), tmp_n.data()));
            for (std::uint32_t i = 0; i < batch_size; ++i) {
                prop_res[i] = std::tuple{static_cast<taylor_outcome>(oc[i]), tmp_a[i], tmp_b[i],
                                         static_cast<std::size_t>(tmp_n[i])};
            }
            dev_new_prop = false;
        }
    }
    void refresh_all()
    {
        refresh_state();
        refresh_time();
        refresh_tc();
        refresh_step_res();
        refresh_prop_res();
    }
    // After a device operation.
    void pull(bool wtc)
    {
        dev_new_state = dev_new_time = true;
        if (wtc) {
            dev_new_tc = true;
            tc_valid = true;
        }
        if (!lazy) {
            refresh_state();
            refresh_time();
            refresh_tc();
        }
    }
    void pull_step_res()
    {
        dev_new_step = true;
        if (!lazy) {
            refresh_step_res();
        }
    }
    void pull_prop_res()
    {
        dev_new_prop = true;
        if (!lazy) {
            refresh_prop_res();
        }
    }
};

namespace
{

// The code paths that work on the host mirrors between device calls (callbacks, events, grids) run in strict mode.
struct strict_scope {
    bool *flag, was;
    template <typename Impl>
    explicit strict_scope(Impl &m) : flag(&m.lazy), was(m.lazy)
    {
        m.refresh_all();
        m.lazy = false;
    }
    ~strict_scope()
    {
        *flag = was;
    }
};

} // namespace

taylor_adaptive_batch<double>::taylor_adaptive_batch() : m_impl(std::make_unique<impl>()) {}

taylor_adaptive_batch<double>::taylor_adaptive_batch(const taylor_adaptive_batch &o)
    : m_impl((o.m_impl->refresh_all(), std::make_unique<impl>(*o.m_impl)))
{
}

taylor_adaptive_batch<double>::taylor_adaptive_batch(taylor_adaptive_batch &&) noexcept = default;

taylor_adaptive_batch<double> &taylor_adaptive_batch<double>::operator=(const taylor_adaptive_batch &o)
{
    if (this != &o) {
        *this = taylor_adaptive_batch(o);
    }
    return *this;
}

taylor_adaptive_batch<double> &taylor_adaptive_batch<double>::operator=(taylor_adaptive_batch &&) noexcept = default;

taylor_adaptive_batch<double>::~taylor_adaptive_batch() = default;

// finalise_ctor_impl(), src/taylor_adaptive_batch.cpp:78-427 (validation order and messages).
void taylor_adaptive_batch<double>::finalise_ctor(std::vector<std::pair<expression, expression>> sys,
                                                  std::vector<double> state, std::uint32_t batch_size, ctor_opts o)
{
    auto &m = *m_impl;

    std::vector<expression> ev_ex;
    for (const auto &e : o.tes) {
        ev_ex.push_back(e.get_expression());
    }
    for (const auto &e : o.ntes) {
        ev_ex.push_back(e.get_expression());
    }
    validate_ode_sys(sys, ev_ex);
    m.tes = std::move(o.tes);
    m.ntes = std::move(o.ntes);

    m.batch_size = batch_size;
    m.high_accuracy = o.high_accuracy;
    m.compact_mode = o.compact_mode;
    m.device = o.device;
    m.devices = o.devices;

    if (batch_size == 0u) {
        throw std::invalid_argument("The batch size in an adaptive Taylor integrator cannot be zero");
    }
    if (state.size() % batch_size != 0u) {
        throw std::invalid_argument("Invalid size detected in the initialization of an adaptive Taylor integrator: "
                                    "the state vector has a size of "
                                    + std::to_string(state.size()) + ", which is not a multiple of the batch size ("
                                    + std::to_string(batch_size) + ")");
    }
    if (state.empty()) {
        state.resize(sys.size() * batch_size);
    }
    if (state.size() / batch_size != sys.size()) {
        throw std::invalid_argument("Inconsistent sizes detected in the initialization of an adaptive Taylor "
                                    "integrator: the state vector has a dimension of "
                                    + std::to_string(state.size() / batch_size) + " and a batch size of "
                                    + std::to_string(batch_size) + ", while the number of equations is "
                                    + std::to_string(sys.size()));
    }
    m.state = std::move(state);

    if (o.time_is_scalar) {
        m.time_hi.assign(batch_size, o.time_scalar);
    } else {
        m.time_hi = std::move(o.time);
    }
    if (m.time_hi.size() != batch_size) {
        throw std::invalid_argument("Invalid size detected in the initialization of an adaptive Taylor integrator: "
                                    "the time vector has a size of "
                                    + std::to_string(m.time_hi.size()) + ", which is not equal to the batch size ("
                                    + std::to_string(batch_size) + ")");
    }
    m.time_lo.assign(batch_size, 0.);

    if (o.tol && (!std::isfinite(*o.tol) || *o.tol < 0)) {
        throw std::invalid_argument("The tolerance in an adaptive Taylor integrator must be finite and positive, "
                                    "but it is "
                                    + fp_to_string(*o.tol) + " instead");
    }
    m.tol = (o.tol && *o.tol != 0) ? *o.tol : std::numeric_limits<double>::epsilon();
    m.dim = static_cast<std::uint32_t>(sys.size());

    std::vector<expression> all_rhs;
    for (const auto &p : sys) {
        all_rhs.push_back(p.second);
    }
    // (The parameters of the event equations count: test/taylor_adaptive_batch.cpp:1015-1060.)
    all_rhs.insert(all_rhs.end(), ev_ex.begin(), ev_ex.end());
    m.n_pars = get_param_size(all_rhs);
    const auto pars_req = static_cast<std::size_t>(m.n_pars) * batch_size;
    if (o.pars.empty()) {
        o.pars.resize(pars_req);
    } else if (o.pars.size() != pars_req) {
        throw std::invalid_argument("Invalid number of parameter values passed to the constructor of an adaptive "
                                    "Taylor integrator in batch mode: "
                                    + std::to_string(o.pars.size())
                                    + " parameter value(s) were passed, but the ODE system contains "
                                    + std::to_string(m.n_pars) + " parameter(s) (in batches of "
                                    + std::to_string(batch_size) + ")");
    }
    m.pars = std::move(o.pars);

    m.order = detail::taylor_order_from_tol(m.tol);

    // Decompose, lower, create the device-resident batch (replaces taylor_add_adaptive_step() + JIT).
    auto dc_ev = taylor_decompose_sys(sys, ev_ex);
    m.dc = std::move(dc_ev.first);
    try {
        m.prog = std::make_shared<hy_program>(
            detail::lower_decomposition(m.dc, m.dim, m.n_pars, m.order, m.high_accuracy));
        m.prog->ev_defs = std::move(dc_ev.second);
    } catch (const detail::not_implemented_error &e) {
        throw not_implemented_error(e.what());
    }
    m.sys = std::move(sys);
    m.make_batch();

    // Buffers (src/taylor_adaptive_batch.cpp:361-402).
    const auto n = static_cast<std::size_t>(batch_size);
    m.tc.assign(static_cast<std::size_t>(m.dim) * (m.order + 1u) * n, 0.);
    m.last_h.assign(n, 0.);
    m.d_out.assign(static_cast<std::size_t>(m.dim) * n, 0.);
    m.step_res.assign(n, std::tuple{taylor_outcome::success, 0.});
    m.prop_res.assign(n, std::tuple{taylor_outcome::success, 0., 0., std::size_t(0)});
    m.oc.assign(n, 0);
    m.tmp_a.assign(n, 0.);
    m.tmp_b.assign(n, 0.);
    m.tmp_n.assign(n, 0);
    m.pin_mirrors();

    // Non-finite initial conditions are rejected (src/taylor_adaptive_batch.cpp:404-423).
    for (const auto x : m.state) {
        if (!std::isfinite(x)) {
            throw std::invalid_argument(
                "A non-finite value was detected in the initial state of an adaptive Taylor integrator");
        }
    }
    for (const auto x : m.time_hi) {
        if (!std::isfinite(x)) {
            throw std::invalid_argument(
                "A non-finite initial time was detected in the initialisation of an adaptive Taylor integrator");
        }
    }
}

void taylor_adaptive_batch<double>::finalise_ctor(const var_ode_sys &vsys, std::vector<double> state,
                                                  std::uint32_t batch_size, ctor_opts o)
{
    const auto n_orig = static_cast<std::size_t>(vsys.get_n_orig_sv());
    const auto &vargs = vsys.get_vargs();
    const auto &aug = vsys.get_sys();
    const auto n = static_cast<std::size_t>(batch_size);
    if (batch_size != 0u && (state.empty() || state.size() == n_orig * n)) {
        // The variational rows: per lane, column j of the STM is e_k when argument j is the state variable x_k, 0 when
        // it is a parameter (dx(t0)/dx_k(t0) = e_k, dx(t0)/dp = 0).
        state.resize(aug.size() * n, 0.);
        for (std::size_t i = 0; i < n_orig; ++i) {
            for (std::size_t j = 0; j < vargs.size(); ++j) {
                if (vargs[j] == aug[i].first) {
                    const auto row = n_orig + i * vargs.size() + j;
                    std::fill(state.begin() + static_cast<std::ptrdiff_t>(row * n),
                              state.begin() + static_cast<std::ptrdiff_t>((row + 1u) * n), 1.);
                }
            }
        }
    }
    finalise_ctor(aug, std::move(state), batch_size, std::move(o));
    auto &m = *m_impl;
    m.vorder = vsys.get_order();
    m.n_orig_sv = vsys.get_n_orig_sv();
    m.vargs = vargs;
    m.tstate.assign(n_orig * n, 0.);
}

const taylor_dc_t &taylor_adaptive_batch<double>::get_decomposition() const
{
    return m_impl->dc;
}
std::uint32_t taylor_adaptive_batch<double>::get_batch_size() const
{
    return m_impl->batch_size;
}
std::uint32_t taylor_adaptive_batch<double>::get_order() const
{
    return m_impl->order;
}
double taylor_adaptive_batch<double>::get_tol() const
{
    return m_impl->tol;
}
bool taylor_adaptive_batch<double>::get_high_accuracy() const
{
    return m_impl->high_accuracy;
}
bool taylor_adaptive_batch<double>::get_compact_mode() const
{
    return m_impl->compact_mode;
}
std::uint32_t taylor_adaptive_batch<double>::get_dim() const
{
    return m_impl->dim;
}
bool taylor_adaptive_batch<double>::is_variational() const noexcept
{
    return m_impl->vorder != 0u;
}
std::uint32_t taylor_adaptive_batch<double>::get_n_orig_sv() const noexcept
{
    return m_impl->vorder != 0u ? m_impl->n_orig_sv : m_impl->dim;
}
const std::vector<std::pair<expression, expression>> &taylor_adaptive_batch<double>::get_sys() const noexcept
{
    return m_impl->sys;
}
std::uint32_t taylor_adaptive_batch<double>::get_vorder() const noexcept
{
    return m_impl->vorder;
}
const std::vector<expression> &taylor_adaptive_batch<double>::get_vargs() const noexcept
{
    return m_impl->vargs;
}

namespace
{

void check_variational(std::uint32_t vorder, const char *what)
{
    if (vorder == 0u) {
        throw std::invalid_argument(std::string("The function ") + what
                                    + " can be invoked only on a variational integrator");
    }
}

} // namespace

std::pair<std::uint32_t, std::uint32_t> taylor_adaptive_batch<double>::get_vslice(std::uint32_t order) const
{
    const auto &m = *m_impl;
    check_variational(m.vorder, "get_vslice()");
    if (order > m.vorder) {
        throw std::invalid_argument("Cannot fetch the slice of the derivatives of order " + std::to_string(order)
                                    + " in a variational integrator of order " + std::to_string(m.vorder));
    }
    return order == 0u ? std::pair{0u, m.n_orig_sv} : std::pair{m.n_orig_sv, m.dim};
}

std::pair<std::uint32_t, std::uint32_t> taylor_adaptive_batch<double>::get_vslice(std::uint32_t component,
                                                                                  std::uint32_t order) const
{
    const auto &m = *m_impl;
    const auto all = get_vslice(order);
    if (component >= m.n_orig_sv) {
        throw std::invalid_argument("Cannot fetch the slice of the derivatives of the component "
                                    + std::to_string(component) + " in a variational integrator with "
                                    + std::to_string(m.n_orig_sv) + " original state variables");
    }
    if (order == 0u) {
        return {component, component + 1u};
    }
    const auto n_args = static_cast<std::uint32_t>(m.vargs.size());
    return {all.first + component * n_args, all.first + (component + 1u) * n_args};
}

std::vector<std::uint32_t> taylor_adaptive_batch<double>::get_mindex(std::uint32_t i) const
{
    const auto &m = *m_impl;
    check_variational(m.vorder, "get_mindex()");
    if (i >= m.dim) {
        throw std::invalid_argument("Cannot fetch the multi-index of the state variable " + std::to_string(i)
                                    + " in a variational integrator with " + std::to_string(m.dim)
                                    + " state variables");
    }
    const auto n_args = static_cast<std::uint32_t>(m.vargs.size());
    std::vector<std::uint32_t> ret(1u + n_args, 0u);
    if (i < m.n_orig_sv) {
        ret[0] = i;
    } else {
        ret[0] = (i - m.n_orig_sv) / n_args;
        ret[1u + (i - m.n_orig_sv) % n_args] = 1u;
    }
    return ret;
}

const std::vector<double> &taylor_adaptive_batch<double>::eval_taylor_map(const std::vector<double> &dx)
{
    auto &m = *m_impl;
    check_variational(m.vorder, "eval_taylor_map()");
    const auto n_args = static_cast<std::uint32_t>(m.vargs.size());
    if (dx.size() != static_cast<std::size_t>(n_args) * m.batch_size) {
        throw std::invalid_argument("Invalid number of values passed to eval_taylor_map(): "
                                    + std::to_string(dx.size()) + " values were passed, but "
                                    + std::to_string(static_cast<std::size_t>(n_args) * m.batch_size)
                                    + " are needed (" + std::to_string(n_args) + " arguments in batches of "
                                    + std::to_string(m.batch_size) + ")");
    }
    // The map is evaluated from the state the user sees (the host mirror in strict mode).
    m.push();
    check(hy_batch_eval_taylor_map(m.batch, m.n_orig_sv, n_args, dx.data(), m.tstate.data(), 0));
    return m.tstate;
}

const std::vector<double> &taylor_adaptive_batch<double>::get_tstate() const noexcept
{
    return m_impl->tstate;
}
const std::vector<double> &taylor_adaptive_batch<double>::get_time() const
{
    m_impl->refresh_time();
    return m_impl->time_hi;
}
const double *taylor_adaptive_batch<double>::get_time_data() const
{
    m_impl->refresh_time();
    return m_impl->time_hi.data();
}

// set_time() / set_dtime(): src/taylor_adaptive_batch.cpp:2120-2232.
void taylor_adaptive_batch<double>::set_time(const std::vector<double> &t)
{
    auto &m = *m_impl;
    if (t.size() != m.batch_size) {
        throw std::invalid_argument("Invalid number of new times specified in a Taylor integrator in batch mode: the "
                                    "batch size is "
                                    + std::to_string(m.batch_size) + ", but the number of specified times is "
                                    + std::to_string(t.size()));
    }
    m.refresh_time(); // (last_h travels with the times)
    std::copy(t.begin(), t.end(), m.time_hi.begin());
    std::fill(m.time_lo.begin(), m.time_lo.end(), 0.);
    m.host_new_time = true;
}
void taylor_adaptive_batch<double>::set_time(double t)
{
    m_impl->refresh_time();
    std::fill(m_impl->time_hi.begin(), m_impl->time_hi.end(), t);
    std::fill(m_impl->time_lo.begin(), m_impl->time_lo.end(), 0.);
    m_impl->host_new_time = true;
}
std::pair<const std::vector<double> &, const std::vector<double> &> taylor_adaptive_batch<double>::get_dtime() const
{
    m_impl->refresh_time();
    return {m_impl->time_hi, m_impl->time_lo};
}
std::pair<const double *, const double *> taylor_adaptive_batch<double>::get_dtime_data() const
{
    m_impl->refresh_time();
    return {m_impl->time_hi.data(), m_impl->time_lo.data()};
}
void taylor_adaptive_batch<double>::set_dtime(const std::vector<double> &hi, const std::vector<double> &lo)
{
    auto &m = *m_impl;
    if (hi.size() != m.batch_size || lo.size() != m.batch_size) {
        throw std::invalid_argument("Invalid number of new times specified in a Taylor integrator in batch mode: the "
                                    "batch size is "
                                    + std::to_string(m.batch_size) + ", but the number of specified times is ("
                                    + std::to_string(hi.size()) + ", " + std::to_string(lo.size()) + ")");
    }
    // dtime_checks(), include/heyoka/detail/taylor_common.hpp:231-249: before the times are touched.
    for (std::uint32_t i = 0; i < m.batch_size; ++i) {
        if (!std::isfinite(hi[i]) || !std::isfinite(lo[i])) {
            throw std::invalid_argument("The components of the double-length representation of the time coordinate "
                                        "must both be finite, but they are "
                                        + detail::fmt_double(hi[i]) + " and " + detail::fmt_double(lo[i]) + " instead");
        }
        if (std::abs(hi[i]) < std::abs(lo[i])) {
            throw std::invalid_argument("The first component of the double-length representation of the time "
                                        "coordinate ("
                                        + detail::fmt_double(hi[i])
                                        + ") must not be smaller in magnitude than the second component ("
                                        + detail::fmt_double(lo[i]) + ")");
        }
    }
    m.refresh_time();
    for (std::uint32_t i = 0; i < m.batch_size; ++i) {
        const auto r = eft_dekker(hi[i], lo[i]); // normalise
        m.time_hi[i] = r.hi;
        m.time_lo[i] = r.lo;
    }
    m.host_new_time = true;
}
void taylor_adaptive_batch<double>::set_dtime(double hi, double lo)
{
    set_dtime(std::vector<double>(m_impl->batch_size, hi), std::vector<double>(m_impl->batch_size, lo));
}

const std::vector<double> &taylor_adaptive_batch<double>::get_state() const
{
    m_impl->refresh_state();
    return m_impl->state;
}
const double *taylor_adaptive_batch<double>::get_state_data() const
{
    m_impl->refresh_state();
    return m_impl->state.data();
}
double *taylor_adaptive_batch<double>::get_state_data()
{
    // The caller may write through the pointer: the host copy is the one that counts at the next call.
    m_impl->refresh_state();
    m_impl->host_new_state = true;
    return m_impl->state.data();
}
const std::vector<double> &taylor_adaptive_batch<double>::get_pars() const
{
    return m_impl->pars;
}
const double *taylor_adaptive_batch<double>::get_pars_data() const
{
    return m_impl->pars.data();
}
double *taylor_adaptive_batch<double>::get_pars_data()
{
    m_impl->host_new_pars = true;
    return m_impl->pars.data();
}
taylor_adaptive_batch<double>::range_t taylor_adaptive_batch<double>::get_state_range()
{
    // (Writable, like the non-const get_state_data().)
    m_impl->refresh_state();
    m_impl->host_new_state = true;
    return {m_impl->state.begin(), m_impl->state.end()};
}
taylor_adaptive_batch<double>::range_t taylor_adaptive_batch<double>::get_pars_range()
{
    m_impl->host_new_pars = true;
    return {m_impl->pars.begin(), m_impl->pars.end()};
}
const std::vector<double> &taylor_adaptive_batch<double>::get_tc() const
{
    m_impl->refresh_tc();
    return m_impl->tc;
}
const std::vector<double> &taylor_adaptive_batch<double>::get_last_h() const
{
    m_impl->refresh_time();
    return m_impl->last_h;
}
host_sync taylor_adaptive_batch<double>::get_host_sync() const
{
    return m_impl->lazy ? host_sync::lazy : host_sync::strict;
}
void taylor_adaptive_batch<double>::set_host_sync(host_sync hs)
{
    auto &m = *m_impl;
    m.refresh_all();
    m.lazy = hs == host_sync::lazy;
    // (Coming back to strict mode: everything is uploaded at the next call anyway.)
}
const std::vector<double> &taylor_adaptive_batch<double>::get_d_output() const
{
    return m_impl->d_out;
}
const std::vector<std::tuple<taylor_outcome, double>> &taylor_adaptive_batch<double>::get_step_res() const
{
    m_impl->refresh_step_res();
    return m_impl->step_res;
}
const std::vector<std::tuple<taylor_outcome, double, double, std::size_t>> &
taylor_adaptive_batch<double>::get_propagate_res() const
{
    m_impl->refresh_prop_res();
    return m_impl->prop_res;
}
hy_batch *taylor_adaptive_batch<double>::get_device_batch()
{
    return m_impl->batch;
}
int taylor_adaptive_batch<double>::get_device() const
{
    return m_impl->device;
}
// Re-creates the device-resident batch on another GPU (or sharded over several); the host mirrors are the master
// copy of state / parameters / time, the Taylor coefficients of the last step are restored if they were valid.
void taylor_adaptive_batch<double>::set_devices(const std::vector<int> &devices)
{
    auto &m = *m_impl;
    if (devices == m.devices && (!devices.empty() || m.batch != nullptr)) {
        return;
    }
    if (m.batch != nullptr) {
        m.refresh_all();
    }
    hy_batch *old = m.batch;
    m.batch = nullptr;
    m.devices = devices;
    m.make_batch();
    if (old != nullptr) {
        m.copy_cooldowns(old, m.batch);
    }
    hy_batch_destroy(old);
    m.host_new_state = m.host_new_pars = m.host_new_time = true;
    if (m.tc_valid) {
        check(hy_batch_upload_tc(m.batch, m.tc.data()));
    }
}
void taylor_adaptive_batch<double>::set_device(int device)
{
    auto &m = *m_impl;
    if (m.devices.empty() && (device == m.device || device < 0)) {
        return;
    }
    if (m.batch != nullptr) {
        m.refresh_all();
    }
    hy_batch *old = m.batch;
    m.batch = nullptr;
    m.devices.clear();
    m.device = device;
    m.make_batch();
    if (old != nullptr) {
        m.copy_cooldowns(old, m.batch);
    }
    hy_batch_destroy(old);
    m.host_new_state = m.host_new_pars = m.host_new_time = true;
    if (m.tc_valid) {
        check(hy_batch_upload_tc(m.batch, m.tc.data()));
    }
}

namespace detail
{

int ensemble_device_count()
{
    return hy_device_count();
}

void ensemble_for_each(std::size_t n_iter, const std::function<void(std::size_t, int)> &fn)
{
    const int n_dev = std::max(1, ensemble_device_count());
    const std::size_t n_workers = std::min<std::size_t>(static_cast<std::size_t>(n_dev), n_iter);
    if (n_workers <= 1u) {
        for (std::size_t i = 0; i < n_iter; ++i) {
            fn(i, -1);
        }
        return;
    }
    std::vector<std::exception_ptr> errs(n_workers);
    std::vector<std::thread> thr;
    for (std::size_t w = 0; w < n_workers; ++w) {
        thr.emplace_back([&, w] {
            try {
                for (std::size_t i = w; i < n_iter; i += n_workers) {
                    fn(i, static_cast<int>(w));
                }
            } catch (...) {
                errs[w] = std::current_exception();
            }
        });
    }
    for (auto &t : thr) {
        t.join();
    }
    for (const auto &e : errs) {
        if (e) {
            std::rethrow_exception(e);
        }
    }
}

} // namespace detail

void taylor_adaptive_batch<double>::set_kernel(int tape_mode, std::uint32_t lpw, std::uint32_t lpt,
                                               std::uint32_t threads, std::uint32_t bpsm)
{
    auto &m = *m_impl;
    check(hy_batch_set_kernel(m.batch, tape_mode, lpw, lpt, threads, bpsm));
    m.tape_mode = tape_mode;
    m.k_lpw = lpw;
    m.k_lpt = lpt;
    m.k_threads = threads;
    m.k_bpsm = bpsm;
}

// ---- stepping (src/taylor_adaptive_batch.cpp:1039-1078) ----
void taylor_adaptive_batch<double>::step_impl(const std::vector<double> *max_delta_ts, bool backward, bool wtc)
{
    auto &m = *m_impl;
    const bool ev = with_events();
    std::optional<strict_scope> strict;
    if (ev && m.lazy) {
        strict.emplace(m); // (the callbacks work on the host mirrors)
    }
    m.push();
    check(hy_batch_step(m.batch, max_delta_ts != nullptr ? max_delta_ts->data() : nullptr, 0, backward ? 1 : 0,
                        wtc ? 1 : 0));
    // With events the Taylor coefficients are written unconditionally (src/taylor_adaptive_batch.cpp:776).
    m.pull(wtc || ev);
    m.pull_step_res();
    if (ev) {
        run_event_callbacks();
    }
}

// The callback part of the events branch of step_impl() (src/taylor_adaptive_batch.cpp:803-1033): the detection, the
// propagation and the cooldowns were done on the device by hy_batch_step().
void taylor_adaptive_batch<double>::run_event_callbacks()
{
    auto &m = *m_impl;
    const auto n_ev = hy_batch_n_events(m.batch);
    if (n_ev == 0u) {
        return;
    }
    std::vector<hy_event_rec> evs(n_ev);
    check(hy_batch_get_events(m.batch, evs.data(), n_ev));
    const auto t_hi = m.time_hi, t_lo = m.time_lo;
    std::vector<std::pair<std::uint32_t, std::exception_ptr>> cb_eptrs;
    for (std::size_t k = 0; k < evs.size();) {
        const auto lane = evs[k].lane;
        std::size_t end = k;
        while (end < evs.size() && evs[end].lane == lane) {
            ++end;
        }
        const double h = m.last_h[lane];
        bool nt_cb_exception = false;
        std::size_t j = k;
        for (; j < end && evs[j].terminal == 0; ++j) {
            auto &cb = m.ntes[evs[j].idx].get_callback();
            // new_time - last_h + t in double-length arithmetic (:889).
            const auto tm = dfl_add(dfl_sub(dfl{t_hi[lane], t_lo[lane]}, dfl{h, 0.}), dfl{evs[j].t, 0.}).hi;
            try {
                cb(*this, tm, evs[j].d_sgn, lane);
            } catch (...) {
                cb_eptrs.emplace_back(lane, std::current_exception());
                nt_cb_exception = true;
                break;
            }
        }
        if (!nt_cb_exception) {
            for (; j < end; ++j) {
                if (evs[j].terminal != 0) {
                    auto &te = m.tes[evs[j].idx];
                    bool te_cb_ret = false;
                    bool thrown = false;
                    if (te.get_callback()) {
                        try {
                            te_cb_ret = te.get_callback()(*this, evs[j].d_sgn, lane);
                        } catch (...) {
                            cb_eptrs.emplace_back(lane, std::current_exception());
                            thrown = true;
                        }
                    }
                    if (!thrown) {
                        const auto ev_idx = static_cast<std::int64_t>(evs[j].idx);
                        m.step_res[lane] = std::tuple{taylor_outcome{te_cb_ret ? ev_idx : (-ev_idx - 1)}, h};
                    }
                    break;
                }
            }
        }
        k = end;
    }
    if (!cb_eptrs.empty()) {
        if (cb_eptrs.size() == 1u) {
            std::rethrow_exception(cb_eptrs[0].second);
        }
        std::string exc_msg = "Two or more exceptions were raised during the execution of event callbacks in a "
                              "batch integrator:\n\n";
        for (auto &[i, eptr] : cb_eptrs) {
            exc_msg += "Batch index #" + std::to_string(i) + ":\n";
            try {
                std::rethrow_exception(eptr);
            } catch (const std::exception &ex) {
                exc_msg += std::string("    Exception type: ") + typeid(ex).name() + "\n";
                exc_msg += std::string("    Exception message: ") + ex.what() + "\n";
            } catch (...) {
                exc_msg += "    Exception type: unknown\n    Exception message: unknown\n";
            }
            exc_msg += '\n';
        }
        throw std::runtime_error(exc_msg);
    }
    const auto same = [](double a, double b) { return a == b || (std::isnan(a) && std::isnan(b)); };
    for (std::uint32_t i = 0; i < m.batch_size; ++i) {
        if (!same(m.time_hi[i], t_hi[i]) || !same(m.time_lo[i], t_lo[i])) {
            throw std::runtime_error("The invocation of one or more event callbacks resulted in the alteration of the "
                                     "time coordinate of the integrator at the batch index "
                                     + std::to_string(i) + " - this is not supported");
        }
    }
}

bool taylor_adaptive_batch<double>::with_events() const
{
    return !m_impl->tes.empty() || !m_impl->ntes.empty();
}
// (Both throw on an integrator without events, src/taylor_adaptive_batch.cpp:2202-2229.)
const std::vector<t_event_batch<double>> &taylor_adaptive_batch<double>::get_t_events() const
{
    if (!with_events()) {
        throw std::invalid_argument("No events were defined for this integrator");
    }
    return m_impl->tes;
}
const std::vector<nt_event_batch<double>> &taylor_adaptive_batch<double>::get_nt_events() const
{
    if (!with_events()) {
        throw std::invalid_argument("No events were defined for this integrator");
    }
    return m_impl->ntes;
}
const std::vector<std::vector<std::optional<std::pair<double, double>>>> &
taylor_adaptive_batch<double>::get_te_cooldowns() const
{
    if (!with_events()) {
        throw std::invalid_argument("No events were defined for this integrator");
    }
    auto &m = *m_impl;
    const std::size_t n_te = m.tes.size(), n = m.batch_size;
    // The device keeps the cooldown state as [n_te][batch] arrays (hy_batch_get_cooldowns()).
    std::vector<std::uint8_t> active(n_te * n);
    std::vector<double> spent(n_te * n), cd(n_te * n);
    check(hy_batch_get_cooldowns(m.batch, active.data(), spent.data(), cd.data()));
    m.te_cooldowns.assign(n, std::vector<std::optional<std::pair<double, double>>>(n_te));
    for (std::size_t k = 0; k < n_te; ++k) {
        for (std::size_t i = 0; i < n; ++i) {
            if (active[k * n + i] != 0u) {
                m.te_cooldowns[i][k].emplace(spent[k * n + i], cd[k * n + i]);
            }
        }
    }
    return m.te_cooldowns;
}
void taylor_adaptive_batch<double>::reset_cooldowns()
{
    if (!with_events()) {
        throw std::invalid_argument("No events were defined for this integrator");
    }
    check(hy_batch_reset_cooldowns(m_impl->batch, -1));
}
void taylor_adaptive_batch<double>::reset_cooldowns(std::uint32_t i)
{
    if (!with_events()) {
        throw std::invalid_argument("No events were defined for this integrator");
    }
    check(hy_batch_reset_cooldowns(m_impl->batch, static_cast<std::int64_t>(i)));
}

// ---- events (src/t_event.cpp, src/nt_event.cpp) ----
t_event_batch<double>::t_event_batch() : t_event_batch(expression{}) {}
void t_event_batch<double>::finalise_ctor(callback_t cb, double cd, event_direction d)
{
    callback = std::move(cb);
    if (!std::isfinite(cd)) {
        throw std::invalid_argument("Cannot set a non-finite cooldown value for a terminal event");
    }
    cooldown = cd;
    if (d < event_direction::negative || d > event_direction::positive) {
        throw std::invalid_argument("Invalid value selected for the direction of a terminal event");
    }
    dir = d;
}
nt_event_batch<double>::nt_event_batch()
    : nt_event_batch(expression{}, [](taylor_adaptive_batch<double> &, double, int, std::uint32_t) {})
{
}
void nt_event_batch<double>::finalise_ctor(event_direction d)
{
    if (!callback) {
        throw std::invalid_argument("Cannot construct a non-terminal event with an empty callback");
    }
    if (d < event_direction::negative || d > event_direction::positive) {
        throw std::invalid_argument("Invalid value selected for the direction of a non-terminal event");
    }
    dir = d;
}

void taylor_adaptive_batch<double>::step(bool wtc)
{
    step_impl(nullptr, false, wtc);
}

void taylor_adaptive_batch<double>::step_backward(bool wtc)
{
    step_impl(nullptr, true, wtc);
}

void taylor_adaptive_batch<double>::step(const std::vector<double> &max_delta_ts, bool wtc)
{
    const auto &m = *m_impl;
    if (max_delta_ts.size() != m.batch_size) {
        throw std::invalid_argument("Invalid number of max timesteps specified in a Taylor integrator in batch mode: "
                                    "the batch size is "
                                    + std::to_string(m.batch_size) + ", but the number of specified timesteps is "
                                    + std::to_string(max_delta_ts.size()));
    }
    for (const auto x : max_delta_ts) {
        if (std::isnan(x)) {
            throw std::invalid_argument(
                "Cannot use a nan max_delta_t in the step() function of an adaptive Taylor integrator in batch mode");
        }
    }
    step_impl(&max_delta_ts, false, wtc);
}

void taylor_adaptive_batch<double>::check_max_delta_t_size(std::size_t n) const
{
    if (n != m_impl->batch_size) {
        throw std::invalid_argument("Invalid number of max timesteps specified in a Taylor integrator in batch mode: "
                                    "the batch size is "
                                    + std::to_string(m_impl->batch_size)
                                    + ", but the number of specified timesteps is " + std::to_string(n));
    }
}

// ---- propagation (src/taylor_adaptive_batch.cpp:1081-1534) ----
std::tuple<std::optional<continuous_output_batch<double>>, step_callback_batch<double>>
taylor_adaptive_batch<double>::propagate_for_vec(const std::vector<double> &delta_ts, prop_opts o)
{
    auto &m = *m_impl;
    if (delta_ts.size() != m.batch_size) {
        throw std::invalid_argument("Invalid number of time intervals specified in a Taylor integrator in batch "
                                    "mode: the batch size is "
                                    + std::to_string(m.batch_size)
                                    + ", but the number of specified time intervals is "
                                    + std::to_string(delta_ts.size()));
    }
    m.refresh_time();
    std::vector<double> hi(m.batch_size), lo(m.batch_size);
    for (std::uint32_t i = 0; i < m.batch_size; ++i) {
        const auto r = dfl_add(dfl{m.time_hi[i], m.time_lo[i]}, dfl{delta_ts[i], 0.});
        hi[i] = r.hi;
        lo[i] = r.lo;
    }
    return propagate_until_impl(hi, lo, std::move(o));
}

std::tuple<std::optional<continuous_output_batch<double>>, step_callback_batch<double>>
taylor_adaptive_batch<double>::propagate_until_vec(const std::vector<double> &ts, prop_opts o)
{
    auto &m = *m_impl;
    if (ts.size() != m.batch_size) {
        throw std::invalid_argument("Invalid number of time limits specified in a Taylor integrator in batch mode: "
                                    "the batch size is "
                                    + std::to_string(m.batch_size) + ", but the number of specified time limits is "
                                    + std::to_string(ts.size()));
    }
    return propagate_until_impl(ts, std::vector<double>(m.batch_size, 0.), std::move(o));
}

// ---- continuous_output_batch<double> ----
continuous_output_batch<double>::continuous_output_batch(hy_cout *h, std::uint32_t batch_size, std::uint32_t dim,
                                                        std::uint32_t order)
    : m_h(h, [](hy_cout *p) { hy_cout_destroy(p); }), m_batch_size(batch_size), m_dim(dim), m_order(order),
      m_output(static_cast<std::size_t>(batch_size) * dim)
{
}

void continuous_output_batch<double>::check_valid() const
{
    if (!m_h) {
        throw std::invalid_argument("Cannot use a default-constructed continuous_output_batch object");
    }
}

const std::vector<double> &continuous_output_batch<double>::operator()(const std::vector<double> &tm)
{
    check_valid();
    if (tm.size() != m_batch_size) {
        throw std::invalid_argument("An invalid time vector was passed to the call operator of continuous_output_batch: "
                                    "the vector size is "
                                    + std::to_string(tm.size()) + ", but a size of " + std::to_string(m_batch_size)
                                    + " was expected instead");
    }
    return (*this)(tm.data());
}

const std::vector<double> &continuous_output_batch<double>::operator()(const double *tm)
{
    check_valid();
    check(hy_cout_eval(m_h.get(), tm, m_output.data()));
    return m_output;
}

const std::vector<double> &continuous_output_batch<double>::operator()(double tm)
{
    check_valid();
    return (*this)(std::vector<double>(m_batch_size, tm));
}

std::pair<std::vector<double>, std::vector<double>> continuous_output_batch<double>::get_bounds() const
{
    check_valid();
    std::vector<double> lb(m_batch_size), ub(m_batch_size);
    check(hy_cout_get_bounds(m_h.get(), lb.data(), ub.data()));
    return {std::move(lb), std::move(ub)};
}

std::size_t continuous_output_batch<double>::get_n_steps() const
{
    check_valid();
    return static_cast<std::size_t>(hy_cout_n_steps(m_h.get()));
}

const std::vector<double> &continuous_output_batch<double>::get_times() const
{
    check_valid();
    if (m_times_hi.empty()) {
        m_times_hi.resize((get_n_steps() + 2u) * m_batch_size);
        check(hy_cout_download(m_h.get(), m_times_hi.data(), nullptr, nullptr));
    }
    return m_times_hi;
}

const std::vector<double> &continuous_output_batch<double>::get_tcs() const
{
    check_valid();
    if (m_tcs.empty()) {
        m_tcs.resize(get_n_steps() * m_dim * (m_order + 1u) * m_batch_size);
        check(hy_cout_download(m_h.get(), nullptr, nullptr, m_tcs.data()));
    }
    return m_tcs;
}

// propagate_grid(): src/taylor_adaptive_batch.cpp:1545-2055. The size checks that need the reference's wording are
// done here, the grid checks and the integration by hy_batch_propagate_grid().
std::tuple<step_callback_batch<double>, std::vector<double>>
taylor_adaptive_batch<double>::propagate_grid_impl(const std::vector<double> &grid, prop_opts o)
{
    auto &m = *m_impl;
    const auto n = m.batch_size;
    const strict_scope strict(m);
    if (grid.empty()) {
        throw std::invalid_argument(
            "Cannot invoke propagate_grid() in an adaptive Taylor integrator in batch mode if the time grid is empty");
    }
    if (grid.size() % n != 0u) {
        throw std::invalid_argument(
            "Invalid grid size detected in propagate_grid() for an adaptive Taylor integrator in batch mode: "
            "the grid has a size of "
            + std::to_string(grid.size()) + ", which is not a multiple of the batch size (" + std::to_string(n) + ")");
    }
    if (!o.max_delta_t.empty() && o.max_delta_t.size() != n) {
        throw std::invalid_argument("Invalid number of max timesteps specified in a Taylor integrator in batch mode: "
                                    "the batch size is "
                                    + std::to_string(n) + ", but the number of specified timesteps is "
                                    + std::to_string(o.max_delta_t.size()));
    }
    if (o.cb || with_events() || !m.devices.empty()) {
        // A step callback (or events, whose callbacks also run on the host) after every step: the reference's loop on the
        // host, one device step per iteration. A batch sharded over several devices takes it too (the grid is sampled
        // through the dense output of the shards).
        return propagate_grid_events(grid, std::move(o));
    }
    std::vector<double> retval(grid.size() * m.dim);
    m.push();
    check(hy_batch_propagate_grid(m.batch, grid.data(), grid.size() / n,
                                  o.max_delta_t.empty() ? nullptr : o.max_delta_t.data(), o.max_steps, retval.data()));
    m.pull(true);
    m.pull_prop_res();
    return {std::move(o.cb), std::move(retval)};
}

// propagate_grid() of an integrator with events and / or with a step callback: the reference's loop
// (src/taylor_adaptive_batch.cpp:1696-2053) on the host - propagate_until() to the first grid point (without the
// callback, :1703-1706), then lock-step steps (with their event callbacks, then the step callback, which may stop the
// propagation and must not alter the time: :2004-2039) interleaved with dense-output sampling of the grid points each
// step covers.
std::tuple<step_callback_batch<double>, std::vector<double>>
taylor_adaptive_batch<double>::propagate_grid_events(const std::vector<double> &grid, prop_opts o)
{
    auto &m = *m_impl;
    const auto n = m.batch_size;
    const auto n_pts = grid.size() / n;
    const double *mdt = o.max_delta_t.empty() ? nullptr : o.max_delta_t.data();
    m.push();
    check(hy_batch_check_grid(m.batch, grid.data(), n_pts, mdt));
    std::vector<double> retval(grid.size() * m.dim, std::numeric_limits<double>::quiet_NaN());
    const double inf = std::numeric_limits<double>::infinity();

    {
        prop_opts po;
        po.max_steps = o.max_steps;
        po.max_delta_t = o.max_delta_t;
        po.write_tc = true;
        propagate_until_impl(std::vector<double>(grid.begin(), grid.begin() + n), std::vector<double>(n, 0.), std::move(po));
    }
    bool all_tl = true;
    for (const auto &r : m.prop_res) {
        all_tl = all_tl && std::get<0>(r) == taylor_outcome::time_limit;
    }
    if (!all_tl) {
        for (auto &r : m.prop_res) {
            std::get<1>(r) = inf;
            std::get<2>(r) = 0.;
            std::get<3>(r) = 0u;
        }
        return {std::move(o.cb), std::move(retval)};
    }
    std::copy(m.state.begin(), m.state.end(), retval.begin());

    std::vector<dfl> rem(n);
    std::vector<char> t_dir(n);
    for (std::uint32_t i = 0; i < n; ++i) {
        rem[i] = dfl_sub(dfl{grid[(n_pts - 1u) * n + i], 0.}, dfl{m.time_hi[i], m.time_lo[i]});
        if (!std::isfinite(rem[i].hi) || !std::isfinite(rem[i].lo)) {
            throw std::invalid_argument("The final time passed to the propagate_grid() function of an adaptive Taylor "
                                        "integrator in batch mode results in an overflow condition");
        }
        t_dir[i] = dfl_ge0(rem[i]) ? 1 : 0;
    }
    std::size_t iter_counter = 0;
    std::vector<std::size_t> ts_count(n, 0), cur_idx(n, 1);
    std::vector<double> min_h(n, inf), max_h(n, 0.), pgrid(n);
    std::vector<dfl> t0(n), t1(n);
    std::vector<unsigned> dflags(n);
    const auto cont_cond = [&]() {
        return std::any_of(cur_idx.begin(), cur_idx.end(), [n_pts](auto idx) { return idx < n_pts; });
    };
    while (cont_cond()) {
        for (std::uint32_t i = 0; i < n; ++i) {
            const dfl cur{m.time_hi[i], m.time_lo[i]}, cmp = dfl_sub(cur, dfl{m.last_h[i], 0.});
            t0[i] = dfl_lt(cmp, cur) ? cmp : cur;
            t1[i] = dfl_lt(cur, cmp) ? cmp : cur;
        }
        std::fill(dflags.begin(), dflags.end(), 1u);
        while (true) {
            std::uint32_t counter = 0;
            for (std::uint32_t i = 0; i < n; ++i) {
                const auto gidx = cur_idx[i];
                if (dflags[i] != 0u && gidx < n_pts) {
                    const dfl g{grid[gidx * n + i], 0.};
                    const bool d_avail = (!dfl_lt(g, t0[i]) && !dfl_lt(t1[i], g)) || (rem[i].hi == 0. && rem[i].lo == 0.);
                    dflags[i] = d_avail ? 1u : 0u;
                    counter += d_avail ? 1u : 0u;
                    pgrid[i] = g.hi;
                } else {
                    dflags[i] = 0u;
                }
            }
            if (counter == 0u) {
                break;
            }
            update_d_output(pgrid);
            for (std::uint32_t i = 0; i < n; ++i) {
                if (dflags[i] != 0u) {
                    for (std::uint32_t j = 0; j < m.dim; ++j) {
                        retval[cur_idx[i] * n * m.dim + j * n + i] = m.d_out[j * n + i];
                    }
                    ++cur_idx[i];
                }
            }
            if (!cont_cond()) {
                break;
            }
        }
        if (!cont_cond()) {
            break;
        }
        if (std::any_of(m.prop_res.begin(), m.prop_res.end(), [](const auto &t) {
                const auto oc = std::get<0>(t);
                return oc == taylor_outcome::cb_stop || (oc > taylor_outcome::success && oc < taylor_outcome{0})
                       || oc == taylor_outcome::step_limit;
            })) {
            break;
        }
        for (std::uint32_t i = 0; i < n; ++i) {
            const double md = mdt != nullptr ? mdt[i] : inf;
            const dfl lim = t_dir[i] ? (dfl_lt(rem[i], dfl{md, 0.}) ? rem[i] : dfl{md, 0.})
                                     : (dfl_lt(rem[i], dfl{-md, 0.}) ? dfl{-md, 0.} : rem[i]);
            pgrid[i] = lim.hi;
        }
        step_impl(&pgrid, false, true);
        bool nfs = false;
        for (std::uint32_t i = 0; i < n; ++i) {
            const auto [oc, h] = m.step_res[i];
            if (oc == taylor_outcome::err_nf_state) {
                nfs = true;
            } else {
                ts_count[i] += static_cast<std::size_t>(h != 0);
                if (oc == taylor_outcome::success) {
                    min_h[i] = std::min(min_h[i], std::abs(h));
                    max_h[i] = std::max(max_h[i], std::abs(h));
                }
                if (h == rem[i].hi) {
                    rem[i] = dfl{0., 0.};
                } else {
                    rem[i] = dfl_sub(dfl{grid[(n_pts - 1u) * n + i], 0.}, dfl{m.time_hi[i], m.time_lo[i]});
                }
            }
            m.prop_res[i] = std::tuple{oc, min_h[i], max_h[i], ts_count[i]};
        }
        if (nfs) {
            break;
        }
        ++iter_counter;
        bool cb_ok = true;
        if (o.cb) {
            const auto thi = m.time_hi, tlo = m.time_lo;
            cb_ok = o.cb(*this);
            if (m.time_hi != thi || m.time_lo != tlo) {
                throw std::runtime_error("The invocation of the callback passed to propagate_grid() resulted in the "
                                         "alteration of the time coordinate of the integrator - this is not supported");
            }
        }
        if (!cb_ok) {
            for (auto &t : m.prop_res) {
                std::get<0>(t) = taylor_outcome::cb_stop;
            }
        } else if (iter_counter == o.max_steps) {
            for (auto &t : m.prop_res) {
                std::get<0>(t) = taylor_outcome::step_limit;
            }
        }
    }
    return {std::move(o.cb), std::move(retval)};
}

std::tuple<std::optional<continuous_output_batch<double>>, step_callback_batch<double>>
taylor_adaptive_batch<double>::propagate_until_impl(const std::vector<double> &hi, const std::vector<double> &lo,
                                                    prop_opts o)
{
    auto &m = *m_impl;
    const auto n = m.batch_size;



    // Validation, src/taylor_adaptive_batch.cpp:1212-1273.
    m.refresh_time();
    for (std::uint32_t i = 0; i < n; ++i) {
        if (!std::isfinite(m.time_hi[i]) || !std::isfinite(m.time_lo[i])) {
            throw std::invalid_argument("Cannot invoke the propagate_until() function of an adaptive Taylor "
                                        "integrator in batch mode if one of the current times is not finite");
        }
    }
    for (std::uint32_t i = 0; i < n; ++i) {
        if (!std::isfinite(hi[i]) || !std::isfinite(lo[i])) {
            throw std::invalid_argument("A non-finite time was passed to the propagate_until() function of an "
                                        "adaptive Taylor integrator in batch mode");
        }
    }
    for (const auto dt : o.max_delta_t) {
        if (std::isnan(dt)) {
            throw std::invalid_argument("A nan max_delta_t was passed to the propagate_until() function of an "
                                        "adaptive Taylor integrator in batch mode");
        }
        if (dt <= 0) {
            throw std::invalid_argument("A non-positive max_delta_t was passed to the propagate_until() function of "
                                        "an adaptive Taylor integrator in batch mode");
        }
    }
    std::vector<dfl> rem(n);
    for (std::uint32_t i = 0; i < n; ++i) {
        rem[i] = dfl_sub(dfl{hi[i], lo[i]}, dfl{m.time_hi[i], m.time_lo[i]});
        if (!std::isfinite(rem[i].hi) || !std::isfinite(rem[i].lo)) {
            throw std::invalid_argument("The final time passed to the propagate_until() function of an adaptive "
                                        "Taylor integrator in batch mode results in an overflow condition");
        }
    }
    const double *mdt = o.max_delta_t.empty() ? nullptr : o.max_delta_t.data();

    if (o.c_output && !with_events()) {
        // The reference's lock-step loop with the recording of the Taylor coefficients, on the device
        // (hy_batch_propagate_until_cout()).
        m.push();
        hy_cout *co = nullptr;
        if (o.cb) {
            // With a step callback (:1476-1500): the library calls back after every recorded iteration; the mirrors are
            // refreshed for the callback, which may alter state and parameters (uploaded again) but not the time.
            struct hook_t {
                taylor_adaptive_batch *self;
                prop_opts *o;
                std::exception_ptr err;
            } hook{this, &o, nullptr};
            const auto tramp = [](void *user) -> int {
                auto &h = *static_cast<hook_t *>(user);
                auto &mm = *h.self->m_impl;
                const bool was_lazy = mm.lazy;
                try {
                    mm.lazy = false;
                    mm.pull(true);
                    mm.pull_prop_res();
                    const auto thi = mm.time_hi, tlo = mm.time_lo;
                    const bool go = h.o->cb(*h.self);
                    if (mm.time_hi != thi || mm.time_lo != tlo) {
                        throw std::runtime_error("The invocation of the callback passed to propagate_until() resulted in "
                                                 "the alteration of the time coordinate of the integrator - this is not "
                                                 "supported");
                    }
                    mm.host_new_state = mm.host_new_pars = true;
                    mm.push();
                    mm.lazy = was_lazy;
                    return go ? 1 : 0;
                } catch (...) {
                    mm.lazy = was_lazy;
                    h.err = std::current_exception();
                    return -1;
                }
            };
            const int st = hy_batch_propagate_until_cout_cb(m.batch, hi.data(), lo.data(), mdt, o.max_steps, tramp, &hook, &co);
            if (hook.err) {
                std::rethrow_exception(hook.err);
            }
            check(st);
        } else {
            check(hy_batch_propagate_until_cout(m.batch, hi.data(), lo.data(), mdt, o.max_steps, &co));
        }
        std::optional<continuous_output_batch<double>> ret;
        if (co != nullptr) {
            ret.emplace(co, n, m.dim, m.order);
        }
        m.pull(true);
        m.pull_prop_res();
        return {std::move(ret), std::move(o.cb)};
    }

    if (!o.cb && !with_events() && !m.lazy && !o.write_tc) {
        // Fast path, strict synchronisation: one call uploads the mirrors, runs the whole loop on the device and
        // brings state, times, last_h and the per-lane results back (no intermediate read-backs).
        check(hy_batch_propagate_until_host(m.batch, m.state.data(), m.n_pars != 0u ? m.pars.data() : nullptr,
                                            m.time_hi.data(), m.time_lo.data(), hi.data(), lo.data(), mdt, o.max_steps,
                                            m.state.data(), m.time_hi.data(), m.time_lo.data(), m.last_h.data(),
                                            m.oc.data(), m.tmp_a.data(), m.tmp_b.data(), m.tmp_n.data()));
        for (std::uint32_t i = 0; i < n; ++i) {
            m.prop_res[i] = std::tuple{static_cast<taylor_outcome>(m.oc[i]), m.tmp_a[i], m.tmp_b[i],
                                       static_cast<std::size_t>(m.tmp_n[i])};
        }
        m.host_new_state = m.host_new_pars = m.host_new_time = false;
        m.dev_new_state = m.dev_new_time = m.dev_new_prop = false;
        return {std::nullopt, std::move(o.cb)};
    }

    if (!o.cb && !with_events()) {
        // Fast path: the whole loop runs on the device.
        m.push();
        check(hy_batch_propagate_until(m.batch, hi.data(), lo.data(), mdt, o.max_steps, o.write_tc ? 1 : 0));
        m.pull(o.write_tc);
        m.pull_prop_res();
        return {std::nullopt, std::move(o.cb)};
    }

    const strict_scope strict(m);
    // Callback / events path: the reference's lock-step loop (src/taylor_adaptive_batch.cpp:1372-1527) on the host, one
    // device step per iteration (host callbacks force a synchronisation per step anyway).
    constexpr auto cb_time_errmsg
        = "The invocation of the callback passed to propagate_until() resulted in the alteration of the "
          "time coordinate of the integrator - this is not supported";
    std::vector<char> t_dir(n);
    std::vector<std::size_t> ts_count(n, 0);
    std::vector<double> min_h(n, std::numeric_limits<double>::infinity()), max_h(n, 0.), cur_max(n);
    for (std::uint32_t i = 0; i < n; ++i) {
        t_dir[i] = dfl_ge0(rem[i]) ? 1 : 0;
    }
    // Continuous output of an integrator with events: the iterations of this loop are recorded on the device
    // (update_c_out(), :1320-1346; make_c_out(), :1277-1317), every step of such an integrator writes its Taylor
    // coefficients.
    struct rec_guard {
        hy_cout_rec *r = nullptr;
        ~rec_guard()
        {
            if (r != nullptr) {
                hy_cout_rec_destroy(r);
            }
        }
    } rec;
    if (o.c_output) {
        m.push();
        check(hy_cout_rec_begin(m.batch, &rec.r));
    }
    const auto finish = [&]() -> std::tuple<std::optional<continuous_output_batch<double>>, step_callback_batch<double>> {
        std::optional<continuous_output_batch<double>> ret;
        if (rec.r != nullptr) {
            std::vector<unsigned char> fwd(n);
            for (std::uint32_t i = 0; i < n; ++i) {
                fwd[i] = t_dir[i] != 0 ? 1 : 0;
            }
            hy_cout *co = nullptr;
            hy_cout_rec *r = rec.r;
            rec.r = nullptr; // (finish() destroys the recorder)
            check(hy_cout_rec_finish(m.batch, r, fwd.data(), &co));
            if (co != nullptr) {
                ret.emplace(co, n, m.dim, m.order);
            }
        }
        return {std::move(ret), std::move(o.cb)};
    };
    std::size_t iter_counter = 0;
    while (true) {
        for (std::uint32_t i = 0; i < n; ++i) {
            const double md = mdt != nullptr ? mdt[i] : std::numeric_limits<double>::infinity();
            const dfl lim = t_dir[i] ? (dfl_lt(rem[i], dfl{md, 0.}) ? rem[i] : dfl{md, 0.})
                                     : (dfl_lt(rem[i], dfl{-md, 0.}) ? dfl{-md, 0.} : rem[i]);
            cur_max[i] = lim.hi;
        }
        step_impl(&cur_max, false, o.write_tc);

        std::uint32_t n_done = 0;
        bool nfs = false, ste_detected = false;
        for (std::uint32_t i = 0; i < n; ++i) {
            const auto [oc, h] = m.step_res[i];
            if (oc == taylor_outcome::err_nf_state) {
                nfs = true;
            } else {
                // A stopping terminal event in any batch element ends the propagation (:1430, :1503).
                ste_detected = ste_detected || (oc > taylor_outcome::success && oc < taylor_outcome{0});
                ts_count[i] += static_cast<std::size_t>(h != 0);
                if (oc == taylor_outcome::success) {
                    const auto ah = std::abs(h);
                    min_h[i] = std::min(min_h[i], ah);
                    max_h[i] = std::max(max_h[i], ah);
                }
                const bool cur_done = (h == rem[i].hi);
                n_done += cur_done ? 1u : 0u;
                if (cur_done) {
                    rem[i] = dfl{0., 0.};
                } else {
                    rem[i] = dfl_sub(dfl{hi[i], lo[i]}, dfl{m.time_hi[i], m.time_lo[i]});
                }
            }
            m.prop_res[i] = std::tuple{oc, min_h[i], max_h[i], ts_count[i]};
        }
        if (nfs) {
            return finish();
        }
        if (rec.r != nullptr) {
            check(hy_cout_rec_append(m.batch, rec.r));
        }
        ++iter_counter;
        if (o.cb) {
            const auto thi = m.time_hi, tlo = m.time_lo;
            const bool ret_cb = o.cb(*this);
            if (m.time_hi != thi || m.time_lo != tlo) {
                throw std::runtime_error(cb_time_errmsg);
            }
            if (!ret_cb) {
                for (auto &r : m.prop_res) {
                    std::get<0>(r) = taylor_outcome::cb_stop;
                }
                return finish();
            }
        }
        if (n_done == n || ste_detected) {
            return finish();
        }
        if (iter_counter == o.max_steps) {
            for (auto &r : m.prop_res) {
                std::get<0>(r) = taylor_outcome::step_limit;
            }
            return finish();
        }
    }
}

// ---- dense output (src/taylor_adaptive_batch.cpp:2251-2327) ----
const std::vector<double> &taylor_adaptive_batch<double>::update_d_output(const std::vector<double> &t, bool rel_time)
{
    auto &m = *m_impl;
    if (t.size() != m.batch_size) {
        throw std::invalid_argument("Invalid number of time coordinates specified for the dense output in a Taylor "
                                    "integrator in batch mode: the batch size is "
                                    + std::to_string(m.batch_size) + ", but the number of time coordinates is "
                                    + std::to_string(t.size()));
    }
    m.refresh_time();
    std::vector<double> tau(m.batch_size);
    for (std::uint32_t i = 0; i < m.batch_size; ++i) {
        if (rel_time) {
            // Relative to the CURRENT time; the kernel expands about the start of the last step (:2276-2280).
            tau[i] = m.last_h[i] + t[i];
        } else {
            // tau = t - (time - last_h) in double-length arithmetic (:2276-2286).
            const auto t0 = dfl_sub(dfl{m.time_hi[i], m.time_lo[i]}, dfl{m.last_h[i], 0.});
            tau[i] = dfl_sub(dfl{t[i], 0.}, t0).hi;
        }
    }
    check(hy_batch_d_output(m.batch, tau.data(), m.d_out.data()));
    return m.d_out;
}

const std::vector<double> &taylor_adaptive_batch<double>::update_d_output(double t, bool rel_time)
{
    return update_d_output(std::vector<double>(m_impl->batch_size, t), rel_time);
}

} // namespace heyoka_b200
