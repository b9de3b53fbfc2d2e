// C ABI, host part: expression handles, model builders, program construction
// (include/heyoka_b200.h sections A and B). No CUDA in this translation unit.
#include <heyoka_b200.h>

#include <algorithm>
#include <cstring>
#include <functional>
#include <limits>
#include <new>
#include <stdexcept>
#include <string>
#include <vector>

#include <heyoka_b200/expression.hpp>
#include <heyoka_b200/model.hpp>
#include <heyoka_b200/taylor_decompose.hpp>
#include <heyoka_b200/var_ode_sys.hpp>

#include "angle_reduce.hpp"
#include "capi_common.hpp"
#include "program.hpp"

namespace hy = heyoka_b200;

struct hy_ex {
    hy::expression ex;
};

namespace heyoka_b200::detail
{

thread_local std::string tl_last_error;

void set_last_error(const std::string &msg)
{
    tl_last_error = msg;
}

int translate_exception()
{
    try {
        throw;
    } catch (const not_implemented_error &e) {
        set_last_error(e.what());
        return HY_ERR_NOT_IMPLEMENTED;
    } catch (const hy::not_implemented_error &e) {
        set_last_error(e.what());
        return HY_ERR_NOT_IMPLEMENTED;
    } catch (const cuda_error &e) {
        set_last_error(e.what());
        return HY_ERR_CUDA;
    } catch (const std::overflow_error &e) {
        set_last_error(e.what());
        return HY_ERR_OVERFLOW;
    } catch (const std::bad_alloc &) {
        set_last_error("Out of host memory");
        return HY_ERR_OVERFLOW;
    } catch (const std::exception &e) {
        set_last_error(e.what());
        return HY_ERR_INVALID_ARG;
    } catch (...) {
        set_last_error("Unknown error");
        return HY_ERR_INVALID_ARG;
    }
}

} // namespace heyoka_b200::detail

using hy::detail::set_last_error;
using hy::detail::translate_exception;

namespace
{

size_t copy_out(const std::string &s, char *buf, size_t buf_len)
{
    if (buf != nullptr && buf_len > 0u) {
        const auto n = std::min(buf_len - 1u, s.size());
        std::memcpy(buf, s.data(), n);
        buf[n] = '\0';
    }
    return s.size();
}

template <typename F>
hy_ex *make_ex(const F &f)
{
    try {
        return new hy_ex{f()};
    } catch (...) {
        translate_exception();
        return nullptr;
    }
}

} // namespace

extern "C" {

const char *hy_last_error(void)
{
    return hy::detail::tl_last_error.c_str();
}

const char *hy_version(void)
{
    return "heyoka_b200 0.1.0 (reference: bluescarni/heyoka 7.12.0 @ 9c91f71)";
}

hy_ex *hy_ex_num(double v)
{
    return make_ex([&] { return hy::expression{v}; });
}

hy_ex *hy_ex_var(const char *name)
{
    return make_ex([&] {
        if (name == nullptr || *name == '\0') {
            throw std::invalid_argument("A variable needs a non-empty name");
        }
        return hy::expression{hy::variable{name}};
    });
}

hy_ex *hy_ex_par(uint32_t idx)
{
    return make_ex([&] { return hy::par[idx]; });
}

hy_ex *hy_ex_time(void)
{
    return make_ex([&] { return hy::time; });
}

hy_ex *hy_ex_binary(char op, const hy_ex *a, const hy_ex *b)
{
    return make_ex([&]() -> hy::expression {
        if (a == nullptr || (b == nullptr && op != 'n')) {
            throw std::invalid_argument("Null expression handle");
        }
        switch (op) {
            case '+':
                return a->ex + b->ex;
            case '-':
                return a->ex - b->ex;
            case '*':
                return a->ex * b->ex;
            case '/':
                return a->ex / b->ex;
            case '^':
                return hy::pow(a->ex, b->ex);
            case 'n':
                return -a->ex;
            default:
                throw std::invalid_argument(std::string("Unknown binary operator '") + op + "'");
        }
    });
}

hy_ex *hy_ex_func(const char *name, const hy_ex *const *args, uint32_t n_args)
{
    return make_ex([&]() -> hy::expression {
        if (name == nullptr) {
            throw std::invalid_argument("Null function name");
        }
        std::vector<hy::expression> v;
        for (uint32_t i = 0; i < n_args; ++i) {
            if (args == nullptr || args[i] == nullptr) {
                throw std::invalid_argument("Null expression handle");
            }
            v.push_back(args[i]->ex);
        }
        const std::string s{name};
        const auto unary = [&](auto f) {
            if (v.size() != 1u) {
                throw std::invalid_argument("The function '" + s + "' takes exactly one argument");
            }
            return f(v[0]);
        };
        if (s == "sum") {
            return hy::sum(std::move(v));
        }
        if (s == "prod") {
            return hy::prod(std::move(v));
        }
        if (s == "sin") {
            return unary([](const auto &x) { return hy::sin(x); });
        }
        if (s == "cos") {
            return unary([](const auto &x) { return hy::cos(x); });
        }
        if (s == "tanh") {
            return unary([](const auto &x) { return hy::tanh(x); });
        }
        if (s == "exp") {
            return unary([](const auto &x) { return hy::exp(x); });
        }
        if (s == "sigmoid") {
            return unary([](const auto &x) { return hy::sigmoid(x); });
        }
        if (s == "relu") {
            return unary([](const auto &x) { return hy::relu(x); });
        }
        if (s == "leaky_relu" || s == "relup") {
            if (v.size() != 2u || !v[1].is_number()) {
                throw std::invalid_argument(s + " needs an argument and a numeric slope");
            }
            return s == "relup" ? hy::relup(v[0], v[1].num()) : hy::relu(v[0], v[1].num());
        }
        if (s == "log") {
            return unary([](const auto &x) { return hy::log(x); });
        }
        if (s == "sqrt") {
            return unary([](const auto &x) { return hy::sqrt(x); });
        }
        if (s == "square") {
            return unary([](const auto &x) { return hy::square(x); });
        }
        throw hy::detail::not_implemented_error("The function '" + s + "' is not implemented");
    });
}

hy_ex *hy_ex_copy(const hy_ex *e)
{
    return make_ex([&] {
        if (e == nullptr) {
            throw std::invalid_argument("Null expression handle");
        }
        return e->ex;
    });
}

void hy_ex_free(hy_ex *e)
{
    delete e;
}

size_t hy_ex_str(const hy_ex *e, char *buf, size_t buf_len)
{
    if (e == nullptr) {
        return copy_out("", buf, buf_len);
    }
    return copy_out(hy::to_string(e->ex), buf, buf_len);
}

hy_ex *hy_ex_diff(const hy_ex *e, const hy_ex *wrt)
{
    return make_ex([&] {
        if (e == nullptr || wrt == nullptr) {
            throw std::invalid_argument("Null expression handle");
        }
        return hy::diff(e->ex, wrt->ex);
    });
}

int hy_var_ode_sys(const hy_ex *const *lhs, const hy_ex *const *rhs, uint32_t n_eq, uint32_t flags,
                   const hy_ex *const *args, uint32_t n_args, uint32_t order, uint32_t *n_out_eq, uint32_t *n_out_args,
                   hy_ex **out_lhs, hy_ex **out_rhs, hy_ex **out_args)
{
    try {
        if ((n_eq != 0u && (lhs == nullptr || rhs == nullptr)) || n_out_eq == nullptr || n_out_args == nullptr
            || (flags == 0u && n_args != 0u && args == nullptr)) {
            throw std::invalid_argument("Null pointer passed to hy_var_ode_sys()");
        }
        std::vector<std::pair<hy::expression, hy::expression>> sys;
        for (uint32_t i = 0; i < n_eq; ++i) {
            if (lhs[i] == nullptr || rhs[i] == nullptr) {
                throw std::invalid_argument("Null expression handle");
            }
            sys.emplace_back(lhs[i]->ex, rhs[i]->ex);
        }
        std::variant<hy::var_args, std::vector<hy::expression>> va;
        if (flags != 0u) {
            if ((flags & ~(HY_VAR_ARGS_VARS | HY_VAR_ARGS_PARAMS | HY_VAR_ARGS_TIME)) != 0u) {
                throw std::invalid_argument("Invalid flags passed to hy_var_ode_sys(): " + std::to_string(flags));
            }
            va = static_cast<hy::var_args>(flags);
        } else {
            std::vector<hy::expression> v;
            for (uint32_t i = 0; i < n_args; ++i) {
                if (args[i] == nullptr) {
                    throw std::invalid_argument("Null expression handle");
                }
                v.push_back(args[i]->ex);
            }
            va = std::move(v);
        }
        const hy::var_ode_sys vsys(sys, va, order);
        const auto &aug = vsys.get_sys();
        *n_out_eq = static_cast<uint32_t>(aug.size());
        *n_out_args = static_cast<uint32_t>(vsys.get_vargs().size());
        if (out_lhs != nullptr && out_rhs != nullptr && out_args != nullptr) {
            for (std::size_t i = 0; i < aug.size(); ++i) {
                out_lhs[i] = new hy_ex{aug[i].first};
                out_rhs[i] = new hy_ex{aug[i].second};
            }
            for (std::size_t j = 0; j < vsys.get_vargs().size(); ++j) {
                out_args[j] = new hy_ex{vsys.get_vargs()[j]};
            }
        }
        return HY_OK;
    } catch (...) {
        return translate_exception();
    }
}

int hy_model_nbody(uint32_t n, const double *masses, uint32_t n_masses, double G, hy_ex **lhs, hy_ex **rhs)
{
    try {
        std::vector<hy::expression> m;
        if (masses == nullptr) {
            m.resize(n, hy::expression{1.});
        } else {
            for (uint32_t i = 0; i < n_masses; ++i) {
                m.emplace_back(masses[i]);
            }
        }
        const auto sys = hy::model::detail::nbody_impl(n, hy::expression{G}, m);
        for (std::size_t i = 0; i < sys.size(); ++i) {
            lhs[i] = new hy_ex{sys[i].first};
            rhs[i] = new hy_ex{sys[i].second};
        }
        return HY_OK;
    } catch (...) {
        return translate_exception();
    }
}

int hy_model_pendulum(double g, double l, hy_ex **lhs, hy_ex **rhs)
{
    try {
        const auto sys = hy::model::detail::pendulum_impl(hy::expression{g}, hy::expression{l});
        for (std::size_t i = 0; i < sys.size(); ++i) {
            lhs[i] = new hy_ex{sys[i].first};
            rhs[i] = new hy_ex{sys[i].second};
        }
        return HY_OK;
    } catch (...) {
        return translate_exception();
    }
}

int hy_model_ffnn(const hy_ex *const *inputs, uint32_t n_in, const uint32_t *nn_hidden, uint32_t n_hidden, uint32_t n_out,
                  const int *act, const double *nn_wb, uint32_t n_wb, hy_ex **out)
{
    try {
        std::vector<hy::expression> in;
        for (uint32_t i = 0; i < n_in; ++i) {
            in.push_back(inputs[i]->ex);
        }
        std::vector<std::uint32_t> hidden(nn_hidden, nn_hidden + n_hidden);
        std::vector<std::function<hy::expression(const hy::expression &)>> acts;
        for (uint32_t i = 0; i < n_hidden + 1u; ++i) {
            switch (act[i]) {
                case 0:
                    acts.emplace_back([](const hy::expression &e) { return e; });
                    break;
                case 1:
                    acts.emplace_back([](const hy::expression &e) { return hy::tanh(e); });
                    break;
                case 2:
                    acts.emplace_back([](const hy::expression &e) { return hy::sin(e); });
                    break;
                case 3:
                    acts.emplace_back([](const hy::expression &e) { return hy::exp(e); });
                    break;
                case 4:
                    acts.emplace_back([](const hy::expression &e) { return hy::sigmoid(e); });
                    break;
                case 5:
                    acts.emplace_back([](const hy::expression &e) { return hy::relu(e); });
                    break;
                default:
                    throw std::invalid_argument("Unknown activation id " + std::to_string(act[i]));
            }
        }
        std::vector<std::uint32_t> n_neurons{n_in};
        n_neurons.insert(n_neurons.end(), hidden.begin(), hidden.end());
        n_neurons.push_back(n_out);
        std::uint32_t expected = 0;
        for (std::size_t i = 1; i < n_neurons.size(); ++i) {
            expected += n_neurons[i - 1u] * n_neurons[i] + n_neurons[i];
        }
        std::vector<hy::expression> wb;
        if (nn_wb != nullptr) {
            for (uint32_t i = 0; i < n_wb; ++i) {
                wb.emplace_back(nn_wb[i]);
            }
        } else {
            for (uint32_t i = 0; i < expected; ++i) {
                wb.push_back(hy::par[i]);
            }
        }
        const auto res = hy::model::detail::ffnn_impl(in, hidden, n_out, acts, wb);
        for (std::size_t i = 0; i < res.size(); ++i) {
            out[i] = new hy_ex{res[i]};
        }
        return HY_OK;
    } catch (...) {
        return translate_exception();
    }
}

int hy_reduce_angles(double *x, uint64_t n)
{
    if (n != 0u && x == nullptr) {
        hy::detail::set_last_error("Null pointer passed to hy_reduce_angles()");
        return HY_ERR_INVALID_ARG;
    }
    for (uint64_t i = 0; i < n; ++i) {
        x[i] = hy::detail::reduce_angle(x[i]);
    }
    return HY_OK;
}

int hy_order_from_tol(double tol, uint32_t *order)
{
    try {
        *order = hy::detail::taylor_order_from_tol(tol);
        return HY_OK;
    } catch (...) {
        return translate_exception();
    }
}

int hy_program_from_sys_ev(const hy_ex *const *lhs, const hy_ex *const *rhs, uint32_t n_eq, const hy_ex *const *evs,
                           uint32_t n_ev, double tol, int high_accuracy, hy_program **out)
{
    try {
        if (lhs == nullptr || rhs == nullptr || out == nullptr || (n_ev != 0u && evs == nullptr)) {
            throw std::invalid_argument("Null pointer passed to hy_program_from_sys()");
        }
        std::vector<std::pair<hy::expression, hy::expression>> sys;
        std::vector<hy::expression> all_rhs, ev_ex;
        for (uint32_t i = 0; i < n_eq; ++i) {
            if (lhs[i] == nullptr || rhs[i] == nullptr) {
                throw std::invalid_argument("Null expression handle");
            }
            sys.emplace_back(lhs[i]->ex, rhs[i]->ex);
            all_rhs.push_back(rhs[i]->ex);
        }
        for (uint32_t i = 0; i < n_ev; ++i) {
            if (evs[i] == nullptr) {
                throw std::invalid_argument("Null expression handle");
            }
            ev_ex.push_back(evs[i]->ex);
            // The parameters of the event equations count (test/taylor_adaptive_batch.cpp:1015-1060).
            all_rhs.push_back(evs[i]->ex);
        }
        hy::validate_ode_sys(sys, ev_ex);

        // Tolerance checks: src/taylor_adaptive_batch.cpp:225-241.
        if (!(tol == tol) || tol == std::numeric_limits<double>::infinity() || tol < 0) {
            throw std::invalid_argument("The tolerance in an adaptive Taylor integrator must be finite and positive, "
                                        "but it is "
                                        + std::to_string(tol) + " instead");
        }
        if (tol == 0) {
            tol = std::numeric_limits<double>::epsilon();
        }
        const auto order = hy::detail::taylor_order_from_tol(tol);

        auto [dc, sv] = hy::taylor_decompose_sys(sys, ev_ex);
        const auto n_pars = hy::get_param_size(all_rhs);
        auto p = hy::detail::lower_decomposition(dc, n_eq, n_pars, order, high_accuracy != 0);
        p.ev_defs = std::move(sv);
        *out = new hy_program(std::move(p));
        return HY_OK;
    } catch (...) {
        return translate_exception();
    }
}

int hy_program_from_sys(const hy_ex *const *lhs, const hy_ex *const *rhs, uint32_t n_eq, double tol, int high_accuracy,
                        hy_program **out)
{
    return hy_program_from_sys_ev(lhs, rhs, n_eq, nullptr, 0u, tol, high_accuracy, out);
}

int hy_program_create(const hy_program_desc *d, hy_program **out)
{
    try {
        if (d == nullptr || out == nullptr) {
            throw std::invalid_argument("Null pointer passed to hy_program_create()");
        }
        if (d->n_uvars < d->n_eq) {
            throw std::invalid_argument("Invalid program: n_uvars < n_eq");
        }
        hy_program p;
        p.n_eq = d->n_eq;
        p.n_uvars = d->n_uvars;
        p.n_pars = d->n_pars;
        p.order = d->order;
        p.high_accuracy = d->high_accuracy != 0;
        p.ops.assign(d->ops, d->ops + (d->n_uvars - d->n_eq));
        p.args.assign(d->args, d->args + d->n_args);
        p.consts.assign(d->consts, d->consts + d->n_consts);
        p.sv_defs.assign(d->sv_defs, d->sv_defs + d->n_eq);
        if (d->n_ev != 0u) {
            if (d->ev_defs == nullptr) {
                throw std::invalid_argument("Invalid program: event equations without their definitions");
            }
            p.ev_defs.assign(d->ev_defs, d->ev_defs + d->n_ev);
            for (const auto u : p.ev_defs) {
                if (u >= p.n_uvars) {
                    throw std::invalid_argument("Invalid program: an event equation refers to a u variable out of range");
                }
            }
        }
        hy::detail::validate_program(p);
        *out = new hy_program(std::move(p));
        return HY_OK;
    } catch (...) {
        return translate_exception();
    }
}

int hy_program_get_desc(const hy_program *p, hy_program_desc *out)
{
    if (p == nullptr || out == nullptr) {
        set_last_error("Null pointer passed to hy_program_get_desc()");
        return HY_ERR_INVALID_ARG;
    }
    *out = p->desc();
    return HY_OK;
}

uint32_t hy_program_dc_size(const hy_program *p)
{
    return p == nullptr ? 0u : p->n_uvars + p->n_eq;
}

size_t hy_program_dc_str(const hy_program *p, char *buf, size_t buf_len)
{
    if (p == nullptr) {
        return copy_out("", buf, buf_len);
    }
    return copy_out(hy::dc_to_string(p->dc), buf, buf_len);
}

int hy_program_costs(const hy_program *p, double *b_min, double *b_tape, double *flops)
{
    if (p == nullptr) {
        set_last_error("Null pointer passed to hy_program_costs()");
        return HY_ERR_INVALID_ARG;
    }
    const auto c = hy::detail::compute_costs(*p);
    if (b_min != nullptr) {
        *b_min = c.b_min;
    }
    if (b_tape != nullptr) {
        *b_tape = c.b_tape;
    }
    if (flops != nullptr) {
        *flops = c.flops;
    }
    return HY_OK;
}

void hy_program_destroy(hy_program *p)
{
    delete p;
}

} // extern "C"
