// var_ode_sys: see include/heyoka_b200/var_ode_sys.hpp for the layout and the scope.
#include <heyoka_b200/var_ode_sys.hpp>

#include <set>
#include <stdexcept>
#include <string>
#include <unordered_map>

namespace heyoka_b200
{

namespace
{

// "∂[(j, 1)]x": heyoka's rendering of the order-1 derivative of x with respect to argument j.
std::string var_name(std::size_t j, const std::string &x)
{
    return "∂[(" + std::to_string(j) + ", 1)]" + x;
}

} // namespace

var_ode_sys::var_ode_sys(const std::vector<std::pair<expression, expression>> &sys,
                         const std::variant<var_args, std::vector<expression>> &args, std::uint32_t order)
{
    if (order == 0u) {
        throw std::invalid_argument("The order of a variational ODE system cannot be zero");
    }
    if (order > 1u) {
        throw not_implemented_error("Variational equations of order " + std::to_string(order)
                                    + " are not implemented: only order 1 is supported");
    }
    if (sys.empty()) {
        throw std::invalid_argument("Cannot formulate the variational equations of an empty ODE system");
    }

    const auto n = sys.size();
    std::unordered_map<std::string, std::size_t> sv_idx;
    std::vector<expression> rhs;
    for (std::size_t i = 0; i < n; ++i) {
        if (!sys[i].first.is_variable()) {
            throw std::invalid_argument("The left-hand side of an ODE must be a variable, but '"
                                        + to_string(sys[i].first) + "' was found instead");
        }
        if (!sv_idx.emplace(sys[i].first.var_name(), i).second) {
            throw std::invalid_argument("The state variable '" + sys[i].first.var_name()
                                        + "' appears more than once in the left-hand sides of the ODE system");
        }
        rhs.push_back(sys[i].second);
    }

    // The arguments a_j.
    if (std::holds_alternative<var_args>(args)) {
        const auto f = std::get<var_args>(args);
        if (f & var_args::time) {
            throw not_implemented_error("Variational equations with respect to the initial time (var_args::time) are "
                                        "not implemented");
        }
        if (f & var_args::vars) {
            for (const auto &p : sys) {
                m_vargs.push_back(p.first);
            }
        }
        if (f & var_args::params) {
            const auto n_pars = get_param_size(rhs);
            for (std::uint32_t i = 0; i < n_pars; ++i) {
                m_vargs.push_back(par[i]);
            }
        }
    } else {
        for (const auto &a : std::get<std::vector<expression>>(args)) {
            if (a.is_func() && a.fn().kind == func_kind::time) {
                throw not_implemented_error("Variational equations with respect to the initial time are not "
                                            "implemented");
            }
            if (!(a.is_param() || (a.is_variable() && sv_idx.count(a.var_name()) != 0u))) {
                throw std::invalid_argument("The argument '" + to_string(a)
                                            + "' of a variational ODE system is neither a state variable of the "
                                              "system nor a parameter");
            }
            for (const auto &b : m_vargs) {
                if (b == a) {
                    throw std::invalid_argument("The argument '" + to_string(a)
                                                + "' appears more than once in the arguments of a variational ODE "
                                                  "system");
                }
            }
            m_vargs.push_back(a);
        }
    }
    if (m_vargs.empty()) {
        throw std::invalid_argument("The set of arguments of a variational ODE system cannot be empty");
    }
    const auto m = m_vargs.size();

    // The variational variables Phi[k][j], checked against every name the system already uses.
    std::set<std::string> used;
    for (const auto &p : sys) {
        used.insert(p.first.var_name());
        for (auto &v : get_variables(p.second)) {
            used.insert(std::move(v));
        }
    }
    std::vector<expression> phi;
    phi.reserve(n * m);
    for (std::size_t k = 0; k < n; ++k) {
        for (std::size_t j = 0; j < m; ++j) {
            auto name = var_name(j, sys[k].first.var_name());
            if (used.count(name) != 0u) {
                throw std::invalid_argument("The name '" + name
                                            + "' of a variational variable collides with a variable of the ODE system");
            }
            phi.emplace_back(variable{std::move(name)});
        }
    }

    // Jacobian df_i/dx_k, zeros kept as the number 0.
    std::vector<expression> jac(n * n);
    for (std::size_t i = 0; i < n; ++i) {
        for (std::size_t k = 0; k < n; ++k) {
            jac[i * n + k] = diff(rhs[i], sys[k].first);
        }
    }

    m_sys = sys;
    m_sys.reserve(n * (1u + m));
    for (std::size_t i = 0; i < n; ++i) {
        for (std::size_t j = 0; j < m; ++j) {
            std::vector<expression> terms;
            for (std::size_t k = 0; k < n; ++k) {
                const auto &J = jac[i * n + k];
                if (J.is_number() && J.num() == 0.) {
                    continue;
                }
                terms.push_back(prod({J, phi[k * m + j]}));
            }
            if (m_vargs[j].is_param()) {
                terms.push_back(diff(rhs[i], m_vargs[j]));
            }
            m_sys.emplace_back(phi[i * m + j], sum(std::move(terms)));
        }
    }
    m_n_orig_sv = static_cast<std::uint32_t>(n);
    m_order = order;
}

} // namespace heyoka_b200
