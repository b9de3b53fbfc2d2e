// heyoka_b200 — variational ODE systems (heyoka >= 5: var_ode_sys, var_args), first order.
//
// A var_ode_sys is an ODE system augmented with its first-order variational equations: the sensitivities
// dx_i/da_j of the state to a set of arguments a_j (state variables, i.e. initial conditions, and runtime parameters).
// For the stepper it is an ordinary ODE system: decomposition, lowering and every kernel take it unchanged.
//
// Layout (heyoka's documented order-1 layout): the augmented state is
//   [x_0 ... x_{n-1}, dx_0/da_0, dx_0/da_1, ..., dx_0/da_{m-1}, dx_1/da_0, ...]
// i.e. component-major, so that rows n.. of the state reshaped to (n, m) are the state-transition matrix. The
// variational variables are named "∂[(j, 1)]x_i" the way heyoka prints them.
//
// Right-hand sides: d/dt dx_i/da_j = sum_k (df_i/dx_k) dx_k/da_j (+ df_i/da_j when a_j is a parameter); partials
// that are identically zero are dropped.
//
// Scope: order 1 only. Orders > 1 and var_args::time (sensitivity to the initial time) are refused with
// not_implemented_error: the multi-index ordering of heyoka's dtens for order >= 2 and the initial conditions of the
// time sensitivity rest on the reference's source, which is not restated here. The argument conventions below
// (vars in LHS order, params in index order, vars before params) follow heyoka's documentation from memory, not a
// fixture.
#ifndef HEYOKA_B200_VAR_ODE_SYS_HPP
#define HEYOKA_B200_VAR_ODE_SYS_HPP

#include <cstdint>
#include <utility>
#include <variant>
#include <vector>

#include <heyoka_b200/exceptions.hpp>
#include <heyoka_b200/expression.hpp>

namespace heyoka_b200
{

// Bit flags selecting the arguments of the variational equations.
//   vars    the state variables, in the LHS order of the system
//   params  par[0 .. n_pars), in index order
//   time    the initial time (not implemented)
// vars | params: the state variables first, then the parameters.
enum class var_args : unsigned { vars = 0b001, params = 0b010, time = 0b100, all = 0b111 };

constexpr var_args operator|(var_args a, var_args b)
{
    return static_cast<var_args>(static_cast<unsigned>(a) | static_cast<unsigned>(b));
}
constexpr bool operator&(var_args a, var_args b)
{
    return (static_cast<unsigned>(a) & static_cast<unsigned>(b)) != 0u;
}

class var_ode_sys
{
    std::vector<std::pair<expression, expression>> m_sys;
    std::vector<expression> m_vargs;
    std::uint32_t m_n_orig_sv = 0, m_order = 1;

public:
    // args: flags, or an explicit list of state variables and / or parameters par[i], kept in the order given.
    // std::invalid_argument: order 0, an empty argument set, duplicates, an entry that is neither a state variable of
    // the system nor a parameter, a generated name that collides with a variable of the system.
    // not_implemented_error: order > 1, var_args::time, heyoka's `time` in the explicit list.
    var_ode_sys(const std::vector<std::pair<expression, expression>> &sys,
                const std::variant<var_args, std::vector<expression>> &args, std::uint32_t order = 1);

    // The augmented system: the original n equations, then the n * m variational equations.
    [[nodiscard]] const std::vector<std::pair<expression, expression>> &get_sys() const noexcept
    {
        return m_sys;
    }
    // The arguments a_0 .. a_{m-1}.
    [[nodiscard]] const std::vector<expression> &get_vargs() const noexcept
    {
        return m_vargs;
    }
    [[nodiscard]] std::uint32_t get_n_orig_sv() const noexcept
    {
        return m_n_orig_sv;
    }
    [[nodiscard]] std::uint32_t get_order() const noexcept
    {
        return m_order;
    }
};

} // namespace heyoka_b200

#endif
