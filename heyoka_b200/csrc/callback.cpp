// callback::angle_reducer (include/heyoka_b200/callback.hpp). The reduction itself is angle_reduce.hpp's, compiled
// here into the library (hy_reduce_angles()).
#include <heyoka_b200/callback.hpp>

#include <algorithm>
#include <stdexcept>
#include <string>
#include <utility>

#include <heyoka_b200.h>
#include <heyoka_b200/taylor.hpp>

namespace heyoka_b200::callback
{

angle_reducer::angle_reducer(std::vector<expression> vars)
{
    if (vars.empty()) {
        throw std::invalid_argument("The list of expressions passed to the constructor of an angle reducer cannot be "
                                    "empty");
    }
    for (auto &v : vars) {
        if (!v.is_variable()) {
            throw std::invalid_argument("The list of expressions passed to the constructor of an angle reducer can "
                                        "contain only variables, but the expression '"
                                        + to_string(v) + "' is not a variable");
        }
        if (std::none_of(m_vars.begin(), m_vars.end(), [&v](const expression &w) { return w == v; })) {
            m_vars.push_back(std::move(v));
        }
    }
}

const std::vector<expression> &angle_reducer::get_vars() const noexcept
{
    return m_vars;
}

std::vector<std::uint32_t> angle_reducer::get_sv_indices(const taylor_adaptive_batch<double> &ta) const
{
    const auto &sys = ta.get_sys();
    std::vector<std::uint32_t> idx;
    idx.reserve(m_vars.size());
    for (const auto &v : m_vars) {
        const auto it = std::find_if(sys.begin(), sys.end(), [&v](const auto &eq) { return eq.first == v; });
        if (it == sys.end()) {
            throw std::invalid_argument("The variable '" + v.var_name()
                                        + "' passed to the angle reducer is not a state variable of the integrator");
        }
        idx.push_back(static_cast<std::uint32_t>(it - sys.begin()));
    }
    return idx;
}

void angle_reducer::pre_hook(taylor_adaptive_batch<double> &ta) const
{
    (void)get_sv_indices(ta);
}

bool angle_reducer::operator()(taylor_adaptive_batch<double> &ta) const
{
    const auto n = ta.get_batch_size();
    double *st = ta.get_state_data();
    for (const auto i : get_sv_indices(ta)) {
        if (hy_reduce_angles(st + static_cast<std::size_t>(i) * n, n) != HY_OK) {
            throw std::runtime_error(hy_last_error());
        }
    }
    return true;
}

} // namespace heyoka_b200::callback
