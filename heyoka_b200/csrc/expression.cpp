// Symbolic front end: see include/heyoka_b200/expression.hpp for the reference map.
#include <heyoka_b200/expression.hpp>

#include <algorithm>
#include <cmath>
#include <cstdio>
#include <set>
#include <sstream>
#include <stdexcept>
#include <unordered_map>
#include <unordered_set>

namespace heyoka_b200
{

const char *func_kind_name(func_kind k)
{
    switch (k) {
        case func_kind::sum:
            return "sum";
        case func_kind::prod:
            return "prod";
        case func_kind::pow:
            return "pow";
        case func_kind::sub:
            return "sub";
        case func_kind::div:
            return "div";
        case func_kind::sum_sq:
            return "sum_sq";
        case func_kind::sin:
            return "sin";
        case func_kind::cos:
            return "cos";
        case func_kind::tanh:
            return "tanh";
        case func_kind::sigmoid:
            return "sigmoid";
        case func_kind::relu:
            return "relu";
        case func_kind::relup:
            return "relup";
        case func_kind::exp:
            return "exp";
        case func_kind::log:
            return "log";
        case func_kind::time:
            return "time";
        case func_kind::num_identity:
            return "num_identity";
    }
    return "?";
}

expression::expression() : m_value(number{0.}) {}
expression::expression(double x) : m_value(number{x}) {}
expression::expression(number n) : m_value(n) {}
expression::expression(variable v) : m_value(std::move(v)) {}
expression::expression(param p) : m_value(p) {}
expression::expression(std::string s) : m_value(variable{std::move(s)}) {}
expression::expression(func_ptr f) : m_value(std::move(f)) {}
expression::expression(func_kind k, std::vector<expression> args)
    : m_value(std::make_shared<const func_node>(func_node{k, std::move(args)}))
{
}

bool operator==(const expression &a, const expression &b)
{
    if (a.value().index() != b.value().index()) {
        return false;
    }
    switch (a.value().index()) {
        case 0: {
            // NOTE: like the reference's number comparison, NaNs compare equal to each other
            // (src/number.cpp operator==), everything else by value.
            const auto x = a.num(), y = b.num();
            return (std::isnan(x) && std::isnan(y)) || x == y;
        }
        case 1:
            return a.var_name() == b.var_name();
        case 2:
            return a.par_idx() == b.par_idx();
        default: {
            if (a.fn_id() == b.fn_id()) {
                return true;
            }
            const auto &fa = a.fn();
            const auto &fb = b.fn();
            if (fa.kind != fb.kind || fa.args.size() != fb.args.size()) {
                return false;
            }
            for (std::size_t i = 0; i < fa.args.size(); ++i) {
                if (!(fa.args[i] == fb.args[i])) {
                    return false;
                }
            }
            return true;
        }
    }
}

bool operator!=(const expression &a, const expression &b)
{
    return !(a == b);
}

namespace
{
inline void hash_combine(std::size_t &seed, std::size_t v)
{
    seed ^= v + 0x9e3779b97f4a7c15ull + (seed << 6) + (seed >> 2);
}
} // namespace

std::size_t hash_value(const expression &e)
{
    switch (e.value().index()) {
        case 0:
            return std::isnan(e.num()) ? std::size_t(0x7ff8) : std::hash<double>{}(e.num());
        case 1:
            return std::hash<std::string>{}(e.var_name());
        case 2:
            return std::hash<std::uint32_t>{}(e.par_idx()) ^ 0xabcdefu;
        default: {
            const auto &f = e.fn();
            std::size_t seed = static_cast<std::size_t>(f.kind) + 17u;
            for (const auto &a : f.args) {
                hash_combine(seed, hash_value(a));
            }
            return seed;
        }
    }
}

std::ostream &operator<<(std::ostream &os, const expression &e)
{
    switch (e.value().index()) {
        case 0: {
            char buf[64];
            std::snprintf(buf, sizeof(buf), "%.17g", e.num());
            os << buf;
            break;
        }
        case 1:
            os << e.var_name();
            break;
        case 2:
            os << "p" << e.par_idx();
            break;
        default: {
            const auto &f = e.fn();
            os << func_kind_name(f.kind) << '(';
            for (std::size_t i = 0; i < f.args.size(); ++i) {
                if (i) {
                    os << ", ";
                }
                os << f.args[i];
            }
            os << ')';
        }
    }
    return os;
}

std::string to_string(const expression &e)
{
    std::ostringstream oss;
    oss << e;
    return oss.str();
}

// ---------------------------------------------------------------------------------------------
// Operators: src/expression_ops.cpp:36-92.
// ---------------------------------------------------------------------------------------------
expression operator+(expression e)
{
    return e;
}

expression operator-(const expression &e)
{
    if (e.is_number()) {
        return expression{-e.num()};
    }
    return prod({expression{-1.}, e});
}

expression operator+(const expression &a, const expression &b)
{
    if (a.is_number() && b.is_number()) {
        return expression{a.num() + b.num()};
    }
    return sum({a, b});
}

expression operator-(const expression &a, const expression &b)
{
    if (a.is_number() && b.is_number()) {
        return expression{a.num() - b.num()};
    }
    return a + -b;
}

expression operator*(const expression &a, const expression &b)
{
    if (a.is_number() && b.is_number()) {
        return expression{a.num() * b.num()};
    }
    return prod({a, b});
}

expression operator/(const expression &a, const expression &b)
{
    if (a.is_number() && b.is_number()) {
        return expression{a.num() / b.num()};
    }
    return prod({a, pow(b, expression{-1.})});
}

expression operator+(const expression &a, double b)
{
    return a + expression{b};
}
expression operator-(const expression &a, double b)
{
    return a - expression{b};
}
expression operator*(const expression &a, double b)
{
    return a * expression{b};
}
expression operator/(const expression &a, double b)
{
    return a / expression{b};
}
expression operator+(double a, const expression &b)
{
    return expression{a} + b;
}
expression operator-(double a, const expression &b)
{
    return expression{a} - b;
}
expression operator*(double a, const expression &b)
{
    return expression{a} * b;
}
expression operator/(double a, const expression &b)
{
    return expression{a} / b;
}
expression &operator+=(expression &x, const expression &e)
{
    return x = x + e;
}
expression &operator-=(expression &x, const expression &e)
{
    return x = x - e;
}
expression &operator*=(expression &x, const expression &e)
{
    return x = x * e;
}
expression &operator/=(expression &x, const expression &e)
{
    return x = x / e;
}

// ---------------------------------------------------------------------------------------------
// sum(): src/math/sum.cpp:548-601.
// ---------------------------------------------------------------------------------------------
expression sum(std::vector<expression> args)
{
    // Numbers to the end, fold them into one.
    const auto n_end_it
        = std::stable_partition(args.begin(), args.end(), [](const expression &ex) { return !ex.is_number(); });

    if (n_end_it != args.end()) {
        for (auto it = n_end_it + 1; it != args.end(); ++it) {
            *n_end_it = expression{n_end_it->num() + it->num()};
        }
        args.erase(n_end_it + 1, args.end());

        if (n_end_it->num() == 0.) {
            if (args.size() == 1u) {
                return std::move(*n_end_it);
            }
            args.pop_back();
        }
    }

    if (args.empty()) {
        return expression{0.};
    }
    if (args.size() == 1u) {
        return std::move(args[0]);
    }

    // Numbers first (semi-canonical form).
    std::stable_partition(args.begin(), args.end(), [](const expression &ex) { return ex.is_number(); });

    return expression{func_kind::sum, std::move(args)};
}

// ---------------------------------------------------------------------------------------------
// prod(): src/math/prod.cpp:913-975.
// ---------------------------------------------------------------------------------------------
expression prod(std::vector<expression> args)
{
    const auto n_end_it
        = std::stable_partition(args.begin(), args.end(), [](const expression &ex) { return !ex.is_number(); });

    if (n_end_it != args.end()) {
        for (auto it = n_end_it + 1; it != args.end(); ++it) {
            *n_end_it = expression{n_end_it->num() * it->num()};
        }
        args.erase(n_end_it + 1, args.end());

        if (n_end_it->num() == 1.) {
            if (args.size() == 1u) {
                return std::move(*n_end_it);
            }
            args.pop_back();
        } else if (n_end_it->num() == 0.) {
            return std::move(*n_end_it);
        }
    }

    if (args.empty()) {
        return expression{1.};
    }
    if (args.size() == 1u) {
        return std::move(args[0]);
    }

    std::stable_partition(args.begin(), args.end(), [](const expression &ex) { return ex.is_number(); });

    return expression{func_kind::prod, std::move(args)};
}

// ---------------------------------------------------------------------------------------------
// pow(): src/math/pow.cpp:1024-1062.
// ---------------------------------------------------------------------------------------------
expression pow(const expression &b, const expression &e)
{
    if (b.is_number() && e.is_number()) {
        return expression{std::pow(b.num(), e.num())};
    }
    if (e.is_number()) {
        if (e.num() == 0.) {
            return expression{1.};
        }
        if (e.num() == 1.) {
            return b;
        }
    }
    return expression{func_kind::pow, {b, e}};
}

expression pow(const expression &b, double e)
{
    return pow(b, expression{e});
}

// src/math/sqrt.cpp:16, src/math/square.cpp.
expression sqrt(const expression &e)
{
    return pow(e, expression{.5});
}

expression square(const expression &e)
{
    return pow(e, expression{2.});
}

namespace
{
// Unary functions fold numeric arguments at construction (e.g. src/math/sin.cpp:406-420).
template <typename F>
expression unary_builder(func_kind k, expression e, const F &f)
{
    if (e.is_number()) {
        return expression{f(e.num())};
    }
    return expression{k, {std::move(e)}};
}
} // namespace

expression sin(expression e)
{
    return unary_builder(func_kind::sin, std::move(e), [](double x) { return std::sin(x); });
}
expression cos(expression e)
{
    return unary_builder(func_kind::cos, std::move(e), [](double x) { return std::cos(x); });
}
expression tanh(expression e)
{
    return unary_builder(func_kind::tanh, std::move(e), [](double x) { return std::tanh(x); });
}
expression sigmoid(expression e)
{
    // 1 / (1 + exp(-x)), src/math/sigmoid.cpp:69-75.
    return unary_builder(func_kind::sigmoid, std::move(e), [](double x) { return 1. / (1. + std::exp(-x)); });
}
expression relu(expression e, double slope)
{
    if (!std::isfinite(slope) || slope < 0) {
        throw std::invalid_argument("The slope parameter for a leaky ReLU must be finite and non-negative, but the value "
                                    + std::to_string(slope) + " was provided instead");
    }
    if (e.is_number()) {
        const double x = e.num();
        return expression{x > 0 ? x : (slope == 0 ? 0. : slope * x)};
    }
    return expression{func_kind::relu, {std::move(e), expression{slope}}};
}
expression relup(expression e, double slope)
{
    if (!std::isfinite(slope) || slope < 0) {
        throw std::invalid_argument("The slope parameter for a leaky ReLU must be finite and non-negative, but the value "
                                    + std::to_string(slope) + " was provided instead");
    }
    if (e.is_number()) {
        return expression{e.num() > 0 ? 1. : slope};
    }
    return expression{func_kind::relup, {std::move(e), expression{slope}}};
}
expression exp(expression e)
{
    return unary_builder(func_kind::exp, std::move(e), [](double x) { return std::exp(x); });
}
expression log(expression e)
{
    return unary_builder(func_kind::log, std::move(e), [](double x) { return std::log(x); });
}

const expression time{func_kind::time, {}};

expression par_impl::operator[](std::uint32_t idx) const
{
    return expression{param{idx}};
}

inline namespace literals
{
expression operator""_dbl(long double x)
{
    return expression{static_cast<double>(x)};
}
expression operator""_dbl(unsigned long long n)
{
    return expression{static_cast<double>(n)};
}
} // namespace literals

namespace detail
{
std::pair<expression, expression> prime_wrapper::operator=(expression rhs) &&
{
    return {std::move(m_lhs), std::move(rhs)};
}
} // namespace detail

detail::prime_wrapper prime(const expression &e)
{
    if (!e.is_variable()) {
        throw std::invalid_argument("Cannot apply the prime() operator to a non-variable expression");
    }
    return detail::prime_wrapper{e};
}

// ---------------------------------------------------------------------------------------------
// Traversal helpers.
// ---------------------------------------------------------------------------------------------
namespace
{
void collect_vars(std::unordered_set<const void *> &seen, std::set<std::string> &out, const expression &e)
{
    // Iterative DFS with a visited set on function identity.
    std::vector<const expression *> stack{&e};
    while (!stack.empty()) {
        const auto *cur = stack.back();
        stack.pop_back();
        if (cur->is_variable()) {
            out.insert(cur->var_name());
        } else if (cur->is_func()) {
            if (!seen.insert(cur->fn_id()).second) {
                continue;
            }
            for (const auto &a : cur->fn().args) {
                stack.push_back(&a);
            }
        }
    }
}
} // namespace

// Sorted (lexicographically) list of unique variable names (src/expression_basic.cpp get_variables()).
std::vector<std::string> get_variables(const expression &e)
{
    std::unordered_set<const void *> seen;
    std::set<std::string> out;
    collect_vars(seen, out, e);
    return {out.begin(), out.end()};
}

std::uint32_t get_param_size(const std::vector<expression> &v)
{
    std::uint32_t ret = 0;
    std::unordered_set<const void *> seen;
    std::vector<const expression *> stack;
    for (const auto &e : v) {
        stack.push_back(&e);
    }
    while (!stack.empty()) {
        const auto *cur = stack.back();
        stack.pop_back();
        if (cur->is_param()) {
            ret = std::max(ret, cur->par_idx() + 1u);
        } else if (cur->is_func()) {
            if (!seen.insert(cur->fn_id()).second) {
                continue;
            }
            for (const auto &a : cur->fn().args) {
                stack.push_back(&a);
            }
        }
    }
    return ret;
}

bool is_time_dependent(const std::vector<expression> &v)
{
    std::unordered_set<const void *> seen;
    std::vector<const expression *> stack;
    for (const auto &e : v) {
        stack.push_back(&e);
    }
    while (!stack.empty()) {
        const auto *cur = stack.back();
        stack.pop_back();
        if (cur->is_func()) {
            if (cur->fn().kind == func_kind::time) {
                return true;
            }
            if (!seen.insert(cur->fn_id()).second) {
                continue;
            }
            for (const auto &a : cur->fn().args) {
                stack.push_back(&a);
            }
        }
    }
    return false;
}

// ---------------------------------------------------------------------------------------------
// Symbolic differentiation. One rule per func_kind a user expression can contain; shared subexpressions are
// differentiated once (cache on function identity).
// ---------------------------------------------------------------------------------------------
namespace
{

bool is_zero(const expression &e)
{
    return e.is_number() && e.num() == 0.;
}

struct differ {
    const expression &wrt;
    std::unordered_map<const void *, expression> cache;

    expression operator()(const expression &e)
    {
        switch (e.value().index()) {
            case 0:
                return expression{0.};
            case 1:
                return expression{wrt.is_variable() && wrt.var_name() == e.var_name() ? 1. : 0.};
            case 2:
                return expression{wrt.is_param() && wrt.par_idx() == e.par_idx() ? 1. : 0.};
            default:
                break;
        }
        if (const auto it = cache.find(e.fn_id()); it != cache.end()) {
            return it->second;
        }
        auto ret = func_rule(e);
        cache.emplace(e.fn_id(), ret);
        return ret;
    }

    expression func_rule(const expression &e)
    {
        const auto &f = e.fn();
        const auto chain = [&](expression outer) {
            auto d = (*this)(f.args[0]);
            return is_zero(d) ? expression{0.} : prod({std::move(outer), std::move(d)});
        };
        switch (f.kind) {
            case func_kind::sum: {
                std::vector<expression> terms;
                for (const auto &a : f.args) {
                    terms.push_back((*this)(a));
                }
                return sum(std::move(terms));
            }
            case func_kind::prod: {
                // Product rule over all factors: sum_i (prod_{k != i} a_k) * a_i'.
                std::vector<expression> terms;
                for (std::size_t i = 0; i < f.args.size(); ++i) {
                    auto d = (*this)(f.args[i]);
                    if (is_zero(d)) {
                        continue;
                    }
                    auto factors = f.args;
                    factors[i] = std::move(d);
                    terms.push_back(prod(std::move(factors)));
                }
                return sum(std::move(terms));
            }
            case func_kind::pow: {
                const auto &x = f.args[0], &ex = f.args[1];
                std::vector<expression> terms;
                auto dx = (*this)(x);
                if (!is_zero(dx)) {
                    auto em1 = ex.is_number() ? expression{ex.num() - 1.} : sum({ex, expression{-1.}});
                    terms.push_back(prod({ex, pow(x, em1), std::move(dx)}));
                }
                if (!ex.is_number()) {
                    auto de = (*this)(ex);
                    if (!is_zero(de)) {
                        terms.push_back(prod({e, log(x), std::move(de)}));
                    }
                }
                return sum(std::move(terms));
            }
            case func_kind::sin:
                return chain(cos(f.args[0]));
            case func_kind::cos:
                return chain(prod({expression{-1.}, sin(f.args[0])}));
            case func_kind::tanh:
                // 1 - tanh(x)^2.
                return chain(sum({expression{1.}, prod({expression{-1.}, pow(e, expression{2.})})}));
            case func_kind::exp:
                return chain(e);
            case func_kind::log:
                return chain(pow(f.args[0], expression{-1.}));
            case func_kind::sigmoid:
                // sigmoid(x) * (1 - sigmoid(x)).
                return chain(prod({e, sum({expression{1.}, prod({expression{-1.}, e})})}));
            case func_kind::relu:
                // The leaky ReLU's derivative keeps its slope.
                return chain(relup(f.args[0], f.args[1].num()));
            case func_kind::relup:
            case func_kind::time:
                return expression{0.};
            case func_kind::sub:
            case func_kind::div:
            case func_kind::sum_sq:
            case func_kind::num_identity:
                break;
        }
        throw std::invalid_argument(std::string("Cannot differentiate the function '") + func_kind_name(f.kind)
                                    + "': it is created by the Taylor decomposition only");
    }
};

} // namespace

expression diff(const expression &e, const expression &wrt)
{
    if (!wrt.is_variable() && !wrt.is_param()) {
        throw std::invalid_argument("Derivatives can be taken only with respect to a variable or a parameter, not "
                                    "with respect to '"
                                    + to_string(wrt) + "'");
    }
    return differ{wrt, {}}(e);
}

} // namespace heyoka_b200
