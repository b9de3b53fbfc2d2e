// heyoka_b200 — symbolic front end (host side).
//
// A minimal restatement of the part of heyoka's expression system that the batch Taylor
// integrator needs: numbers, variables, runtime parameters and n-ary elementary functions,
// with the same construction-time constant folding as the reference so that the Taylor
// decomposition (decompose.hpp) comes out in the same shape.
//
// Reference (bluescarni/heyoka @ 9c91f71):
//   include/heyoka/expression.hpp            class expression, prime(), make_vars(), par[]
//   src/expression_ops.cpp:45-92             operator- / + / * / / folding rules
//   src/math/sum.cpp:548-601                 sum(): numbers folded, partitioned first
//   src/math/prod.cpp:913-975                prod(): same, with 0/1 special cases
//   src/math/pow.cpp:1024-1062               pow(): x**0, x**1, number**number
#ifndef HEYOKA_B200_EXPRESSION_HPP
#define HEYOKA_B200_EXPRESSION_HPP

#include <array>
#include <cstdint>
#include <functional>
#include <memory>
#include <ostream>
#include <string>
#include <utility>
#include <variant>
#include <vector>

namespace heyoka_b200
{

struct number {
    double v;
};

struct variable {
    std::string name;
};

struct param {
    std::uint32_t idx;
};

// Elementary functions known to the Taylor machinery. Each one maps to one family of device
// recurrences (csrc/program.h opcodes); the reference's equivalent is one func_iface UDF per
// function (include/heyoka/func.hpp:117-147).
enum class func_kind : std::uint8_t {
    sum,          // src/math/sum.cpp
    prod,         // src/math/prod.cpp
    pow,          // src/math/pow.cpp
    sub,          // src/detail/sub.cpp          (created by sum_to_sub only)
    div,          // src/detail/div.cpp          (created by prod_to_div only)
    sum_sq,       // src/detail/sum_sq.cpp       (created by sum_to_sum_sq only)
    sin,          // src/math/sin.cpp
    cos,          // src/math/cos.cpp
    tanh,         // src/math/tanh.cpp
    exp,          // src/math/exp.cpp
    log,          // src/math/log.cpp
    sigmoid,      // src/math/sigmoid.cpp
    relu,         // src/math/relu.cpp (args: x, slope as a number)
    relup,        // src/math/relu.cpp (derivative of the ReLU; args: x, slope as a number)
    time,         // src/math/time.cpp
    num_identity, // src/detail/num_identity.cpp (created by the decomposition only)
};

const char *func_kind_name(func_kind);

class expression;

struct func_node {
    func_kind kind;
    std::vector<expression> args;
};

class expression
{
public:
    using func_ptr = std::shared_ptr<const func_node>;
    using value_type = std::variant<number, variable, param, func_ptr>;

    expression();
    expression(double);
    explicit expression(number);
    explicit expression(variable);
    explicit expression(param);
    explicit expression(std::string);
    explicit expression(func_ptr);
    expression(func_kind, std::vector<expression>);

    const value_type &value() const
    {
        return m_value;
    }

    bool is_number() const
    {
        return m_value.index() == 0;
    }
    bool is_variable() const
    {
        return m_value.index() == 1;
    }
    bool is_param() const
    {
        return m_value.index() == 2;
    }
    bool is_func() const
    {
        return m_value.index() == 3;
    }
    double num() const
    {
        return std::get<number>(m_value).v;
    }
    const std::string &var_name() const
    {
        return std::get<variable>(m_value).name;
    }
    std::uint32_t par_idx() const
    {
        return std::get<param>(m_value).idx;
    }
    const func_node &fn() const
    {
        return *std::get<func_ptr>(m_value);
    }
    // Identity of a function node (used by the traversal caches, like func::get_ptr()).
    const void *fn_id() const
    {
        return std::get<func_ptr>(m_value).get();
    }

private:
    value_type m_value;
};

// Structural comparison and hashing (src/expression_ops.cpp:376-398, std::hash<expression>).
bool operator==(const expression &, const expression &);
bool operator!=(const expression &, const expression &);
std::size_t hash_value(const expression &);
std::ostream &operator<<(std::ostream &, const expression &);
std::string to_string(const expression &);

// Arithmetic (src/expression_ops.cpp).
expression operator+(expression);
expression operator-(const expression &);
expression operator+(const expression &, const expression &);
expression operator-(const expression &, const expression &);
expression operator*(const expression &, const expression &);
expression operator/(const expression &, const expression &);
expression operator+(const expression &, double);
expression operator-(const expression &, double);
expression operator*(const expression &, double);
expression operator/(const expression &, double);
expression operator+(double, const expression &);
expression operator-(double, const expression &);
expression operator*(double, const expression &);
expression operator/(double, const expression &);
expression &operator+=(expression &, const expression &);
expression &operator-=(expression &, const expression &);
expression &operator*=(expression &, const expression &);
expression &operator/=(expression &, const expression &);

// Function builders.
expression sum(std::vector<expression>);
expression prod(std::vector<expression>);
expression pow(const expression &, const expression &);
expression pow(const expression &, double);
expression sqrt(const expression &);
expression square(const expression &);
expression sin(expression);
expression cos(expression);
expression tanh(expression);
expression sigmoid(expression);
// relu(x) / leaky ReLU with a finite, non-negative slope (src/math/relu.cpp:51-60).
expression relu(expression, double slope = 0.);
expression relup(expression, double slope = 0.);
expression exp(expression);
expression log(expression);

// The time variable (include/heyoka/math/time.hpp: `heyoka::time`).
extern const expression time;

// Runtime parameters: par[i] (include/heyoka/param.hpp).
struct par_impl {
    expression operator[](std::uint32_t) const;
};
inline constexpr par_impl par{};

inline namespace literals
{
expression operator""_dbl(long double);
expression operator""_dbl(unsigned long long);
} // namespace literals

// make_vars("x", "v") -> std::array<expression, 2> (include/heyoka/expression.hpp:300-330).
template <typename... Args>
inline auto make_vars(const Args &...strs)
{
    return std::array<expression, sizeof...(Args)>{expression{variable{std::string(strs)}}...};
}

// prime(x) = rhs (include/heyoka/expression.hpp:254-288).
namespace detail
{
struct prime_wrapper {
    expression m_lhs;
    std::pair<expression, expression> operator=(expression) &&;
};
} // namespace detail

detail::prime_wrapper prime(const expression &);

// Helpers used by the decomposition (src/expression_basic.cpp).
std::vector<std::string> get_variables(const expression &);
std::uint32_t get_param_size(const std::vector<expression> &);
bool is_time_dependent(const std::vector<expression> &);

// Symbolic derivative of e with respect to wrt, a variable or a parameter par[i] (heyoka's diff(), restated from
// its documented rules: the reference's source is not in this tree). Every result is built through the folding
// builders sum() / prod() / pow(), so that zeros and ones fold away. The functions that only the decomposition
// creates (sub, div, sum_sq, num_identity) are refused with std::invalid_argument.
expression diff(const expression &e, const expression &wrt);

} // namespace heyoka_b200

namespace std
{
template <>
struct hash<heyoka_b200::expression> {
    size_t operator()(const heyoka_b200::expression &e) const
    {
        return heyoka_b200::hash_value(e);
    }
};
} // namespace std

#endif
