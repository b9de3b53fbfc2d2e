// heyoka_b200 — callback::angle_reducer: heyoka's built-in step callback (include/heyoka/callback/angle_reducer.hpp,
// src/callback/angle_reducer.cpp) that keeps a list of angular state variables in [0, 2pi) after every step of
// propagate_*().
//
// The semantics are restated from heyoka's documentation; they were not checked against the reference source:
//   - constructed from a non-empty list of variables (a variable listed twice is reduced once); an empty list or an
//     expression that is not a variable: std::invalid_argument;
//   - at the start of every propagate_for() / propagate_until() / propagate_grid() (the reference's pre_hook()), every
//     listed variable must be a state variable of the integrator, else std::invalid_argument naming it, before any
//     step; the state is not reduced there;
//   - after every step of propagate_*(), where the reference calls the step callback (after the continuous-output
//     recording and the dense output of the grid points the step covers), every listed variable that is finite and
//     outside [0, 2pi) is replaced by x - 2pi * floor(x / 2pi) (2pi the nearest double, with fix-ups so that the
//     result is in [0, 2pi)); non-finite values are left alone. The callback returns true. step() never reduces.
//
// taylor_adaptive_batch<double> recognises the reducer passed as kw::callback (std::function::target()) and, when the
// integrator has no events and its kernel supports it, runs the reduction on the device inside the propagation loop
// (hy_batch_set_angles()) instead of calling back to the host after every step. Wrapping the reducer in a lambda
// hides its type: the call then takes the host loop, with the reducer as an ordinary step callback, and gives the same
// bits.
#ifndef HEYOKA_B200_CALLBACK_HPP
#define HEYOKA_B200_CALLBACK_HPP

#include <cstdint>
#include <vector>

#include <heyoka_b200/expression.hpp>

namespace heyoka_b200
{

template <typename T>
class taylor_adaptive_batch;

namespace callback
{

class angle_reducer
{
    std::vector<expression> m_vars;

public:
    explicit angle_reducer(std::vector<expression> vars);

    // Reduces the listed state variables of every lane; returns true.
    bool operator()(taylor_adaptive_batch<double> &) const;
    // Checks that every listed variable is a state variable of the integrator.
    void pre_hook(taylor_adaptive_batch<double> &) const;

    // The listed variables, without repetitions, in the order first given.
    [[nodiscard]] const std::vector<expression> &get_vars() const noexcept;
    // Their indices among the state variables of the integrator (std::invalid_argument for a variable that is not one).
    [[nodiscard]] std::vector<std::uint32_t> get_sv_indices(const taylor_adaptive_batch<double> &) const;
};

} // namespace callback

} // namespace heyoka_b200

#endif
