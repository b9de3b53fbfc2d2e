"""Step callbacks: callback.angle_reducer (include/heyoka_b200/callback.hpp, heyoka's
include/heyoka/callback/angle_reducer.hpp).

The semantics are restated from heyoka's documentation; they were not checked against the reference source."""
import ctypes as C

from ._capi import lib, check


def _is_variable(e):
    # d e / d var(repr(e)) is 1 only for the variable of that name (a parameter, a number or a function gives 0).
    from . import diff, expression
    return isinstance(e, expression) and repr(diff(e, expression(repr(e)))) == "1"


def reduce_angles(x):
    """Reduces a contiguous float64 numpy array into [0, 2pi) in place where it is finite (hy_reduce_angles(): the
    arithmetic of the device reduction, with the same bits)."""
    check(lib.hy_reduce_angles(x.ctypes.data_as(C.POINTER(C.c_double)), x.size))


class angle_reducer:
    """Keeps the listed state variables in [0, 2pi) after every step of propagate_*().

    Passed as the callback of propagate_until() / propagate_for() / propagate_grid(), the reduction runs on the device
    inside the propagation loop when the integrator has no events and its kernel supports it. Wrapping the reducer in a
    function hides it: the call then takes the host loop, with the reducer as an ordinary step callback (same bits).
    The reducer is also callable as reducer(ta): it reduces ta.state in place and returns True."""

    def __init__(self, vars):  # noqa: A002 - the reference's argument name
        vars = list(vars)
        if not vars:
            raise ValueError("The list of expressions passed to the constructor of an angle reducer cannot be empty")
        self._names = []
        for v in vars:
            if not _is_variable(v):
                raise ValueError("The list of expressions passed to the constructor of an angle reducer can contain "
                                 "only variables, but the expression '%r' is not a variable" % (v,))
            if repr(v) not in self._names:
                self._names.append(repr(v))

    @property
    def vars(self):
        from . import expression
        return [expression(n) for n in self._names]

    def sv_indices(self, ta):
        """Indices of the listed variables among the state variables of ta (ValueError for one that is not)."""
        idx = []
        for name in self._names:
            if name not in ta._sv_names:
                raise ValueError("The variable '%s' passed to the angle reducer is not a state variable of the "
                                 "integrator" % name)
            idx.append(ta._sv_names.index(name))
        return idx

    def pre_hook(self, ta):
        self.sv_indices(ta)

    def __call__(self, ta):
        for i in self.sv_indices(ta):
            reduce_angles(ta.state[i])
        return True
