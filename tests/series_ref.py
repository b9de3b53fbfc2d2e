"""A high-precision reference for Taylor jets: truncated power series on mpmath (50 digits), and the opcode systems
that tests/test_series_reference.py (oracle, CPU) and tests/test_gpu_coop_shapes.py (device kernels) run against it.

The jet of x' = f(x, p, t) is built from its definition, order by order: x^[n+1] = f(x truncated at degree n)^[n] /
(n + 1), with f evaluated by series arithmetic that shares nothing with the recurrences of the kernels or the oracle:
quotients by long division, log as the integral of a'/a, sin / cos as the imaginary / real part of exp(i a), tanh and
sigmoid as quotients of exponentials, pow(a, alpha) as exp(alpha log a). Only exp is a recurrence (e' = e a').

Every system is written once as a lambda over a backend `m` (like closed_form_cases.py): hb_backend builds the
heyoka_b200 program, mp_backend evaluates the series. Each opcode appears with the operand kinds it accepts (state
variable, u variable, number, parameter); coop_opcodes() lists what a system lowers to, and the tests assert it."""
import mpmath
import numpy as np

import heyoka_b200 as hb

mp = mpmath.MPContext()  # (a context of its own: the global mpmath.mp, which sympy uses, keeps its precision)
mp.dps = 50
mpf = mp.mpf


def order_tol(order):
    """The tolerance that gives a Taylor order: 0 (the default, order 20) for 20, else exp(-2 (order - 1)) nudged up by
    0.1 % so that the rounding of the logarithm cannot change the order (order = ceil(1 - ln(tol) / 2))."""
    return 0. if order == 20 else float(np.exp(-2. * (order - 1)) * 1.001)


# ---- truncated power series -----------------------------------------------------------------------------------------

class Series:
    """Coefficients c[0..d] of a power series truncated at degree d (mpf, or mpc inside sin / cos)."""

    __slots__ = ("c",)

    def __init__(self, c):
        self.c = list(c)

    @property
    def deg(self):
        return len(self.c) - 1

    @staticmethod
    def const(v, deg):
        return Series([mpf(v)] + [mpf(0)] * deg)

    def _lift(self, o):
        return o if isinstance(o, Series) else Series.const(o, self.deg)

    def __add__(self, o):
        o = self._lift(o)
        return Series([a + b for a, b in zip(self.c, o.c)])

    __radd__ = __add__

    def __sub__(self, o):
        o = self._lift(o)
        return Series([a - b for a, b in zip(self.c, o.c)])

    def __rsub__(self, o):
        return self._lift(o) - self

    def __neg__(self):
        return Series([-a for a in self.c])

    def __mul__(self, o):
        o = self._lift(o)
        a, b = self.c, o.c
        return Series([mp.fsum(a[j] * b[k - j] for j in range(k + 1)) for k in range(len(a))])

    __rmul__ = __mul__

    def __truediv__(self, o):
        # Long division: q b = a.
        o = self._lift(o)
        a, b = self.c, o.c
        q = []
        for k in range(len(a)):
            q.append((a[k] - mp.fsum(q[k - j] * b[j] for j in range(1, k + 1))) / b[0])
        return Series(q)

    def __rtruediv__(self, o):
        return self._lift(o) / self

    def deriv(self):
        return Series([k * self.c[k] for k in range(1, len(self.c))] or [mpf(0)])

    def integ(self, c0):
        return Series([c0] + [self.c[k] / (k + 1) for k in range(len(self.c))])


def s_exp(a):
    # e' = e a': k e^[k] = sum_{j=1..k} j a^[j] e^[k-j].
    e = [mp.exp(a.c[0])]
    for k in range(1, len(a.c)):
        e.append(mp.fsum(j * a.c[j] * e[k - j] for j in range(1, k + 1)) / k)
    return Series(e)


def s_log(a):
    if a.deg == 0:
        return Series([mp.log(a.c[0])])
    da = a.deriv()
    return (da / Series(a.c[:-1])).integ(mp.log(a.c[0]))


def s_sqrt(a):
    # s^2 = a, term by term.
    s = [mp.sqrt(a.c[0])]
    for k in range(1, len(a.c)):
        s.append((a.c[k] - mp.fsum(s[j] * s[k - j] for j in range(1, k))) / (2 * s[0]))
    return Series(s)


def s_sincos(a):
    z = s_exp(Series([mp.mpc(0, 1) * c for c in a.c]))
    return Series([mp.im(c) for c in z.c]), Series([mp.re(c) for c in z.c])


def s_tanh(a):
    e2 = s_exp(2 * a)
    return (e2 - 1) / (e2 + 1)


def s_sigmoid(a):
    return 1 / (1 + s_exp(-a))


def s_pow(a, alpha):
    out = s_exp(alpha * s_log(a))
    out.c[0] = mp.power(a.c[0], alpha)
    return out


# ---- backends -------------------------------------------------------------------------------------------------------

class mp_backend:
    """Evaluates a right-hand side on series truncated at degree `deg`, for one lane (its parameters and time)."""

    def __init__(self, deg, pars, t0):
        self.deg, self.pars, self.t0 = deg, [mpf(p) for p in pars], mpf(t0)

    def c(self, v):
        return Series.const(v, self.deg)

    def p(self, i):
        return Series.const(self.pars[i], self.deg)

    def t(self):
        return Series([self.t0, mpf(1)] + [mpf(0)] * (self.deg - 1)) if self.deg else Series([self.t0])

    def sum(self, terms):
        out = self.c(0)
        for x in terms:
            out = out + x
        return out

    def sin(self, a):
        return s_sincos(a)[0]

    def cos(self, a):
        return s_sincos(a)[1]

    def tanh(self, a):
        return s_tanh(a)

    def exp(self, a):
        return s_exp(a)

    def log(self, a):
        return s_log(a)

    def sqrt(self, a):
        return s_sqrt(a)

    def square(self, a):
        return a * a

    def sigmoid(self, a):
        return s_sigmoid(a)

    def pow(self, a, e):
        """e: a number (m.c) or a parameter (m.p): both are constant series here."""
        return s_pow(a, e.c[0])

    def relu(self, a, slope=0.):
        # Gated on the order-0 value of the argument (src/math/relu.cpp).
        if a.c[0] > 0:
            return Series(a.c)
        return Series([mpf(slope) * x for x in a.c])

    def relup(self, a, slope=0.):
        return Series.const(1 if a.c[0] > 0 else slope, self.deg)


class hb_backend:
    """Builds heyoka_b200 expressions."""

    def c(self, v):
        return hb.expression(float(v))

    def p(self, i):
        return hb.par[i]

    def t(self):
        return hb.time

    def sum(self, terms):
        return hb.sum(list(terms))

    def pow(self, a, e):
        return hb.pow(a, e)

    def relu(self, a, slope=0.):
        return hb.relu(a, slope)

    def relup(self, a, slope=0.):
        return hb.relup(a, slope)

    def __getattr__(self, name):
        if name in ("sin", "cos", "tanh", "exp", "log", "sqrt", "square", "sigmoid"):
            return getattr(hb, name)
        raise AttributeError(name)


def series_jet(rhs, x0, pars, t0, order):
    """The jet [n_eq, order + 1] of x' = rhs(m, x) from x(t0) = x0 (one lane), in mpf."""
    X = [[mpf(v)] for v in x0]
    for n in range(order):
        m = mp_backend(n, pars, t0)
        f = rhs(m, [Series(x) for x in X])
        for i, fi in enumerate(f):
            X[i].append((fi.c[n] if isinstance(fi, Series) else (mpf(fi) if n == 0 else mpf(0))) / (n + 1))
    return X


def series_jets(sysdef, state, pars, t0, order):
    """float64 array [n_eq, order + 1, batch] of the reference jets of every lane."""
    batch = state.shape[1]
    t0 = np.broadcast_to(np.asarray(t0, dtype=np.float64), (batch,))
    lanes = [series_jet(sysdef.rhs, state[:, i], pars[:, i] if pars is not None else [], t0[i], order)
             for i in range(batch)]
    out = np.array([[[float(lanes[b][v][o]) for b in range(batch)] for o in range(order + 1)]
                    for v in range(state.shape[0])])
    return out


def normalised_err(tc, ref):
    """max over variables, orders and lanes of |tc - ref| / E(v, o), E(v, o) = max over lanes |ref[v, o]| (no |h|^o
    weight). A coefficient that is 0 in every lane is normalised by the largest coefficient of its variable."""
    E = np.max(np.abs(ref), axis=2, keepdims=True)
    Ev = np.max(np.abs(ref), axis=(1, 2), keepdims=True)
    E = np.where(E > 0, E, np.broadcast_to(Ev, E.shape))
    return float(np.max(np.abs(tc - ref) / E))


# ---- the opcode systems ---------------------------------------------------------------------------------------------

class System:
    """rhs(m, x) -> list of right-hand sides; state(batch, centred) -> [n_eq, batch]; pars(batch) -> [n_pars, batch] or
    None; t0(batch) -> initial times. `ops`: the opcodes (and pow algorithms, as ("POW_VN", algo)) the program must
    contain. `transcendental`: an op whose order-0 value goes through libm (sin, cos, tanh, exp, log, sigmoid, general
    pow, CFUNC): centred initial conditions make those exact, so the all-clamped propagation, which leaves the
    centre, is run only on the other systems. `arrays`: build the program from raw arrays instead (opcodes that the
    symbolic front end does not produce)."""

    def __init__(self, name, n_eq, rhs, state, ops, pars=None, t0=None, transcendental=False, arrays=None):
        self.name, self.n_eq, self.rhs, self._state, self.ops = name, n_eq, rhs, state, ops
        self._pars, self._t0, self.transcendental, self.arrays = pars, t0, transcendental, arrays

    def state(self, batch, centred=True, seed=0):
        return np.ascontiguousarray(self._state(batch, centred, np.random.default_rng(seed)), dtype=np.float64)

    def pars(self, batch):
        return None if self._pars is None else np.ascontiguousarray(self._pars(batch), dtype=np.float64)

    def t0(self, batch):
        return np.zeros(batch) if self._t0 is None else np.asarray(self._t0(batch), dtype=np.float64)

    def hb_sys(self):
        xs = hb.make_vars(*["x%d" % i for i in range(self.n_eq)])
        return [(x, r) for x, r in zip(xs, self.rhs(hb_backend(), list(xs)))]

    def program(self, order):
        if self.arrays is not None:
            return self.arrays(order)
        tol = order_tol(order)
        P = hb.Program(self.hb_sys(), tol=tol)
        assert P.order == order, (self.name, order, P.order)
        return P


def _lin(batch, lo, hi):
    return np.linspace(lo, hi, batch)


def _spread(batch, lo, hi, rng, centred):
    """Lanes that differ by O(1): an even grid over [lo, hi] in a shuffled order (neighbouring lanes differ)."""
    v = _lin(batch, lo, hi)
    return v[rng.permutation(batch)] if not centred else v[::-1].copy()


def _state(rows):
    """rows: per state variable (centred value or None, lo, hi). Centred: the given value in every lane; otherwise
    (and for None) an O(1) spread, rolled by the variable's index so that no lane has every variable at the middle of
    its range."""
    def f(batch, centred, rng):
        out = []
        for k, (c, lo, hi) in enumerate(rows):
            if centred and c is not None:
                out.append(np.full(batch, float(c)))
            else:
                out.append(np.roll(_spread(batch, lo, hi, rng, centred), k))
        return np.array(out)
    return f


def _pow_vp_arrays(order):
    """x0' = pow(x1, par0), x1' = -x0: u2 = POW_VP(u1, par 0), u3 = NEG(u0)."""
    ops = [[19, 1, 0, 0], [7, 0, 0, 0]]
    R = lambda k, i: (k << 30) | i  # noqa: E731
    return hb.Program.from_arrays(2, 4, 1, order, ops, [], [], [R(0, 2), R(0, 3)])


def _vn_arrays(order):
    """x0' = (x0 (x1 - 2.5)) / 3, x1' = x0 / 3: u2 = SUB_VN(u1, c0), u3 = MUL_VV(u0, u2), u4 = DIV_VN(u3, c1),
    u5 = DIV_VN(u0, c1). (The front end folds x - number into a sum and x / number into a product.)"""
    ops = [[3, 1, 0, 0], [8, 0, 2, 0], [14, 3, 1, 0], [14, 0, 1, 0]]
    return hb.Program.from_arrays(2, 6, 0, order, ops, [], [2.5, 3.], [4, 5])


SYSTEMS = [
    # SUB / MUL / DIV in every variant, NEG; operands state variables, u variables, numbers, parameters.
    System("arith", 3,
           lambda m, x: [(x[1] - x[2]) * (m.p(0) - x[1]) + (x[1] - m.c(2.5)) / x[2],
                         m.c(3.) / (x[2] + x[0]) - (x[0] - m.p(1)) * m.c(0.75) + x[0] / m.p(0),
                         m.p(1) / (x[1] * x[0] + m.c(4.)) - m.c(1.5) * x[1] + m.p(0) * x[0] - (m.c(0.5) - x[1] * x[2])
                         - (x[0] - x[1]) / m.c(3.) + (m.p(1) - x[0] * x[1]) * x[2] - (-x[0])],
           _state([(None, -1., 1.), (None, -1.5, 1.5), (None, 1.5, 3.)]),
           {"SUB_VV", "SUB_NV", "SUB_VP", "SUB_PV", "NEG", "MUL_VV", "MUL_NV", "MUL_PV", "DIV_VV", "DIV_NV", "DIV_PV",
            "DIV_VP", "SUM"},
           pars=lambda b: [_lin(b, 1.25, 2.5), _lin(b, -1., 1.)]),
    # SUB_VN and DIV_VN: only reachable from raw arrays.
    System("arith_vn", 2, lambda m, x: [x[0] * (x[1] - m.c(2.5)) / m.c(3.), x[0] / m.c(3.)],
           _state([(None, 0.5, 1.5), (None, -1.5, 1.5)]), {"SUB_VN", "DIV_VN", "MUL_VV"}, arrays=_vn_arrays),
    # SUM with more than 8 terms (split), every operand kind.
    System("long_sum", 2,
           lambda m, x: [m.sum([x[1], m.c(0.5), x[0] * x[1], m.p(0), m.c(-1.25), x[1] * x[1], m.p(1), x[0],
                                m.c(2.), x[0] * x[0] * x[1], m.p(0) * x[1]]),
                         m.sum([-x[0], x[1] * m.c(0.5), m.c(1.), m.p(1) * x[0], x[1] * x[1] * x[0], m.p(0)])],
           _state([(None, -0.5, 0.5), (None, -0.6, 0.6)]), {"SUM", "MUL_VV", "MUL_PV"},
           pars=lambda b: [_lin(b, -0.5, 0.5), _lin(b, 0.25, 0.75)]),
    # SQRT, SQUARE, SUM_SQ (numbers and parameters at order 0).
    System("sqrt_square", 3,
           lambda m, x: [m.sqrt(x[1]) + m.square(x[2]) - m.c(2.),
                         m.sqrt(x[0] * x[2] + m.c(3.)) - m.square(x[0] * x[1]),
                         m.square(x[0]) + m.square(x[1]) + m.square(m.c(0.5)) + m.square(m.p(0)) - m.c(4.)],
           _state([(None, -0.5, 0.5), (None, 1., 2.), (None, -1., 1.)]), {"SQRT", "SQUARE", "SUM_SQ"},
           pars=lambda b: [_lin(b, -1., 1.)]),
    # POW_VN: every order-0 algorithm (small integers and halves of both signs, the general one at a centred base).
    System("pow", 3,
           lambda m, x: [m.pow(x[1], m.c(3.)) - m.pow(x[2], m.c(-2.)) + m.pow(x[0] + m.c(1.), m.c(0.3)),
                         m.pow(x[2], m.c(1.5)) - m.pow(x[1] * x[2] + m.c(2.), m.c(-1.5)),
                         m.pow(x[0] * x[1] + m.c(1.), m.c(-0.7)) - m.pow(x[1] * x[1] + m.c(1.), m.c(2.5))],
           _state([(0., -0.3, 0.3), (None, 0.5, 1.5), (None, 1., 2.)]),
           {("POW_VN", 0), ("POW_VN", 1), ("POW_VN", 2), ("POW_VN", 3), ("POW_VN", 4)}, transcendental=True),
    # POW_VP: only reachable from raw arrays (the front end rewrites pow(x, par) as exp(par log x)).
    System("pow_vp", 2, lambda m, x: [m.pow(x[1], m.p(0)), -x[0]],
           _state([(None, -1., 1.), (1., 0.5, 1.5)]), {"POW_VP", "NEG"}, pars=lambda b: _lin(b, -1.5, 2.5)[None],
           transcendental=True, arrays=_pow_vp_arrays),
    # SIN / COS of a state variable and of a u variable; positions fed by velocities (depth-2 fused propagation).
    System("trig", 4,
           lambda m, x: [x[1], m.c(-2.) * m.sin(x[0]) + m.cos(x[0] * x[2]) * x[3],
                         x[3], m.cos(x[2]) - m.sin(x[0] * x[3]) * x[1]],
           _state([(0., -1., 1.), (None, -1., 1.), (0., -1., 1.), (None, -1.5, 1.5)]), {"SIN", "COS"},
           transcendental=True),
    System("tanh_exp_log", 3,
           lambda m, x: [m.tanh(x[0]) + m.tanh(x[0] * x[1]) * x[2],
                         m.exp(x[0]) - m.exp(x[0] * x[2]) + m.log(x[2]) * x[1],
                         m.log(x[0] * x[1] + m.c(1.)) - x[1]],
           _state([(0., -0.5, 0.5), (None, 0.5, 2.), (1., 0.5, 2.)]), {"TANH", "EXP", "LOG"}, transcendental=True),
    System("sigmoid", 2,
           lambda m, x: [m.sigmoid(x[0]) * x[1] - m.c(0.5), m.sigmoid(x[0] * x[1]) - x[0]],
           _state([(0., -1., 1.), (None, -2., 2.)]), {"SIGMOID"}, transcendental=True),
    # RELU / RELUP, plain and leaky, of state and u variables whose order-0 values are < 0, 0 and > 0 across lanes.
    System("relu", 3,
           lambda m, x: [m.relu(x[1]) + m.relup(x[2], 0.02) * x[1] - x[0],
                         m.relu(x[2], 0.01) - m.relup(x[1]) * x[0] + m.relu(x[0] * x[2]),
                         m.relu(x[0] - x[1], 0.1) * x[1] - m.c(0.25) * x[2]],
           _state([(None, -1., 1.), (None, -1.5, 1.5), (None, -2., 2.)]), {"RELU", "RELUP"}),
    # TIME (per-lane initial times) and CFUNC of parameters (centred: cos(0) = 1, exp(0) = 1).
    System("time_cfunc", 2,
           lambda m, x: [m.t() * x[1] + m.cos(m.p(0)) - x[0] * m.exp(m.p(1)), m.t() - x[0] * x[1]],
           _state([(None, -1., 1.), (None, -1., 1.)]), {"TIME", "CFUNC"},
           pars=lambda b: np.zeros((2, b)), t0=lambda b: _lin(b, -1.5, 2.), transcendental=True),
]

SYSTEMS_BY_NAME = {s.name: s for s in SYSTEMS}

OPNAMES = ["SUM", "SUM_SQ", "SUB_VV", "SUB_VN", "SUB_NV", "SUB_VP", "SUB_PV", "NEG", "MUL_VV", "MUL_NV", "MUL_PV",
           "DIV_VV", "DIV_NV", "DIV_PV", "DIV_VN", "DIV_VP", "SQUARE", "SQRT", "POW_VN", "POW_VP", "SIN", "COS", "TANH",
           "EXP", "LOG", "TIME", "CFUNC", "SIGMOID", "RELU", "RELUP"]


def coop_opcodes(P):
    """The opcodes of a program, with ("POW_VN", algorithm) for each pow by a number."""
    out = set()
    for op in P.ops_array():
        name = OPNAMES[op[0]]
        out.add(name)
        if name == "POW_VN":
            out.add(("POW_VN", int(op[3]) >> 8))
    return out
