"""Variational equations of order 1 on the CPU: symbolic differentiation (hb.diff) against sympy, the structure and
right-hand sides of hb.var_ode_sys, and variational systems integrated by the oracle against closed forms, det(Phi)
and central differences. The device paths are in test_gpu_variational.py."""
import numpy as np
import pytest
import sympy as sp

import heyoka_b200 as hb
import oracle
from test_random_expressions import Gen


def eval_rhs(sys_, state, pars=None):
    """Right-hand sides of sys_ at one point (one lane): the order-1 Taylor coefficients of the state variables in the
    oracle's jet."""
    P = hb.Program(sys_, tol=1e-3)
    st = np.asarray(state, dtype=np.float64).reshape(P.n_eq, 1)
    pr = None if pars is None else np.asarray(pars, dtype=np.float64).reshape(-1, 1)
    return oracle.jet(P, st, pars=pr)[1, :P.n_eq]


def close(got, want, rtol=1e-13):
    got, want = np.asarray(got, dtype=float), np.asarray(want, dtype=float)
    return np.all(np.abs(got - want) <= rtol * np.maximum(np.abs(want), 1.0))


# ---- hb.diff ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(16))
def test_diff_random_expressions_against_sympy(seed):
    g = Gen(5000 + seed)
    hv = hb.make_vars("x0", "x1")
    sv = sp.symbols("x0:2")
    sp0 = sp.Symbol("p0")
    e, se = g.expr(4, list(zip(hv, sv)) + [(hb.par[0], sp0)])
    z = hb.expression("z")
    derivs = [hb.diff(e, hv[0]), hb.diff(e, hv[1]), hb.diff(e, hb.par[0])]
    sys_ = [(hv[0], derivs[0]), (hv[1], derivs[1]), (z, derivs[2])]
    for _ in range(3):
        pt = g.rng.uniform(-1.0, 1.0, 3)
        got = eval_rhs(sys_, [pt[0], pt[1], 0.0], pars=[pt[2]])
        subs = {sv[0]: pt[0], sv[1]: pt[1], sp0: pt[2]}
        want = [float(sp.N(sp.diff(se, s).subs(subs), 30)) for s in (sv[0], sv[1], sp0)]
        assert close(got, want), (seed, repr(e), got, want)


def test_diff_identities():
    x, y = hb.make_vars("x", "y")
    assert repr(hb.diff(x, x)) == "1"
    assert repr(hb.diff(x, y)) == "0"
    assert repr(hb.diff(hb.par[0], hb.par[0])) == "1"
    assert repr(hb.diff(hb.par[0], hb.par[1])) == "0"
    assert repr(hb.diff(hb.par[0], x)) == "0"
    assert repr(hb.diff(hb.time, x)) == "0"
    assert repr(hb.diff(3.5, x)) == "0"
    # Zeros and ones fold away.
    assert repr(hb.diff(x * y, x)) == "y"
    assert repr(hb.diff(hb.sin(y), x)) == "0"
    assert repr(hb.diff(hb.cos(x), x)) == "prod(-1, sin(x))"
    assert repr(hb.diff(hb.relu(x, 0.25), x)) == repr(hb.relup(x, 0.25))
    assert repr(hb.diff(hb.relup(x), x)) == "0"


def test_diff_refusals():
    x = hb.make_vars("x")[0]
    for wrt in (hb.expression(1.0), hb.sin(x), hb.time):
        with pytest.raises(ValueError):
            hb.diff(x, wrt)


def test_diff_functions_against_sympy():
    """One closed check per rule, including the non-numeric exponent of pow and the leaky ReLU."""
    x, y = hb.make_vars("x", "y")
    sx, sy = sp.symbols("x y")
    cases = [(hb.pow(x, y), sx ** sy), (hb.tanh(x * y), sp.tanh(sx * sy)), (hb.sigmoid(x), 1 / (1 + sp.exp(-sx))),
             (hb.log(x) * hb.exp(y), sp.log(sx) * sp.exp(sy)), (hb.sin(x) * hb.cos(y) * x, sp.sin(sx) * sp.cos(sy) * sx),
             (hb.sqrt(x + y), sp.sqrt(sx + sy))]
    pt = {sx: 0.7, sy: 1.3}
    for e, se in cases:
        sys_ = [(x, hb.diff(e, x)), (y, hb.diff(e, y))]
        got = eval_rhs(sys_, [0.7, 1.3])
        want = [float(sp.diff(se, s).subs(pt)) for s in (sx, sy)]
        assert close(got, want), (repr(e), got, want)
    r = hb.relu(x, 0.25)
    for v, want in ((0.7, 1.0), (-0.7, 0.25)):
        assert eval_rhs([(x, hb.diff(r, x))], [v])[0] == want


# ---- hb.var_ode_sys -----------------------------------------------------------------------------------------------
def osc_sys():
    x, v = hb.make_vars("x", "v")
    return [(x, v), (v, -hb.par[0] ** 2 * x)], (x, v)


def test_var_ode_sys_structure():
    sys_, (x, v) = osc_sys()
    cases = [(hb.var_args.vars, ["x", "v"]), (hb.var_args.params, ["p0"]),
             (hb.var_args.vars | hb.var_args.params, ["x", "v", "p0"]), ([hb.par[0], v], ["p0", "v"])]
    for args, want in cases:
        vs = hb.var_ode_sys(sys_, args)
        m = len(want)
        assert [repr(a) for a in vs.vargs] == want
        assert vs.n_orig_sv == 2 and vs.order == 1 and len(vs.sys) == 2 * (1 + m)
        names = [repr(p[0]) for p in vs.sys]
        assert names == ["x", "v"] + ["∂[(%d, 1)]%s" % (j, c) for c in ("x", "v") for j in range(m)]
        assert hb.Program(vs).n_eq == 2 * (1 + m)


def test_var_ode_sys_rhs_against_sympy():
    g = Gen(77)
    hv = hb.make_vars("x0", "x1")
    sv = sp.symbols("x0:2")
    sps = sp.symbols("p0:2")
    leaves = list(zip(hv, sv)) + [(hb.par[0], sps[0]), (hb.par[1], sps[1])]
    f = [g.expr(3, leaves) for _ in range(2)]
    sys_ = [(hv[i], f[i][0]) for i in range(2)]
    for args, sargs in ((hb.var_args.vars | hb.var_args.params, list(sv) + list(sps)),
                        ([hb.par[1], hv[1], hb.par[0]], [sps[1], sv[1], sps[0]])):
        vs = hb.var_ode_sys(sys_, args)
        n, m = 2, len(sargs)
        for _ in range(3):
            x = g.rng.uniform(-1, 1, n)
            phi = g.rng.uniform(-1, 1, (n, m))
            p = g.rng.uniform(-1, 1, 2)
            got = eval_rhs(vs.sys, np.concatenate([x, phi.ravel()]), pars=p)
            subs = dict(zip(sv, x)) | dict(zip(sps, p))
            J = np.array([[float(sp.diff(f[i][1], sv[k]).subs(subs)) for k in range(n)] for i in range(n)])
            dfa = np.array([[float(sp.diff(f[i][1], a).subs(subs)) if a in sps else 0.0 for a in sargs]
                            for i in range(n)])
            want = np.concatenate([[float(f[i][1].subs(subs)) for i in range(n)], (J @ phi + dfa).ravel()])
            assert close(got, want, 1e-12), (got, want)


def test_var_ode_sys_drops_zero_partials():
    """N-body: d(xdot)/dx = 0, so the variational rows of the positions are sums of velocity sensitivities only."""
    vs = hb.var_ode_sys(hb.model.nbody(2), hb.var_args.vars)
    assert len(vs.sys) == 12 * 13
    # d/dt dx0/da_j = dvx0/da_j: a single variable, no products with zero.
    assert repr(vs.sys[12][1]) == "∂[(0, 1)]vx_0"


def test_var_ode_sys_refusals():
    sys_, (x, v) = osc_sys()
    with pytest.raises(ValueError):
        hb.var_ode_sys(sys_, hb.var_args.vars, order=0)
    with pytest.raises(NotImplementedError):
        hb.var_ode_sys(sys_, hb.var_args.vars, order=2)
    with pytest.raises(NotImplementedError):
        hb.var_ode_sys(sys_, hb.var_args.vars | hb.var_args.time)
    with pytest.raises(NotImplementedError):
        hb.var_ode_sys(sys_, [x, hb.time])
    with pytest.raises(ValueError):
        hb.var_ode_sys(sys_, [])
    with pytest.raises(ValueError):
        hb.var_ode_sys(sys_, [x, v, x])
    with pytest.raises(ValueError):
        hb.var_ode_sys(sys_, [x, hb.expression("w")])
    with pytest.raises(ValueError):
        hb.var_ode_sys(sys_, [x, hb.sin(v)])
    with pytest.raises(ValueError):  # no parameters in the pendulum: an empty argument set
        hb.var_ode_sys(hb.model.pendulum(), hb.var_args.params)
    # A generated name that collides with a variable of the system.
    y = hb.expression("∂[(0, 1)]x")
    with pytest.raises(ValueError):
        hb.var_ode_sys([(x, y), (y, -x)], hb.var_args.vars)


def test_initial_state_fill():
    """The constructor's fill: per lane, STM column j is e_k for the argument x_k, 0 for a parameter (2 x 3 here, so
    that a fill by rows differs)."""
    sys_, (x, v) = osc_sys()
    vs = hb.var_ode_sys(sys_, [v, hb.par[0], x])
    st = np.array([[1.0, 2.0], [3.0, 4.0]])
    full = hb._var_initial_state(vs, st, 2)
    phi = full[2:].reshape(2, 3, 2)
    want = np.array([[0, 0, 1], [1, 0, 0]], dtype=float)
    assert np.array_equal(full[:2], st)
    for lane in range(2):
        assert np.array_equal(phi[:, :, lane], want)
    assert np.array_equal(hb._var_initial_state(vs, np.zeros(0), 2)[:2], np.zeros((2, 2)))


# ---- the oracle on variational systems ----------------------------------------------------------------------------
def osc_closed_form(x0, v0, w, t):
    c, s = np.cos(w * t), np.sin(w * t)
    x = x0 * c + v0 / w * s
    v = -x0 * w * s + v0 * c
    phi = np.array([[c, s / w, -x0 * t * s + v0 * (t * c / w - s / w ** 2)],
                    [-w * s, c, -x0 * (s + w * t * c) - v0 * t * s]])
    return np.array([x, v]), phi


def osc_state(lanes):
    x0 = np.linspace(0.3, 1.1, lanes)
    v0 = np.linspace(-0.5, 0.4, lanes)
    w = np.linspace(0.8, 1.7, lanes)
    return x0, v0, w


def test_oracle_oscillator_closed_form():
    sys_, (x, v) = osc_sys()
    vs = hb.var_ode_sys(sys_, [x, v, hb.par[0]])
    P = hb.Program(vs)
    x0, v0, w = osc_state(4)
    st = hb._var_initial_state(vs, np.stack([x0, v0]), 4)
    o = oracle.OracleIntegrator(P, st, 4, pars=w[None, :])
    o.propagate_until(3.0)
    for lane in range(4):
        xs, phi = osc_closed_form(x0[lane], v0[lane], w[lane], 3.0)
        assert close(o.state[:2, lane], xs, 1e-12)
        assert close(o.state[2:, lane].reshape(2, 3), phi, 1e-12), (o.state[2:, lane].reshape(2, 3), phi)


def three_body_state(lanes):
    base = np.array([1.0, 0, 0, 0, 0.9, 0.05, -0.5, 0.866, 0, -0.78, -0.45, 0, -0.5, -0.866, 0.1, 0.78, -0.45, 0])
    return base[:, None] + 1e-3 * np.arange(lanes)[None, :]


def flow_cases():
    return [("pendulum", hb.model.pendulum(), np.array([[0.4, 1.0, -0.3], [0.1, 0.0, 0.5]]), 3.0),
            ("3body", hb.model.nbody(3), three_body_state(2), 1.0)]


@pytest.mark.parametrize("case", [c[0] for c in flow_cases()])
def test_oracle_det_phi_and_central_differences(case):
    name, sys_, x0, tf = next(c for c in flow_cases() if c[0] == case)
    n, lanes = x0.shape
    vs = hb.var_ode_sys(sys_, hb.var_args.vars)
    o = oracle.OracleIntegrator(hb.Program(vs), hb._var_initial_state(vs, x0, lanes), lanes)
    o.propagate_until(tf)
    phis = [o.state[n:, lane].reshape(n, n) for lane in range(lanes)]
    for phi in phis:
        assert abs(np.linalg.det(phi) - 1.0) < 1e-9, np.linalg.det(phi)
    # Central differences from perturbed initial conditions (one lane per perturbation, no variational equations).
    P = hb.Program(sys_)
    errs = []
    for delta in (1e-3, 5e-4):
        st = np.concatenate([x0[:, :1] + s * delta * np.eye(n) for s in (1.0, -1.0)], axis=1)
        op = oracle.OracleIntegrator(P, st, 2 * n)
        op.propagate_until(tf)
        fd = (op.state[:, :n] - op.state[:, n:]) / (2 * delta)
        errs.append(np.max(np.abs(fd - phis[0])))
    assert errs[0] < 1e-4, errs
    assert 3.0 < errs[0] / errs[1] < 5.0, errs  # O(delta^2)
