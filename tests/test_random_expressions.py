"""Random right-hand sides (seeded): the jet computed by decomposition + lowering + oracle against jets obtained by
symbolic differentiation along the flow (sympy, 30 digits). Pins the host pipeline (expression folding, Taylor
decomposition, CSE, lowering) and every recurrence of the oracle on compositions the fixed fixtures do not cover.
The generator keeps arguments inside the domain of log / sqrt / pow / division. CPU only."""
import numpy as np
import pytest
import sympy as sp

import heyoka_b200 as hb
import oracle

ORDER, TOL = 4, 0.0025  # tol -> order 4 (ceil(-ln(tol) / 2 + 1))


class Gen:
    def __init__(self, seed):
        self.rng = np.random.default_rng(seed)

    def const(self):
        return float(self.rng.choice([-2.5, -1.25, -0.5, 0.75, 1.5, 3.0]))

    def expr(self, depth, leaves):
        """Returns (hb expression, sympy expression)."""
        r = self.rng
        if depth == 0 or r.random() < 0.15:
            k = int(r.integers(len(leaves)))
            return leaves[k]
        kind = r.choice(["add", "sub", "mul", "div", "sin", "cos", "tanh", "exp", "log", "sqrt", "square", "pow",
                         "sigmoid", "neg", "cmul"])
        a, sa = self.expr(depth - 1, leaves)
        if kind in ("add", "sub", "mul", "div"):
            b, sb = self.expr(depth - 1, leaves)
            if kind == "add":
                return a + b, sa + sb
            if kind == "sub":
                return a - b, sa - sb
            if kind == "mul":
                return a * b, sa * sb
            return a / (2.5 + hb.sin(b)), sa / (sp.Rational(5, 2) + sp.sin(sb))  # denominator in [1.5, 3.5]
        if kind == "sin":
            return hb.sin(a), sp.sin(sa)
        if kind == "cos":
            return hb.cos(a), sp.cos(sa)
        if kind == "tanh":
            return hb.tanh(a), sp.tanh(sa)
        if kind == "exp":
            return hb.exp(hb.tanh(a)), sp.exp(sp.tanh(sa))  # bounded argument
        if kind == "log":
            return hb.log(2.0 + hb.cos(a)), sp.log(2 + sp.cos(sa))
        if kind == "sqrt":
            return hb.sqrt(3.0 + hb.sin(a)), sp.sqrt(3 + sp.sin(sa))
        if kind == "square":
            return hb.square(a), sa ** 2
        if kind == "pow":
            e = float(r.choice([-1.5, -0.5, 1.5, 3.0, -2.0, 0.3]))
            return hb.pow(2.0 + hb.tanh(a), e), (2 + sp.tanh(sa)) ** sp.nsimplify(e)
        if kind == "sigmoid":
            return hb.sigmoid(a), 1 / (1 + sp.exp(-sa))
        if kind == "neg":
            return -a, -sa
        c = self.const()
        return c * a, sp.nsimplify(c) * sa


def sympy_jet(rhs, syms, ic, order):
    derivs = [list(syms), list(rhs)]
    for _ in range(2, order + 1):
        derivs.append([sum(sp.diff(e, s) * f for s, f in zip(syms, rhs)) for e in derivs[-1]])
    subs = {s: sp.nsimplify(v) for s, v in zip(syms, ic)}
    return np.array([[float(sp.N(derivs[k][i].subs(subs) / sp.factorial(k), 30)) for k in range(order + 1)]
                     for i in range(len(syms))])


def build_case(seed):
    g = Gen(1000 + seed)
    n_eq = 2 + seed % 2
    hvars = hb.make_vars(*["x%d" % i for i in range(n_eq)])
    svars = sp.symbols("x0:%d" % n_eq)
    leaves = list(zip(hvars, svars))
    rhs = [g.expr(3, leaves) for _ in range(n_eq)]
    sys_ = [(hvars[i], rhs[i][0]) for i in range(n_eq)]
    ic = g.rng.uniform(-1.0, 1.0, (n_eq, 3)).round(3)
    return sys_, [r[1] for r in rhs], svars, ic


@pytest.mark.gpu
@pytest.mark.parametrize("seed", range(16))
def test_random_rhs_gpu_against_oracle(seed):
    """The same random systems on the GPU (the automatic kernel, the HBM-tape kernel and the cooperative kernel with
    its tape in global memory): one step with write_tc and a short propagation against the oracle (no sympy on this
    path: the oracle is pinned on the CPU)."""
    sys_, _, _, ic = build_case(seed)
    P = hb.Program(sys_, tol=1e-12)
    for kernel in (dict(tape="auto"), dict(tape="hbm"), dict(tape="global")):
        ta = hb.taylor_adaptive_batch(sys_, ic, 3, tol=1e-12, kernel=kernel)
        o = oracle.OracleIntegrator(P, ic, 3, mode=oracle.FMA)
        ta.step(write_tc=True)
        o.step(write_tc=True)
        w = np.abs(o.last_h)[None, None, :] ** np.arange(P.order + 1)[None, :, None]
        scale = np.maximum(np.max(np.abs(o.tc[:, 0, :]), axis=0), 1.0)[None, None, :]
        assert np.max(np.abs(ta.tc - o.tc) * w / scale) < 1e-12, (seed, kernel)
        assert np.max(np.abs(ta.last_h / o.last_h - 1)) < 1e-10
        ta.propagate_until(0.5)
        o.propagate_until(0.5)
        assert [r[3] for r in ta.propagate_res] == [int(x) for x in o.n_steps], (seed, kernel)
        assert np.max(np.abs(ta.state - o.state) / np.maximum(np.abs(o.state), 1.0)) < 1e-11, (seed, kernel)


@pytest.mark.parametrize("seed", range(16))
def test_random_rhs_against_symbolic_jets(seed):
    sys_, srhs, svars, ic = build_case(seed)
    n_eq = len(svars)
    P = hb.Program(sys_, tol=TOL)
    assert P.order == ORDER
    batch = 3
    expected = np.stack([sympy_jet(srhs, svars, ic[:, lane], ORDER) for lane in range(batch)], axis=2)
    scale = np.maximum(np.max(np.abs(expected), axis=(0, 2)), 1.0)  # per order
    for mode in (oracle.PAIRWISE, oracle.SEQ, oracle.FMA):
        o = oracle.OracleIntegrator(P, ic, batch, mode=mode)
        o.step(write_tc=True)
        err = np.max(np.abs(o.tc - expected) / scale[None, :, None])
        assert err < 2e-13, (seed, mode, err, P.dc_str())
