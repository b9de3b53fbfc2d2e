"""Event families for the exact-root tests of event detection (tests/test_event_roots_cpu.py on the oracle,
tests/test_gpu_event_roots.py on the device) — TEST INFRASTRUCTURE.

Every family runs on a clock system x' = 1 with a per-lane start x(0) = s, through the normal front end, so the jet
computes the coefficients of the event equations in the usual way. The roots of an event are put in parameters, e.g.
prod_k (x - par[k]). When the event polynomials have degree below p - 1 the norms of orders p and p - 1 are zero and the
step is exactly max_delta_t ("clamped"): no pow() is involved and the device must reproduce the oracle bit for bit.
Families with free steps (non-polynomial events, or degree p) are marked clamped=False.

A family is data: its order (through tol), lanes, initial state, parameters, terminal and non-terminal events, and the
max_delta_t of each step (None: a free step forwards).
"""
import math

import numpy as np

import heyoka_b200 as hb

ANY, POS, NEG = hb.event_direction.any, hb.event_direction.positive, hb.event_direction.negative


def tol_for_order(p):
    """A tolerance that gives Taylor order p (order = ceil(-ln(tol) / 2 + 1), src/taylor_01.cpp)."""
    return math.exp(-2.0 * (p - 1.5))


def _prod(x, factors):
    e = x - factors[0]
    for f in factors[1:]:
        e = e * (x - f)
    return e


class Family:
    def __init__(self, name, order, s, pars, tes=(), ntes=(), mdts=(1.0,), clamped=True):
        """s: [B] start of the clock; pars: [n_pars, B]; tes: [(expr builder, cooldown, direction)];
        ntes: [(expr builder, direction)], builders take (x, par); mdts: per step, a scalar or [B] max_delta_t, None
        for a free step forwards."""
        self.name, self.order = name, order
        self.s = np.atleast_1d(np.asarray(s, dtype=np.float64))
        self.B = self.s.size
        self.pars = None if pars is None else np.asarray(pars, dtype=np.float64).reshape(-1, self.B)
        self.tes, self.ntes, self.mdts, self.clamped = list(tes), list(ntes), list(mdts), clamped

    @property
    def tol(self):
        return tol_for_order(self.order)

    @property
    def n_te(self):
        return len(self.tes)

    @property
    def n_ev(self):
        return len(self.tes) + len(self.ntes)

    @property
    def dirs(self):
        return [d for _, _, d in self.tes] + [d for _, d in self.ntes]

    def build(self, mk, lanes=None):
        """The integrator of this family made by mk (hb.taylor_adaptive_batch or oracle.OracleEventIntegrator), on all
        lanes or on a subset."""
        idx = np.arange(self.B) if lanes is None else np.asarray(lanes)
        x, = hb.make_vars("x")
        sys = [(x, hb.expression(1.0))]
        pars = None if self.pars is None else np.ascontiguousarray(self.pars[:, idx])
        te = [hb.t_event_batch(f(x, hb.par), callback=lambda ta, d_sgn, i: True, cooldown=c, direction=d)
              for f, c, d in self.tes]
        nte = [hb.nt_event_batch(f(x, hb.par), lambda ta, t, d_sgn, i: None, direction=d) for f, d in self.ntes]
        ta = mk(sys, self.s[idx][None, :].copy(), len(idx), pars=pars, tol=self.tol, t_events=te, nt_events=nte)
        assert ta.get_order() == self.order, (self.name, ta.get_order())
        return ta

    def mdt(self, k, lanes=None):
        m = self.mdts[k]
        if m is None:
            return None
        n = self.B if lanes is None else len(lanes)
        m = np.broadcast_to(np.asarray(m, dtype=np.float64), (self.B,))
        return np.ascontiguousarray(m if lanes is None else m[np.asarray(lanes)]).reshape(n)

    def __repr__(self):
        return self.name


def _sorted_roots(rng, K, B, lo, hi, gap):
    """K roots per lane, uniform in (lo, hi), at least gap apart; [K, B]."""
    out = np.empty((K, B))
    for b in range(B):
        while True:
            r = np.sort(rng.uniform(lo, hi, K))
            if K == 1 or np.min(np.diff(r)) >= gap:
                out[:, b] = r
                break
    return out


def _product_event(K):
    return lambda x, par: _prod(x, [par[k] for k in range(K)])


def families():
    rng = np.random.default_rng(20261016)
    F = []
    # K simple roots over two clamped steps of length 1 (degree K <= p - 2 at order 33).
    for K in (1, 2, 3, 5, 8, 12, 16, 20):
        F.append(Family("simple_K%d" % K, 33, np.zeros(4), _sorted_roots(rng, K, 4, 0.03, 1.97, 0.02),
                        ntes=[(_product_event(K), ANY)], mdts=(1.0, 1.0)))
    F.append(Family("simple_K5_backward", 33, np.zeros(4), _sorted_roots(rng, 5, 4, -1.97, -0.03, 0.02),
                    ntes=[(_product_event(5), ANY)], mdts=(-1.0, -1.0)))
    # K = p: degree p, so the step is free (the norm of order p is not zero).
    for p in (20, 33, 47):
        F.append(Family("simple_K%d_order%d_free" % (p, p), p, np.zeros(3), _sorted_roots(rng, p, 3, 0.0, 2.0, 0.005),
                        ntes=[(_product_event(p), ANY)], mdts=(None, None), clamped=False))

    # Chebyshev T_K(2x - 1): roots cos((2j - 1) pi / 2K), clustered at the ends of [0, 1].
    def cheb(K):
        def f(x, par):
            y = 2.0 * x - 1.0
            t0, t1 = hb.expression(1.0), y
            for _ in range(K - 1):
                t0, t1 = t1, 2.0 * y * t1 - t0
            return t1
        return f
    for K in (5, 12):
        F.append(Family("chebyshev_T%d" % K, 20, [0.0, 1e-3, -2e-3], None, ntes=[(cheb(K), ANY)], mdts=(1.0,)))

    # Close pairs (x - r)(x - r - 2^-k), k = 4 .. 52, and a well separated root at 0.8; one lane per k.
    ks = np.arange(4, 53, 4)
    F.append(Family("close_pairs", 20, np.zeros(len(ks)),
                    np.stack([np.full(len(ks), 0.3), 0.3 + 2.0 ** -ks.astype(float), np.full(len(ks), 0.8)]),
                    ntes=[(_product_event(3), ANY)], mdts=(1.0,)))
    # Multiple roots: a double, a triple, two doubles; each with a simple root for the completeness check.
    mp_ = np.array([[0.3, 0.45, 0.61], [0.5, 0.2, 0.37], [0.7, 0.66, 0.12], [0.9, 0.85, 0.93]])
    F.append(Family("multiple_roots", 20, np.zeros(3), mp_,
                    ntes=[(lambda x, par: (x - par[0]) * (x - par[0]) * (x - par[3]), ANY),
                          (lambda x, par: (x - par[1]) * (x - par[1]) * (x - par[1]) * (x - par[3]), ANY),
                          (lambda x, par: (x - par[0]) * (x - par[0]) * (x - par[2]) * (x - par[2]) * (x - par[3]),
                           ANY)], mdts=(1.0,)))
    # A root exactly at the start of the step (x(0) = par[0]: the constant coefficient is exactly zero).
    s0 = np.array([0.0, 0.25, -0.5, 3.0])
    F.append(Family("root_at_start", 20, s0, np.stack([s0, s0 + 0.6]), ntes=[(_product_event(2), ANY)],
                    mdts=(1.0, 1.0)))
    # A root exactly at h, one ulp inside and one ulp outside; x - 0.5 for the completeness check.
    ends = np.array([1.0, np.nextafter(1.0, 0.0), np.nextafter(1.0, 2.0)])
    F.append(Family("root_at_end", 20, np.zeros(3), ends[None, :],
                    ntes=[(lambda x, par: x - 0.5, ANY), (lambda x, par: x - par[0], ANY)], mdts=(1.0, 1.0)))
    # The clamp of a root that lands on or past h to nextafter(h, 0) (ev_kernels.cuh:463). For a normal h it cannot
    # run: the root finder returns tau <= 1 - 2^-53 and fl(tau h) < |h|. On a subnormal step it can: h = 2^-1030 is
    # 2^44 units of 2^-1074, 3x - par[0] with par[0] = 3h - 2^-1074 has its root a third of a unit below h, so
    # fl(tau h) = h and the record is moved to nextafter(h, 0). x - par[1] (= h / 2) is the well-conditioned root.
    hs = 2.0 ** -1030
    F.append(Family("root_clamped_to_h", 10, np.zeros(2), np.array([[3.0 * hs - 5e-324] * 2, [hs / 2] * 2]),
                    ntes=[(lambda x, par: 3.0 * x - par[0], ANY), (lambda x, par: x - par[1], ANY)], mdts=(hs,)))
    # Non-polynomial events: their top coefficients are not zero; free steps, then steps clamped at 0.05.
    s4 = np.array([0.0, 0.1, 0.2, 0.3])
    nonpoly = [(lambda x, par: hb.sin(10.0 * x), ANY), (lambda x, par: hb.exp(x) - 1.5, ANY)]
    F.append(Family("nonpolynomial_free", 20, s4, None, ntes=nonpoly, mdts=(None,) * 3, clamped=False))
    F.append(Family("nonpolynomial_short", 20, s4, None, ntes=nonpoly, mdts=(0.05,) * 2, clamped=False))
    # Directions, terminal and non-terminal events together, two identical terminal events (the smaller index wins).
    mx = _sorted_roots(rng, 5, 5, 0.05, 2.9, 0.1)
    A = lambda x, par: (x - par[0]) * (x - par[1]) * (x - par[2])  # noqa: E731
    Bq = lambda x, par: (x - par[3]) * (x - par[4])  # noqa: E731
    F.append(Family("mixed_directions", 20, np.zeros(5), mx, tes=[(A, -1.0, POS), (A, -1.0, POS)],
                    ntes=[(Bq, NEG), (Bq, ANY), (A, ANY)], mdts=(1.0,) * 5))
    # Cooldowns: a terminal event with cooldown c = 0.2 at t1, then roots at t1 + c / 2 (suppressed) and t1 + 2c
    # (reported); forwards and backwards, the cooldown boundary inside the next step.
    t1 = np.array([0.2, 0.3, 0.45])
    cdf = lambda x, par: (x - par[0]) * (x - par[1]) * (x - par[2])  # noqa: E731
    F.append(Family("cooldown_forward", 20, np.zeros(3), np.stack([t1, t1 + 0.1, t1 + 0.4]),
                    tes=[(cdf, 0.2, ANY)], ntes=[(lambda x, par: x - par[1], ANY)], mdts=(1.0,) * 4))
    F.append(Family("cooldown_backward", 20, np.zeros(3), -np.stack([t1, t1 + 0.1, t1 + 0.4]),
                    tes=[(cdf, 0.2, ANY)], ntes=[(lambda x, par: x - par[1], ANY)], mdts=(-1.0,) * 4))
    # The automatic cooldown: after the terminal event the next step starts on (or next to) the root.
    # (x - 0.1: a non-terminal root before the terminal one, for the completeness check.)
    F.append(Family("cooldown_automatic", 20, np.zeros(3), np.stack([t1, t1 + 0.3]), tes=[(_product_event(2), -1.0, ANY)],
                    ntes=[(lambda x, par: x - 0.1, ANY)], mdts=(1.0,) * 4))
    # Orders 3, 4, 10, 40 (degree <= p - 2) and 47 (the 20-root calibration case).
    for p, K in ((3, 1), (4, 2), (10, 4), (40, 8)):
        F.append(Family("order%d" % p, p, np.zeros(2), _sorted_roots(rng, K, 2, 0.03, 1.97, 0.05),
                        ntes=[(_product_event(K), ANY)], mdts=(1.0, 1.0)))
    F.append(Family("order47_K20", 47, np.zeros(3), _sorted_roots(rng, 20, 3, 0.05, 0.95, 0.01),
                    ntes=[(_product_event(20), ANY)], mdts=(1.0,)))
    return F


def overflow_family(B=64):
    """More records in one step than the device's record array holds (max(B n_ev, 1024)): B lanes of a 20-root
    non-terminal event, roots well spread over the step."""
    rng = np.random.default_rng(5)
    return Family("record_overflow", 33, np.zeros(B), _sorted_roots(rng, 20, B, 0.02, 0.98, 0.02),
                  ntes=[(_product_event(20), ANY)], mdts=(1.0,))


def many_candidates_family(B=8500):
    """More (event, lane) candidates than the detection kernel has threads (64 x 132 on an H100), so its threads loop."""
    rng = np.random.default_rng(6)
    return Family("many_candidates", 10, np.zeros(B), rng.uniform(0.05, 0.95, (1, B)),
                  ntes=[(_product_event(1), ANY)], mdts=(1.0,))


def sample_lanes(B, n=2):
    """At most n lanes, the first and the last included (the exact reference costs milliseconds per polynomial)."""
    return sorted(set(np.linspace(0, B - 1, min(n, B)).round().astype(int).tolist()))


def against_exact_roots(fam, ta, cd, lanes):
    """Check the records of the step just taken against the exact roots of the event polynomials the integrator
    reports (root_ref.check()), for the given lanes. The window of a lane is [0, last_h): the step, or the part of it
    before the terminal event that cut it (non-terminal events past it are not reported, and a terminal root before it
    would have cut the step earlier). Returns (problems, notes, findings, number of well-conditioned roots checked)."""
    import root_ref
    evs = ta._b.events()
    tce = ta._b.tc_events(fam.n_ev)
    h = ta.last_h
    problems, notes, findings, n_well = [], [], [], 0
    for lane in lanes:
        if h[lane] == 0 or not np.isfinite(h[lane]):
            continue
        for k in range(fam.n_ev):
            term = k < fam.n_te
            idx = k if term else k - fam.n_te
            recs = [(e[4], e[3]) for e in evs if e[0] == lane and e[2] == term and e[1] == idx]
            roots = root_ref.exact_roots(tce[k, :, lane], h[lane])
            cut = root_ref.cooldown_cut(h[lane], cd[0][k, lane], cd[1][k, lane], cd[2][k, lane]) if term else 0.0
            pr, no, fi, nw = root_ref.check(recs, roots, h[lane], fam.dirs[k], cut)
            where = "%s lane %d event %d (%s): " % (fam.name, lane, k, "terminal" if term else "non-terminal")
            problems += [where + s for s in pr]
            notes += [where + s for s in no]
            findings += [where + s for s in fi]
            n_well += nw
    return problems, notes, findings, n_well


def run(fam, mk, lanes=None, on_step=None):
    """Step the family's integrator through its steps. on_step(k, ta, cd_before, mdt) after every step, cd_before the
    cooldown state (active, spent, cooldown) [n_te, B] the step started from."""
    ta = fam.build(mk, lanes)
    for k in range(len(fam.mdts)):
        cd = ta._b.cooldowns(fam.n_te) if fam.n_te else None
        m = fam.mdt(k, lanes)
        ta.step(max_delta_ts=m)
        if on_step is not None:
            on_step(k, ta, cd, m)
    return ta
