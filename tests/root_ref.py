"""Exact real roots of an event polynomial inside a step — TEST INFRASTRUCTURE.

The event detection of the device (csrc/ev_kernels.cuh) and of the oracle (oracle/taylor_oracle.c) looks for the roots
of p(t) = a_0 + a_1 t + ... + a_p t^p, the Taylor polynomial of an event equation over one step, in [0, h) (forwards)
or (h, 0] (backwards). Both restate the same algorithm, so agreeing with each other says nothing about a misreading they
share. This module answers the same question exactly: the coefficients, as the integrator reports them (tc_events()),
are turned into rationals, and the real roots of that rational polynomial are isolated with sympy and refined to 45
digits. Their multiplicities come from the square-free factorisation.

Tolerance of a reported time (derivation). Let q(tau) = sum_i a_i h^i tau^i be the polynomial on [0, 1) that the root
finder works on, tau* = t*/h the exact root, u = 2^-53 and gamma_n = n u / (1 - n u).
  - Rescaling: q_i is computed as a_i * fl(h^i), fl(h^i) by i - 1 products. |fl(q_i) - q_i| <= gamma_{p+1} |q_i|.
  - Horner over p terms at tau: |fl(q)(tau) - fl(q(tau))| <= gamma_{2p} sum |fl(q_i)| tau^i.
  So the computed value differs from q(tau) by at most gamma_{3p+1} S(tau), S(tau) = sum |a_i h^i| tau^i: wherever
  |q(tau)| exceeds that, the computed sign is the true sign. The root finder (TOMS 748) ends on a bracket [a, b] whose
  computed values change sign (or vanish at a), so the bracket is within gamma_{3p+1} S / |q'(tau*)| of tau* to first
  order. For a root of multiplicity m the first-order term is the m-th: (gamma_{3p+1} S / |q^(m)(tau*) / m!|)^(1/m).
  - Termination: |b - a| <= 4 eps min(|a|, |b|) (eps = 2^-52), so the midpoint a/2 + b/2 is within 2 eps tau of either
    end, plus one rounding of the midpoint (u tau) and one of root * h (u |t|); 8 eps tau covers all three.
  - The clamp of a root that lands on or past h to nextafter(h, 0) moves it by one ulp of h.
  tol(t*) = |h| (gamma_{3p+1} S(tau*) / |q^(m)(tau*) / m!|)^(1/m) + 8 eps |t*| + ulp(h).
This is a bound for the roots it applies to, not a fit. It is a first-order bound, so it is only used for roots whose
tolerance is small next to their distance to every other root (complex ones included), to the ends of the step and to a
cooldown boundary: WELL_MARGIN times smaller. Such a root is "well conditioned"; the others are clusters, even
multiplicities and step ends, about which this reference says nothing beyond "a reported time must be near a root".

On an x86-64 CPU one polynomial of degree 47 takes a few seconds, mostly for its complex roots (the separation); the
callers sample lanes.
"""
import math
from fractions import Fraction

import mpmath as mp
import numpy as np
import sympy as sp

U = 2.0 ** -53
EPS = 2.0 ** -52
WELL_MARGIN = 16.0
_X = sp.Symbol("t")
_DPS = 60


def gamma(n):
    return n * U / (1 - n * U)


class Root:
    """A real root of an event polynomial. t: Fraction (45 digits, or exact when rational), mult, sgn: sign of the time
    derivative of the event function where the root is crossed (odd multiplicity; 0 for even), tol: bound on the error
    of a computed event time, sep: distance to the nearest other root (complex included), in_step: t in [0, h) or
    (h, 0], well: the completeness check applies (set by expected())."""

    def __init__(self, t, mult, sgn, tol, sep, in_step):
        self.t, self.mult, self.sgn, self.tol, self.sep, self.in_step = t, mult, sgn, tol, sep, in_step
        self.well = False

    @property
    def tf(self):
        return float(self.t)

    def __repr__(self):
        return "Root(t=%.17g, mult=%d, sgn=%d, tol=%.2e, sep=%.2e%s%s)" % (
            self.tf, self.mult, self.sgn, self.tol, self.sep, ", in step" if self.in_step else "",
            ", well" if self.well else "")


class Roots(list):
    """The real roots, and .complex: the non-real ones (approximate)."""
    complex = ()


def _dyadic(tau):
    """tau = k / 2^j: a point the bisection of [0, 1) can land on exactly."""
    d = tau.denominator
    return d & (d - 1) == 0 and d <= 2 ** 60


def _sgn(x):
    return (x > 0) - (x < 0)


def _qq(f):
    return sp.Rational(f.numerator, f.denominator)


def _frac(r):
    r = sp.Rational(r)
    return Fraction(int(r.p), int(r.q))


def _in_step(t, H):
    return (0 <= t < H) if H > 0 else (H < t <= 0)


def _refined(f, s, t, eps):
    if s == t:
        return s, t
    return f.refine_root(s, t, eps=eps)


def exact_roots(coeffs, h):
    """The real roots of sum_i coeffs[i] t^i (exact, the doubles read as rationals) within an eighth of a step of the step
    [0, h) / (h, 0], sorted by |t|: those inside the step, and those just outside it, which can explain a reported time
    next to an end. Each root carries its tolerance and whether the completeness check applies to it (see the module
    docstring)."""
    p = len(coeffs) - 1
    A = [Fraction(float(v)) for v in coeffs]
    while len(A) > 1 and A[-1] == 0:
        A.pop()
    if len(A) == 1:
        return Roots()
    H = Fraction(float(h))
    P = sp.Poly([_qq(v) for v in reversed(A)], _X, domain=sp.QQ)
    lo, hi = (min(Fraction(0), H) - abs(H) / 8, max(Fraction(0), H) + abs(H) / 8)
    eps_iv = _qq(abs(H)) / sp.Integer(10) ** 45
    mp.mp.dps = _DPS
    # All roots, complex included, for the separation of each real root (a margin, so 30 digits are plenty).
    try:
        with mp.workdps(30):
            allr = mp.polyroots([mp.mpf(v.numerator) / v.denominator for v in reversed(A)], maxsteps=100, extraprec=60)
    except mp.libmp.libhyper.NoConvergence:
        allr = [complex(r) for r in np.roots([float(v) for v in reversed(A)])]
    cplx = [complex(z) for z in allr if abs(complex(z).imag) > 0]
    hm = mp.mpf(float(h))
    qa = [mp.mpf(v.numerator) / v.denominator * hm ** i for i, v in enumerate(A)]  # q_i = a_i h^i, exact enough
    g = gamma(3 * p + 1)
    out = Roots()
    out.complex = cplx
    _, factors = P.sqf_list()
    for f, m in factors:
        if f.degree() == 0:
            continue
        for (s, t), _k in f.intervals(inf=_qq(lo), sup=_qq(hi)):
            s, t = _refined(f, s, t, eps_iv)
            # Refine until the interval does not straddle an end of the step unless the root is that end.
            for _ in range(200):
                if s == t or all(not (s < e < t) for e in (0, _qq(H))):
                    break
                s, t = f.refine_root(s, t, eps=(t - s) / 16)
            r = _frac(s) if s == t else (_frac(s) + _frac(t)) / 2
            # The sign of the crossing: the sign of P just past the root (the 45-digit interval holds no other root of
            # P); P^(m) at the root is m! times the leading coefficient of the expansion of P there.
            dm = P.diff((_X, m))
            cm = _frac(dm.eval(_qq(r)))
            if m % 2 == 1 and s != t:
                cm = abs(cm) * _sgn(_frac(P.eval(t)))
            sgn = _sgn(cm) if m % 2 == 1 else 0
            tau = mp.mpf(r.numerator) / r.denominator / hm
            S = sum(abs(c) * abs(tau) ** i for i, c in enumerate(qa))
            qm = abs(mp.mpf(cm.numerator) / cm.denominator) * abs(hm) ** m / mp.factorial(m)
            tol = float(abs(hm) * (g * S / qm) ** (mp.mpf(1) / m) + 8 * EPS * abs(mp.mpf(r.numerator) / r.denominator)) \
                + math.ulp(float(h))
            rc = mp.mpf(r.numerator) / r.denominator
            d = sorted(float(abs(mp.mpc(z) - rc)) for z in allr)
            # The m copies of this root in allr are the m nearest; the next one is the nearest other root.
            sep = d[m] if len(d) > m else math.inf
            out.append(Root(r, m, sgn, tol, sep, _in_step(r, H)))
    out.sort(key=lambda R: abs(R.t))
    return out


def cooldown_cut(h, cd_on, spent, cooldown):
    """How far into the step (as a length) a terminal event is still in cooldown. The kernels compute it rescaled to
    the step, lb_offset = (cooldown - spent) / |h| forwards and (cooldown + spent) / |h| backwards (spent is negative
    then; ev_kernels.cuh:389-398), and drop the roots with tau < lb_offset. 0 when the event is not in cooldown."""
    if not cd_on:
        return 0.0
    return (cooldown - spent) if h >= 0 else (cooldown + spent)


def expected(roots, h, direction=0, cut=0.0):
    """Apply the event's direction and the cooldown cut (a length, cooldown_cut()) to the exact roots in the step, and
    mark the well-conditioned ones. Returns (kept, dropped, against): kept = roots past the cooldown boundary with the
    requested crossing sign (even multiplicities kept: they are exceptions, never well conditioned), dropped = roots the
    cooldown removes, against = roots past the boundary whose crossing sign is against the requested direction."""
    H = abs(float(h))
    kept, dropped, against = [], [], []
    for R in roots:
        if not R.in_step:
            continue
        room = min(abs(R.tf), H - abs(R.tf), R.sep, abs(abs(R.tf) - cut) if cut > 0 else math.inf)
        R.well = R.mult == 1 and WELL_MARGIN * R.tol <= room
        if cut > 0 and abs(R.tf) < cut:
            dropped.append(R)
        elif direction != 0 and R.mult % 2 == 1 and R.sgn != direction:
            against.append(R)
        else:
            kept.append(R)
    return kept, dropped, against


def _kind(R, h, cut):
    if R.mult > 1:
        return "multiplicity %d" % R.mult
    if min(abs(R.tf), abs(float(h)) - abs(R.tf)) < WELL_MARGIN * R.tol:
        return "step end"
    if cut > 0 and abs(abs(R.tf) - cut) < WELL_MARGIN * R.tol:
        return "cooldown boundary"
    return "cluster"


def check(records, roots, h, direction=0, cut=0.0):
    """Compare the records of one (lane, event) over one step, [(t, d_sgn)], with the exact roots.
    Completeness: every well-conditioned root that passes the filters gives exactly one record within its tolerance,
    with its crossing sign. No spurious events: a record's derivative sign is the requested direction (if any), and the
    record is within the tolerance of a root that passes the filters, or of a root the check names as an exception (a
    root the check does not apply to, just outside the step, or within its tolerance of the cooldown boundary). A record
    at a root the cooldown removes, or at a well-conditioned root crossed against the requested direction, is a
    failure. Returns (problems, notes, findings, n_well): problems are failures, notes name what happened at every root
    the check does not apply to, findings (also in notes) the known departures of the shared algorithm from the exact
    answer."""
    kept, dropped, against = expected(roots, h, direction, cut)
    problems, notes, findings = [], [], []
    near = lambda R, t: abs(t - R.tf) <= R.tol  # noqa: E731
    Hf = Fraction(float(h))
    # Known findings about the algorithm the device and the oracle share (see tests/README.md):
    # (1) a root exactly on a point the bisection reaches (tau = k / 2^j with a short j; the start of the step is
    #     tau = 0) is reported by the start-of-interval path of every interval that begins there, and again by the root
    #     finder, which returns the lower end of a bracket where the polynomial is exactly zero: identical records;
    # (2) so in the isolating interval that begins at a root at t = 0, the root finder returns t = 0 and the one root
    #     of that interval, the first root of the polynomial after t = 0, is not reported.
    at_zero = any(R.t == 0 for R in kept)
    first_after_zero = next((R for R in roots if R.in_step and R.t != 0), None) if at_zero else None
    for R in kept:
        hits = [r for r in records if near(R, r[0])]
        if R.well:
            tau = abs(R.t / Hf)
            if (len(hits) > 1 and _dyadic(tau) and tau.denominator <= 2 ** 24 and len(set(hits)) == 1
                    and hits[0][1] == R.sgn):
                findings.append("root exactly at the bisection point tau = %s (t = %.17g): %d identical records"
                                % (tau, R.tf, len(hits)))
            elif not hits and R is first_after_zero:
                findings.append("root at t = %.17g not reported: its isolating interval begins at the root at t = 0"
                                % R.tf)
            elif len(hits) != 1:
                problems.append("root %r: %d records %r" % (R, len(hits), hits))
            elif hits[0][1] != R.sgn:
                problems.append("root %r: record %r has the wrong derivative sign" % (R, hits[0]))
        else:
            notes.append("%s at t=%.17g (tol %.1e, sep %.1e): %d record(s)" % (_kind(R, h, cut), R.tf, R.tol, R.sep,
                                                                              len(hits)))
    boundary = [R for R in dropped if cut - abs(R.tf) <= R.tol]
    for r in records:
        if direction != 0 and r[1] != direction:
            problems.append("record %r has a derivative sign against the requested direction %d" % (r, direction))
        if any(near(R, r[0]) for R in kept):
            continue
        if any(near(R, r[0]) for R in boundary):
            notes.append("cooldown boundary: record %r within the tolerance of a root at the boundary" % (r,))
            continue
        if any(near(R, r[0]) for R in dropped):
            problems.append("record %r is at a root in the cooldown (the first %.17g of the step)" % (r, cut))
            continue
        bad = [R for R in against if R.well and near(R, r[0])]
        if bad:
            problems.append("record %r is at %r, crossed against the requested direction" % (r, bad[0]))
            continue
        if any(near(R, r[0]) for R in against):
            notes.append("%s crossed against the direction: record %r" % (
                _kind([R for R in against if near(R, r[0])][0], h, cut), r))
            continue
        if any(near(R, r[0]) for R in roots if not R.in_step):
            notes.append("root just outside the step: record %r" % (r,))
            continue
        z = min(roots.complex, key=lambda z: abs(z - r[0]), default=None)
        if z is not None and abs(z.imag) <= 1e-6 * abs(float(h)) and abs(r[0] - z.real) <= 1e3 * abs(z.imag):
            notes.append("complex pair %.17g +- %.1ei next to the real axis (a rounded double root): record %r"
                         % (z.real, abs(z.imag), r))
            continue
        problems.append("record %r is not near any root that passes the filters" % (r,))
    return problems, notes + findings, findings, sum(R.well for R in kept)
