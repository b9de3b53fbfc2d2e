"""Continuous output, propagate_grid() and dense output held bit for bit to a host restatement of the device
arithmetic, on the coefficients and times the device recorded itself, and within a derived bound of an exact evaluation.

Why not the oracle. The oracle takes its own steps (its pow is glibc's, the device's is libdevice's) and its default
dense output is Horner with the product and the sum rounded apart, while the device fuses them: against it only a
tolerance of ~1e-13 holds, and at that tolerance the polynomial of the neighbouring step, or an h computed without the
low word of the time, still passes. Here the device's own recording is the input of both sides:

- the restatement (tests/cpp/cout_emul.cpp, plain C++ with std::fma and -ffp-contract=off, no device header) repeats
  k_cout_eval's step selection (upper_bound over the padded times, its two decrements), its h = (t - t_k).hi in
  double-length arithmetic, eval_poly() (Horner with fma, or the compensated sum of the monomials in high-accuracy
  mode), grid_covered()'s closed window with rem0, and update_d_output()'s tau. The device must equal it bit for bit;
- the exact reference picks its step by its own rule (forward lanes: the step whose [t_k, t_k+1) holds t, backward
  lanes mirrored, times outside the recording clamped to the first or last step), evaluates that polynomial in rationals
  at h* = t - (t_k.hi + t_k.lo), and allows the error the arithmetic can make (bound() below).

The checkers are shown to fail on synthetic slips (the neighbouring step, h from t_k.hi only, step k +- slab_iters,
the neighbouring lane, unfused Horner) on recordings of the CPU oracle, without a GPU.

The slab sizes of the GPU tests rest on the recorder's formula (hy_cout_rec, batch.cu): an iteration takes
n_eq * (order + 1) * n * 8 bytes, and a slab holds clamp(64 MiB / that, 1, 4096) iterations. For the pendulum at order
20 that is 336 bytes per lane: 1 iteration per slab for n >= 199,729, 3 for n = 2^16 + 3, 195 for n = 1024, the cap of
4096 for n = 4. The time rows grow at 64, 128, ... rows.
"""
import ctypes as C
import functools
import os
import subprocess
from fractions import Fraction

import numpy as np
import pytest

import heyoka_b200 as hb
import oracle
from common import FFNN_TOL, ffnn_batch_state, sys_ffnn, sys_pendulum, sys_two_body, two_body_batch_state
from test_gpu_parity import KERNELS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "build", "libcout_emul.so")
U = 2.0 ** -53  # unit roundoff of binary64
HORNER, COMPENSATED, UNFUSED = 0, 1, 2  # evaluation modes of cout_emul.cpp


# ---- the restatement (tests/cpp/cout_emul.cpp) ----------------------------------------------------------------------

@functools.cache
def _emul():
    src = os.path.join(ROOT, "tests", "cpp", "cout_emul.cpp")
    os.makedirs(os.path.dirname(SO), exist_ok=True)
    if not os.path.exists(SO) or os.path.getmtime(SO) < os.path.getmtime(src):
        tmp = "%s.%d" % (SO, os.getpid())
        subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-shared", "-fPIC", src, "-o", tmp], check=True)
        os.replace(tmp, SO)
    return C.CDLL(SO)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _f(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def select(t_hi, t_lo, tm):
    """k_cout_eval's step for every lane at times tm [n]."""
    n = t_hi.shape[1]
    k = np.empty(n, dtype=np.int64)
    _emul().ce_select(C.c_uint64(n), C.c_uint64(t_hi.shape[0]), _p(t_hi), _p(t_lo), _p(_f(tm)), _p(k))
    return k


def h_of(t_hi, t_lo, k, tm, hi_only=False):
    n = t_hi.shape[1]
    h = np.empty(n)
    _emul().ce_h(C.c_uint64(n), _p(t_hi), _p(t_lo), _p(np.ascontiguousarray(k, dtype=np.int64)), _p(_f(tm)),
                 C.c_int(int(hi_only)), _p(h))
    return h


def evaluate(tcs, k, h, mode, src=None):
    """P_k[lane] at h[lane] for every lane, tcs [n_steps, n_eq, order + 1, n]; src: the lane whose coefficients are used."""
    _, n_eq, p1, n = tcs.shape
    out = np.empty((n_eq, n))
    s = None if src is None else np.ascontiguousarray(src, dtype=np.uint64)
    _emul().ce_eval(C.c_uint(n_eq), C.c_uint(p1 - 1), C.c_uint64(n), C.c_int(mode), _p(tcs),
                    _p(np.ascontiguousarray(k, dtype=np.int64)), None if s is None else _p(s), _p(_f(h)), _p(out))
    return out


def restate_cout(rec, tm, ha):
    tcs, t_hi, t_lo = rec
    k = select(t_hi, t_lo, tm)
    return evaluate(tcs, k, h_of(t_hi, t_lo, k, tm), COMPENSATED if ha else HORNER)


def restate_d_output(tc, t, t_hi, t_lo, last_h, ha, rel_time):
    n = tc.shape[2]
    tau = np.empty(n)
    _emul().ce_tau(C.c_uint64(n), C.c_int(int(rel_time)), _p(_f(np.broadcast_to(t, (n,)))), _p(_f(t_hi)), _p(_f(t_lo)),
                   _p(_f(last_h)), _p(tau))
    return evaluate(_f(tc[None]), np.zeros(n, dtype=np.int64), tau, COMPENSATED if ha else HORNER), tau


class GridRestatement:
    """propagate_grid()'s output, rebuilt from the steps of a twin integrator: grid point 0 is the state after the
    propagation to grid[0], then every step's window (grid_covered()) is sampled on that step's coefficients."""

    def __init__(self, grid, ha):
        self.grid, self.mode = _f(grid), COMPENSATED if ha else HORNER
        self.n_pts, self.n = grid.shape
        self.cur = np.ones(self.n, dtype=np.uint64)
        self.out = None

    def sample(self, t_hi, t_lo, last_h, rem0, tc):
        n_eq, p1, n = tc.shape
        _emul().ce_grid_sample(C.c_uint(n_eq), C.c_uint(p1 - 1), C.c_uint64(n), C.c_int(self.mode), C.c_uint64(self.n_pts),
                               _p(self.grid), _p(_f(t_hi)), _p(_f(t_lo)), _p(_f(last_h)),
                               _p(np.ascontiguousarray(rem0, dtype=np.uint8)), _p(_f(tc)), _p(self.cur), _p(self.out))


def dfl_sub(ahi, alo, bhi, blo):
    """Double-length a - b with Knuth's and Dekker's sums, in numpy (no contraction: every operation rounds)."""
    def two_sum(a, b):
        x = a + b
        z = x - a
        return x, (a - (x - z)) + (b - z)
    bhi, blo = -np.asarray(bhi, dtype=np.float64), -np.asarray(blo, dtype=np.float64)
    xh, yh = two_sum(np.asarray(ahi, dtype=np.float64), bhi)
    xl, yl = two_sum(np.asarray(alo, dtype=np.float64), blo)
    s = xh + (yh + xl)
    e = (xh - s) + (yh + xl)
    r = s + (e + yl)
    return r, (s - r) + (e + yl)


# ---- the exact reference ------------------------------------------------------------------------------------------

def exact_step(rec, lane, t):
    """The reference's step for time t on a lane: forward, the last step whose start is <= t (so the step whose
    [t_k, t_k+1) holds t, zero-length steps never hold one); backward mirrored; clamped to [0, n_steps - 1]."""
    tcs, t_hi, t_lo = rec
    n_steps = tcs.shape[0]
    fwd = t_hi[-1, lane] > 0  # the padding row: +inf forwards, -inf backwards
    T = [Fraction(t_hi[k, lane]) + Fraction(t_lo[k, lane]) for k in range(n_steps)]
    tq = Fraction(t)
    ks = [k for k in range(n_steps) if (T[k] <= tq if fwd else T[k] >= tq)]
    k = ks[-1] if ks else 0
    return k, tq - T[k]


def exact_poly(c, h):
    r = Fraction(0)
    for cj in reversed(c):
        r = r * h + Fraction(cj)
    return r


def bound(c, h, ha):
    """What the evaluation of P = sum c_j h^j at the computed h (= h* rounded once, |h - h*| <= u |h*|) may differ from
    P(h*), u = 2^-53, S = sum |c_j| |h|^j at the larger |h|:
    - Horner with fma: one rounding per order, gamma_p S (gamma_p = p u / (1 - p u));
    - compensated summation: monomial j carries j roundings of the powers and one of the product, (j + 1) u |c_j| |h|^j,
      and the compensated sum adds 2 u |P| and second-order terms, bounded by p^2 u^2 S;
    - the rounding of h: |P'| u |h*| <= u |h*| sum j |c_j| |h|^(j - 1).
    The second-order remainders of all three are covered by 4 p^2 u^2 S. Calibrated on the oracle's recordings
    (test_exact_bound_holds_on_oracle_recordings): the largest error seen is 0.36 of this bound, so a slip has to
    stay within three times the rounding error of a correct evaluation to pass."""
    p = len(c) - 1
    hm = abs(float(h)) * (1. + 2. * U)
    a = np.abs(np.asarray(c, dtype=np.float64))
    powers = hm ** np.arange(p + 1)
    terms = a * powers
    S = float(np.sum(terms))
    S1 = float(np.sum(np.arange(1, p + 1) * a[1:] * powers[:-1]))
    if ha:
        ev = float(np.sum((np.arange(p + 1) + 1.) * U * terms)) + 2. * U * abs(float(exact_poly(c, h)))
    else:
        ev = p * U / (1. - p * U) * S
    return ev + U * hm * S1 + 4. * p * p * U * U * S


def exact_errors(rec, lanes, tm, vals, ha):
    """Largest |value - P_k(h*)| / bound over the lanes and state variables, with the reference's own step k."""
    tcs = rec[0]
    worst = 0.
    for lane in lanes:
        k, hs = exact_step(rec, lane, tm[lane])
        for i in range(tcs.shape[1]):
            c = tcs[k, i, :, lane].tolist()
            b = bound(c, hs, ha)
            err = abs(float(Fraction(vals[i, lane]) - exact_poly(c, hs)))
            worst = max(worst, err / b if b > 0 else (np.inf if err > 0 else 0.))
    return worst


def assert_exact(rec, lanes, tm, vals, ha, what=""):
    w = exact_errors(rec, lanes, tm, vals, ha)
    assert w <= 1., "%s: error %.3g times the bound" % (what, w)


def assert_bits(a, b, what=""):
    a, b = np.asarray(a), np.asarray(b)
    bad = np.argwhere(a.view(np.uint64) != b.view(np.uint64))
    assert bad.size == 0, "%s: %d values differ, first at %s: %r != %r" % (
        what, len(bad), tuple(bad[0]), a[tuple(bad[0])], b[tuple(bad[0])])


# ---- query times ----------------------------------------------------------------------------------------------------

def query_rows(rec, rng, n_inner=3):
    """Rows of times [m, n], per lane: every recorded time (exact step boundaries where t_lo = 0), points inside steps,
    the first and last time, and times before and after the recording."""
    tcs, t_hi, t_lo = rec
    N = tcs.shape[0]
    rows = [t_hi[k] for k in range(N + 1)]
    step = t_hi[1:N + 1] - t_hi[:N]
    for _ in range(n_inner):
        k = rng.integers(0, N, t_hi.shape[1])
        f = rng.uniform(0.05, 0.95, t_hi.shape[1])
        rows.append(t_hi[k, np.arange(t_hi.shape[1])] + f * step[k, np.arange(t_hi.shape[1])])
    span = np.abs(t_hi[N] - t_hi[0]) + 1.
    rows += [t_hi[0] - span, t_hi[N] + span, t_hi[0] + span * 0.5, t_hi[N] - span * 0.5]
    return np.array(rows)


def sample_lanes(n, m=12, seed=0):
    if n <= m:
        return list(range(n))
    rng = np.random.default_rng(seed)
    return sorted({0, n - 1, *rng.choice(n, m - 2, replace=False).tolist()})


# ---- CPU: the restatement and the checkers on the oracle's recordings -----------------------------------------------

def _oracle_recording(ha, tol=0., t0=None, n=6, tf_span=6.0, mdt=None):
    """A pendulum recording of the oracle (its own steps): lanes forwards and backwards, started at t0 (per lane)."""
    P = hb.Program(sys_pendulum(), tol=tol, high_accuracy=ha)
    rng = np.random.default_rng(3)
    st = np.array([rng.uniform(-1., 1., n), rng.uniform(-0.5, 0.5, n)])
    t0 = np.zeros(n) + 0.1 if t0 is None else np.asarray(t0, dtype=np.float64)
    o = oracle.OracleIntegrator(P, st, n, time=t0, mode=oracle.FMA)
    sign = np.where(np.arange(n) % 3 == 1, -1., 1.)
    co = o.propagate_until_cout(t0 + sign * tf_span * (1. + 0.1 * np.arange(n)), max_delta_t=mdt)
    return P, co, (co.tcs, co.t_hi, co.t_lo)


def test_restatement_equals_oracle_high_accuracy():
    """In high-accuracy mode the oracle's dense output is the compensated sum with every operation rounded on its own,
    the device's form: the restatement equals OracleCOut (the reference's continuous output restated) bit for bit."""
    _, co, rec = _oracle_recording(True)
    rng = np.random.default_rng(5)
    for tm in query_rows(rec, rng):
        assert_bits(restate_cout(rec, tm, True), co(tm), "t = %r" % tm[0])


def test_default_mode_differs_from_oracle_where_horner_is_unfused():
    """In the default mode the device fuses Horner's product and sum (fma), the oracle rounds them apart (its
    -ffp-contract=off build): the two differ at some points, and the restatement with the unfused form equals the
    oracle everywhere, so the fma is the whole difference."""
    _, co, rec = _oracle_recording(False)
    rng = np.random.default_rng(6)
    n_diff = n_all = 0
    for tm in query_rows(rec, rng):
        ref = co(tm)
        k = select(rec[1], rec[2], tm)
        h = h_of(rec[1], rec[2], k, tm)
        assert_bits(evaluate(rec[0], k, h, UNFUSED), ref)
        fused = evaluate(rec[0], k, h, HORNER)
        n_diff += int(np.count_nonzero(fused != ref))
        n_all += fused.size
    assert 0 < n_diff < n_all, (n_diff, n_all)


@pytest.mark.parametrize("ha", [False, True])
def test_exact_bound_holds_on_oracle_recordings(ha):
    """The restatement lies within bound() of the exact evaluation at every query, lane and variable. The largest
    ratio seen is 0.36 (0.30 / 0.18 fused, 0.33 / 0.36 compensated, starting near 0 / near 2^40); the assertion keeps
    the bound at least twice the largest error. Also with a start near 2^40, where the low word of the times matters."""
    for t0 in (None, 2.0 ** 40 + np.array([0.1, 0.2, 0.3, 0.4, 0.5, 0.6])):
        _, _, rec = _oracle_recording(ha, t0=t0)
        rng = np.random.default_rng(7)
        worst = 0.
        for tm in query_rows(rec, rng):
            worst = max(worst, exact_errors(rec, range(tm.size), tm, restate_cout(rec, tm, ha), ha))
        assert worst < 0.5, worst


def _slips(rec, tm, ha, slab_iters):
    """Evaluations that are each wrong in one way."""
    tcs, t_hi, t_lo = rec
    N, n = tcs.shape[0], tcs.shape[3]
    mode = COMPENSATED if ha else HORNER
    k = select(t_hi, t_lo, tm)
    h = h_of(t_hi, t_lo, k, tm)
    # The neighbouring step, evaluated at its own h (an off-by-one of the search).
    kn = np.where(k + 1 < N, k + 1, k - 1)
    ks = np.where(k + slab_iters < N, k + slab_iters, k - slab_iters)
    return {
        "neighbouring step": evaluate(tcs, kn, h_of(t_hi, t_lo, kn, tm), mode),
        "h from t_k.hi only": evaluate(tcs, k, h_of(t_hi, t_lo, k, tm, hi_only=True), mode),
        "step k +- slab_iters": evaluate(tcs, ks, h_of(t_hi, t_lo, ks, tm), mode),
        "neighbouring lane": evaluate(tcs, k, h, mode, src=(np.arange(n) + 1) % n),
        "unfused Horner": evaluate(tcs, k, h, UNFUSED),
    }


def test_checkers_reject_slips():
    """On an oracle recording started near 2^40 (non-dyadic steps: t_lo != 0) at tol 1e-10 (neighbouring polynomials
    differ by ~1e-10, far above the rounding bound), each slip fails the bit-for-bit check, and all but the unfused
    Horner fail the exact check (unfused Horner is as accurate as the fused one: the exact check cannot see it)."""
    t0 = 2.0 ** 40 + np.array([0.1, 0.2, 0.3, 0.4, 0.5, 0.6])
    _, _, rec = _oracle_recording(False, tol=1e-10, t0=t0)
    assert rec[0].shape[0] > 8 and np.count_nonzero(rec[2][1:-1]) > rec[2][1:-1].size // 2
    rng = np.random.default_rng(8)
    rows = query_rows(rec, rng, n_inner=6)
    inside = rows[rec[0].shape[0] + 1:rec[0].shape[0] + 7]  # the points inside steps
    bit_fail, exact_fail = {}, {}
    for tm in inside:
        good = restate_cout(rec, tm, False)
        assert_exact(rec, range(tm.size), tm, good, False, "the restatement itself")
        for name, v in _slips(rec, tm, False, slab_iters=4).items():
            bit_fail[name] = bit_fail.get(name, False) or not np.array_equal(v, good)
            exact_fail[name] = exact_fail.get(name, False) or exact_errors(rec, range(tm.size), tm, v, False) > 1.
    assert all(bit_fail.values()), bit_fail
    assert exact_fail == {"neighbouring step": True, "h from t_k.hi only": True, "step k +- slab_iters": True,
                          "neighbouring lane": True, "unfused Horner": False}, exact_fail


# ---- GPU: the recording -------------------------------------------------------------------------------------------

def _times(co):
    """The recorded times (hi, lo), [n_steps + 2, n]: get_times() returns the high words only."""
    n = co.get_batch_size()
    hi, lo = np.empty((co.get_n_steps() + 2, n)), np.empty((co.get_n_steps() + 2, n))
    hb.check(hb.lib.hy_cout_download(co._h, hb._dptr(hi), hb._dptr(lo), None))
    return hi, lo


def recording(co):
    hi, lo = _times(co)
    assert_bits(co.get_times(), hi, "get_times()")
    return _f(co.get_tcs()), hi, lo


def _capture(log):
    """A step callback that keeps, after every iteration, the state (before the callback could change it), the time,
    last_h and the Taylor coefficients."""
    def cb(ta):
        log.append((ta.state.copy(), ta.dtime[0].copy(), ta.dtime[1].copy(), ta.last_h.copy(), ta.tc.copy()))
        return True
    return cb


def _three_body_state(n, seed=2):
    rng = np.random.default_rng(seed)
    st = np.zeros((18, n))
    st[6], st[10] = 1., 1.                    # body 1: x = 1, vy = 1
    st[12], st[16] = -2., -0.7                # body 2: x = -2, vy = -0.7
    st += rng.uniform(-1e-2, 1e-2, st.shape) * (st != 0)
    return st


# Every kernel shape that takes the system: the cooperative shapes and k_hbm on the pendulum, the one-thread-per-lane
# N-body kernel on the two-body system, the N-body kernel's shapes on three bodies, k_nn on a small dense network.
REC_CASES = [(name, k, "pendulum") for name, k in KERNELS.items() if not k["tape"].startswith("nbody")]
REC_CASES += [(name, k, "two_body") for name, k in KERNELS.items() if k["tape"] == "nbody-lane"]
REC_CASES += [(name, k, "three_body") for name, k in KERNELS.items() if k["tape"] == "nbody"]
REC_CASES += [("nn", dict(tape="nn"), "ffnn")]


def _rec_system(which, n):
    if which == "pendulum":
        rng = np.random.default_rng(1)
        return sys_pendulum(), np.array([rng.uniform(-2., 2., n), rng.uniform(-1., 1., n)]), {}, 3.0
    if which == "two_body":
        return sys_two_body(), two_body_batch_state(n), {}, 2.0
    if which == "three_body":
        return hb.model.nbody(3, masses=[1., 0.01, 0.001]), _three_body_state(n), {}, 2.0
    return sys_ffnn(), ffnn_batch_state(n), dict(tol=FFNN_TOL), 0.5


@pytest.mark.gpu
@pytest.mark.parametrize("ha", [False, True])
@pytest.mark.parametrize("name,kernel,which", REC_CASES, ids=[c[0] + "-" + c[2] for c in REC_CASES])
def test_recorder_in_place(name, kernel, which, ha):
    """The step kernel writes each iteration's coefficients into the recorder's slot in place. Against what a step
    callback sees after every iteration: get_tcs()[k] is that iteration's tc, times row k + 1 its (hi, lo) time, the
    order-0 row of tcs[k] the state before step k, and the restated evaluation of tcs[k] at last_h_k the state after
    it (the independent check of the in-place write: every kernel's state update is eval_poly()'s arithmetic). A
    recording without the callback is the same, bit for bit."""
    n = 5
    sys_, st, kw, tf = _rec_system(which, n)
    tfs = tf * (1. + 0.2 * np.arange(n))  # lanes that finish early take zero-length steps
    log = []
    ta = hb.taylor_adaptive_batch(sys_, st, n, high_accuracy=ha, kernel=kernel, **kw)
    co = ta.propagate_until(tfs, c_output=True, callback=_capture(log))
    assert ta._b.kernel_info()["tape"] == kernel["tape"].replace("smem-notmem", "smem")  # (one kernel, two names)
    tcs, t_hi, t_lo = recording(co)
    assert tcs.shape[0] == len(log) > 3
    mode = COMPENSATED if ha else HORNER
    before = st
    for k, (s, hi, lo, lh, tc) in enumerate(log):
        assert_bits(tcs[k], tc, "tcs[%d]" % k)
        assert_bits(t_hi[k + 1], hi, "t_hi[%d]" % (k + 1))
        assert_bits(t_lo[k + 1], lo, "t_lo[%d]" % (k + 1))
        assert_bits(tcs[k][:, 0, :], before, "order 0 of tcs[%d]" % k)
        assert_bits(evaluate(tcs, np.full(n, k), lh, mode), s, "state after step %d" % k)
        before = s
    ta2 = hb.taylor_adaptive_batch(sys_, st, n, high_accuracy=ha, kernel=kernel, **kw)
    co2 = ta2.propagate_until(tfs, c_output=True)
    for a, b in zip(recording(co2), (tcs, t_hi, t_lo)):
        assert_bits(a, b, "recording without a callback")
    assert_bits(ta2.state, ta.state)


# ---- GPU: the evaluation ------------------------------------------------------------------------------------------

def check_cout(co, rec, ha, rows, lanes, what=""):
    """co(t) equals the restatement at every lane and query time, and the sampled lanes lie within the exact bound."""
    for r, tm in enumerate(rows):
        got = co(tm).copy()
        assert_bits(got, restate_cout(rec, tm, ha), "%s, query row %d" % (what, r))
        assert_exact(rec, lanes, tm, got, ha, "%s, query row %d" % (what, r))


def _mixed_batch(n, rng):
    """Pendulum lanes by kind (lane % 6): forward with clamped dyadic steps (boundaries are doubles), backward,
    forward and finishing early, target = start time, a start near 2^40 with non-dyadic steps (t_lo != 0), forward
    with free steps."""
    kind = np.arange(n) % 6
    st = np.array([rng.uniform(-2., 2., n), rng.uniform(-1., 1., n)])
    t0 = np.where(kind == 4, 2.0 ** 40 + 0.1 * rng.uniform(1., 2., n), rng.uniform(-1., 1., n))
    span = np.select([kind == 1, kind == 2, kind == 3], [-2.0, 0.7, 0.], 2.0 + rng.uniform(0., 0.1, n))
    mdt = np.where(kind == 0, 2.0 ** -3, np.inf)
    t0 = np.where(kind == 0, np.round(t0 * 8.) / 8., t0)
    return st, t0, t0 + span, mdt, kind


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 127, 129, 2 ** 16 + 3])
def test_cout_eval_mixed_batch(n):
    """Forward, backward and mixed lanes in one batch, a lane finishing early (its times repeat over zero-length
    steps), a lane whose target is its start, a start near 2^40; batch tails around k_cout_eval's 128-thread CTAs.
    Both evaluation modes; exact step boundaries, points inside steps, the first and last time, times outside."""
    rng = np.random.default_rng(n)
    st, t0, tf, mdt, kind = _mixed_batch(n, rng)
    for ha in (False, True):
        ta = hb.taylor_adaptive_batch(sys_pendulum(), st, n, time=t0, high_accuracy=ha)
        co = ta.propagate_until(tf, c_output=True, max_delta_t=mdt)
        rec = recording(co)
        N = rec[0].shape[0]
        assert N > 8
        if n > 4:
            assert np.any(rec[2][1:N + 1] != 0.)                  # t_lo != 0 somewhere
            assert np.all(rec[1][N, kind == 3] == t0[kind == 3])  # a lane that never moved
            early = kind == 2
            assert np.all(rec[1][N, early] == rec[1][N - 1, early])
        lb, ub = co.get_bounds()
        assert_bits(lb, rec[1][0])
        assert_bits(ub, rec[1][N])
        rows = query_rows(rec, rng)
        tm_inside = rows[N + 1]
        if n > 1000:
            rows = rows[np.r_[0:3, N // 2, N - 1:rows.shape[0]]]
        check_cout(co, rec, ha, rows, sample_lanes(n, 8), "n = %d, ha = %s" % (n, ha))
        if n > 4:
            # On the lanes started near 2^40 the low word of the times moves the result.
            big = np.nonzero(kind == 4)[0]
            tm = tm_inside
            k = select(rec[1], rec[2], tm)
            slip = evaluate(rec[0], k, h_of(rec[1], rec[2], k, tm, hi_only=True), COMPENSATED if ha else HORNER)
            assert np.any(slip[:, big] != co(tm)[:, big])
        del co, rec  # (at n = 2^16 + 3 a recording takes a few hundred MB on the host and on the device)


def _ev_pendulum():
    x, v = hb.make_vars("x", "v")
    return [(x, v), (v, -9.8 * hb.sin(x))], v


@pytest.mark.gpu
def test_cout_eval_cut_recordings():
    """Recordings cut by max_steps, by a step callback's stop, and by a stopping terminal event (recorded through
    append(): its last time is the event time)."""
    n = 6
    rng = np.random.default_rng(4)
    st = np.array([rng.uniform(0.5, 1., n), np.zeros(n)])
    for ha in (False, True):
        ta = hb.taylor_adaptive_batch(sys_pendulum(), st, n, high_accuracy=ha)
        co = ta.propagate_until(10., c_output=True, max_steps=7)
        rec = recording(co)
        assert rec[0].shape[0] == 7 and ta.propagate_res[0][0] == hb.taylor_outcome.step_limit
        check_cout(co, rec, ha, query_rows(rec, rng), range(n), "max_steps")
        ta = hb.taylor_adaptive_batch(sys_pendulum(), st, n, high_accuracy=ha)
        count = []
        co = ta.propagate_until(10., c_output=True, callback=lambda t: count.append(1) or len(count) < 5)
        rec = recording(co)
        assert rec[0].shape[0] == 5 and ta.propagate_res[0][0] == hb.taylor_outcome.cb_stop
        check_cout(co, rec, ha, query_rows(rec, rng), range(n), "callback stop")
        sys_, v = _ev_pendulum()
        st_ev = st.copy()
        st_ev[1] = 3.0  # v crosses zero at the first turning point, after a few steps
        ta = hb.taylor_adaptive_batch(sys_, st_ev, n, high_accuracy=ha, t_events=[hb.t_event_batch(v)])
        co = ta.propagate_until(10., c_output=True, max_delta_t=0.05)
        rec = recording(co)
        N = rec[0].shape[0]
        assert_bits(rec[1][N], ta.time, "the last recorded time is the event time")
        assert np.all(ta.time < 10.)
        check_cout(co, rec, ha, query_rows(rec, rng), range(n), "terminal event")


def _slab_iters(n_eq, order, n):
    return int(min(max((64 << 20) // (n_eq * (order + 1) * n * 8), 1), 4096))


@pytest.mark.gpu
@pytest.mark.parametrize("n,mdt,tf,per_slab", [(2 ** 18, 2.0 ** -7, 3 * 2.0 ** -7, 1), (2 ** 16 + 3, 2.0 ** -7, 12 * 2.0 ** -7, 3),
                                               (1024, 2.0 ** -10, 0.5, 195), (4, 2.0 ** -14, 0.6, 4096)])
def test_cout_eval_across_slabs(n, mdt, tf, per_slab):
    """The recording lives in slabs of slab_iters iterations (the formula in the module docstring gives per_slab):
    queries in the first and the last iteration of every slab, every lane with the restatement, sampled lanes with the
    exact reference. n = 4 records more than 8192 iterations, through the time rows' reallocations."""
    assert _slab_iters(2, 20, n) == per_slab
    rng = np.random.default_rng(9)
    st = np.array([rng.uniform(-2., 2., n), rng.uniform(-1., 1., n)])
    ta = hb.taylor_adaptive_batch(sys_pendulum(), st, n)
    assert ta.get_order() == 20
    co = ta.propagate_until(tf, c_output=True, max_delta_t=mdt)
    rec = recording(co)
    N = rec[0].shape[0]
    assert N >= round(tf / mdt) > 2 * per_slab
    lanes = sample_lanes(n, 6)
    for s in range(-(-N // per_slab)):
        for k in {s * per_slab, min((s + 1) * per_slab, N) - 1}:
            for f in (0.5, 0.):
                tm = rec[1][k] + f * (rec[1][k + 1] - rec[1][k])
                got = co(tm).copy()
                assert_bits(got, restate_cout(rec, tm, False), "slab %d, iteration %d" % (s, k))
                assert_exact(rec, lanes, tm, got, False, "slab %d, iteration %d" % (s, k))


@pytest.mark.gpu
def test_cout_eval_tie_with_angle_reducer():
    """A rotating pendulum reduced into [0, 2pi) by the angle reducer: at a boundary t_k+1 where the angle was reduced
    the two candidate polynomials differ by 2pi. co(t_k+1) is step k+1's (reduced) order-0 coefficient (upper_bound:
    the first time greater than t_k+1 starts step k+2); when the last step reduces, co(t_N) is the unreduced end of that
    step (the padding row leaves step N - 1), which is not ta.state. Both follow from recording before the callback."""
    x, _ = hb.make_vars("x", "v")
    n = 3
    st = np.array([np.zeros(n), np.array([8., 9., 10.])])
    mdt = 2.0 ** -6
    for ha in (False, True):
        ta = hb.taylor_adaptive_batch(sys_pendulum(), st, n, high_accuracy=ha)
        co = ta.propagate_until(2.0, c_output=True, max_delta_t=mdt, callback=hb.callback.angle_reducer([x]))
        tcs, t_hi, t_lo = rec = recording(co)
        N = tcs.shape[0]
        assert np.all(t_lo == 0.) and np.all(t_hi[1:N + 1] == np.arange(1, N + 1)[:, None] * mdt)
        mode = COMPENSATED if ha else HORNER
        ends = np.array([evaluate(tcs, np.full(n, k), np.full(n, mdt), mode) for k in range(N)])  # [N, n_eq, n]
        red = np.abs(ends[:-1, 0, :] - tcs[1:, 0, 0, :]) > 1.   # reduced at the end of step k
        assert np.all(red.sum(axis=0) >= 2)
        for lane in range(n):
            for k in np.nonzero(red[:, lane])[0]:
                tm = t_hi[k + 1].copy()
                got = co(tm)
                assert got[0, lane] == tcs[k + 1, 0, 0, lane] and got[1, lane] == tcs[k + 1, 1, 0, lane]
                assert got[0, lane] != ends[k, 0, lane]
                assert_bits(got, restate_cout(rec, tm, ha))
        # The last step reduces: a lane alone (a lane of a batch that got there first would end on zero-length steps)
        # propagated to its last reducing boundary takes the same clamped steps.
        for lane in range(n):
            last = np.nonzero(red[:, lane])[0][-1] + 1
            tf = last * mdt
            ta = hb.taylor_adaptive_batch(sys_pendulum(), st[:, lane:lane + 1], 1, high_accuracy=ha)
            co = ta.propagate_until(tf, c_output=True, max_delta_t=mdt, callback=hb.callback.angle_reducer([x]))
            rec2 = recording(co)
            assert rec2[0].shape[0] == last
            got = co(tf).copy()
            assert_bits(got[:, 0], ends[last - 1, :, lane], "co(t_N): the unreduced end of the last step")
            assert_bits(got, restate_cout(rec2, np.array([tf]), ha))
            assert got[0, 0] != ta.state[0, 0] and got[0, 0] >= 2 * np.pi
            red_state = got.copy()
            hb.callback.reduce_angles(red_state[0])
            assert_bits(ta.state, red_state)


# ---- GPU: propagate_grid() and dense output -------------------------------------------------------------------------

def _twin_grid(sys_, st, t0, grid, mdt, ha, callback=None):
    """propagate_grid() and the restatement of its output from a twin integrator's steps."""
    n = st.shape[1]
    ta = hb.taylor_adaptive_batch(sys_, st, n, time=t0, high_accuracy=ha)
    out = ta.propagate_grid(grid, max_delta_t=mdt)
    tw = hb.taylor_adaptive_batch(sys_, st, n, time=t0, high_accuracy=ha)
    tw.propagate_until(grid[0].copy(), max_delta_t=mdt, write_tc=True)
    assert np.all(tw.last_h == 0.)
    R = GridRestatement(grid, ha)
    R.out = np.full((grid.shape[0], st.shape[0], n), np.nan)
    R.out[0] = tw.state
    # The remaining time to the last grid point (rem0: zero in both words); after a step it is zero when the step
    # took what remained (h == rem.hi), else recomputed from the new time.
    tf = grid[-1]
    rem = dfl_sub(tf, 0., tw.dtime[0], tw.dtime[1])
    R.sample(tw.dtime[0], tw.dtime[1], tw.last_h, (rem[0] == 0.) & (rem[1] == 0.), tw.tc)
    log = []
    tw.propagate_until(tf.copy(), max_delta_t=mdt, c_output=True, callback=_capture(log))
    for _, hi, lo, lh, tc in log:
        took = lh == rem[0]
        r = dfl_sub(tf, 0., hi, lo)
        rem = (np.where(took, 0., r[0]), np.where(took, 0., r[1]))
        R.sample(hi, lo, lh, (rem[0] == 0.) & (rem[1] == 0.), tc)
    assert_bits(tw.state, ta.state, "the twin took the same steps")
    assert_bits(tw.dtime[0], ta.dtime[0])
    assert_bits(tw.dtime[1], ta.dtime[1])
    assert [r[3] for r in tw.propagate_res] == [r[3] for r in ta.propagate_res]
    return ta, out, R.out, log


@pytest.mark.gpu
@pytest.mark.parametrize("ha", [False, True])
@pytest.mark.parametrize("direction", [1., -1.])
def test_propagate_grid_bits(ha, direction):
    """Every grid output equals grid_covered()'s window sampled with eval_poly() at tau = (g - (t - last_h)).hi on the
    twin's steps: grid points on step boundaries (dyadic clamped steps) and inside steps, lanes done early (rem0 covers
    the rest), forward and backward grids (a grid has one direction in all lanes). grid[0] must be the current time, so
    the first sampling is on the zero-length step of the propagation to grid[0] (covering no later point). Also within
    the exact bound of the step the window picked."""
    n = 8
    rng = np.random.default_rng(12)
    st = np.array([rng.uniform(-2., 2., n), rng.uniform(-1., 1., n)])
    t0 = np.zeros(n)
    kind = np.arange(n) % 3
    span = direction * np.where(kind == 1, 0.75, 2.)                 # kind 1: done early
    n_pts = 33
    grid = np.linspace(0., 1., n_pts)[:, None] * span
    on_boundaries = kind != 2                                        # kind 2: points inside steps
    grid[:, on_boundaries] = np.round(grid[:, on_boundaries] * 64.) / 64.  # many points on the 2^-5 step boundaries
    mdt = np.full(n, 2.0 ** -5)
    ta, out, want, log = _twin_grid(sys_pendulum(), st, t0, grid, mdt, ha)
    assert not np.any(np.isnan(out))
    assert_bits(out, want, "propagate_grid()")
    # Exact bound: the window's step, rebuilt from the twin's capture (k = the first step whose window holds g).
    tcs = np.array([c[4] for c in log])
    for lane in sample_lanes(n, 4):
        for j in (n_pts // 3, n_pts - 2):
            g = grid[j, lane]
            found = False
            for k, (_, hi, lo, lh, _) in enumerate(log):
                a, b = sorted([Fraction(hi[lane]) + Fraction(lo[lane]) - Fraction(lh[lane]),
                               Fraction(hi[lane]) + Fraction(lo[lane])])
                if a <= Fraction(g) <= b and lh[lane] != 0.:
                    start = Fraction(hi[lane]) + Fraction(lo[lane]) - Fraction(lh[lane])
                    for i in range(2):
                        c = tcs[k, i, :, lane].tolist()
                        err = abs(float(Fraction(out[j, i, lane]) - exact_poly(c, Fraction(g) - start)))
                        assert err <= bound(c, Fraction(g) - start, ha)
                    found = True
                    break
            assert found, (lane, j)


@pytest.mark.gpu
def test_propagate_grid_reducing_boundary():
    """With the angle reducer, a grid point on a boundary where the angle was reduced takes the step that ends there
    (the window is closed): the output is unreduced there, unlike co(t) at the same time."""
    x, _ = hb.make_vars("x", "v")
    n = 2
    st = np.array([np.zeros(n), np.array([8., 9.])])
    mdt = 2.0 ** -6
    for ha in (False, True):
        ta = hb.taylor_adaptive_batch(sys_pendulum(), st, n, high_accuracy=ha)
        co = ta.propagate_until(2.0, c_output=True, max_delta_t=mdt, callback=hb.callback.angle_reducer([x]))
        tcs, t_hi, _ = recording(co)
        mode = COMPENSATED if ha else HORNER
        ends = np.array([evaluate(tcs, np.full(n, k), np.full(n, mdt), mode) for k in range(tcs.shape[0])])
        red = np.abs(ends[:-1, 0, :] - tcs[1:, 0, 0, :]) > 1.
        kb = np.array([np.nonzero(red[:, lane])[0][0] for lane in range(n)])  # step ending on the first reduction
        grid = np.array([np.zeros(n), (kb + 1) * mdt, np.full(n, 2.0)])
        tg = hb.taylor_adaptive_batch(sys_pendulum(), st, n, high_accuracy=ha)
        out = tg.propagate_grid(grid, max_delta_t=mdt, callback=hb.callback.angle_reducer([x]))
        want = ends[kb, :, np.arange(n)].T
        assert_bits(out[1], want, "the unreduced end of the step")
        assert np.all(out[1, 0] >= 2 * np.pi)
        assert np.all(co(grid[1])[0] != out[1, 0])


@pytest.mark.gpu
@pytest.mark.parametrize("ha", [False, True])
def test_update_d_output_bits(ha):
    """update_d_output(t) and update_d_output(t, rel_time=True) equal the restatement on ta.tc bit for bit and lie
    within the exact bound: tau inside the step, at 0 and last_h, outside it, and at a time near 2^40 with t_lo != 0."""
    n = 5
    rng = np.random.default_rng(21)
    st = np.array([rng.uniform(-2., 2., n), rng.uniform(-1., 1., n)])
    for t0 in (0., 2.0 ** 40 + 0.1):
        ta = hb.taylor_adaptive_batch(sys_pendulum(), st, n, time=t0, high_accuracy=ha)
        ta.propagate_until(t0 + 1.3, write_tc=True)
        ta.step(write_tc=True)
        t_hi, t_lo, lh, tc = ta.dtime[0].copy(), ta.dtime[1].copy(), ta.last_h.copy(), ta.tc.copy()
        if t0 != 0.:
            assert np.all(t_lo != 0.)
        start = [Fraction(t_hi[i]) + Fraction(t_lo[i]) - Fraction(lh[i]) for i in range(n)]
        for f in (0.37, 0., 1., -0.5, 1.5):
            rel = (f - 1.) * lh
            absolute = (t_hi - lh) + f * lh
            for rel_time, t in ((True, rel), (False, absolute)):
                got = ta.update_d_output(t, rel_time=rel_time).copy()
                want, tau = restate_d_output(tc, t, t_hi, t_lo, lh, ha, rel_time)
                assert_bits(got, want, "f = %g, rel_time = %s" % (f, rel_time))
                for i in range(n):
                    # rel_time: relative to the current time, so h* = last_h + t (rounded once, like h in bound()).
                    hs = Fraction(lh[i]) + Fraction(t[i]) if rel_time else Fraction(t[i]) - start[i]
                    for j in range(2):
                        c = tc[j, :, i].tolist()
                        err = abs(float(Fraction(got[j, i]) - exact_poly(c, hs)))
                        assert err <= bound(c, hs, ha), (f, rel_time, i, j)
