"""The angle reducer (callback.angle_reducer) without a GPU: the shared reduction (hy_reduce_angles(), the arithmetic the
kernels use) over hard inputs, against a numpy restatement (same bits) and against mpmath (congruence modulo fl(2pi));
the constructor's errors; the Python front end's host loop over the CPU oracle, against the same run with a numpy
callback."""
import math

import mpmath as mp
import numpy as np
import pytest

import heyoka_b200 as hb
import oracle

TWO_PI = 6.283185307179586  # fl(2 pi)
assert TWO_PI == float(2 * mp.pi)


def ref_reduce(x):
    """numpy restatement of angle_reduce.hpp::reduce_angle(): each operation rounded on its own."""
    x = np.float64(x)
    if not np.isfinite(x):
        return x
    r = x
    tp = np.float64(TWO_PI)
    while not (r >= 0.0 and r < tp):
        q = np.floor(r / tp)
        m = tp * q
        if np.isfinite(m):
            r = r - m
        else:
            q = q * np.float64(0.5)
            m2 = tp * q
            r = (r - m2) - m2
        if r < 0.0:
            r = r + tp
        if r >= tp:
            r = r - tp
    return r


def hard_inputs():
    xs = [0.0, -0.0, 5e-324, -5e-324, 2.2250738585072014e-308, -2.2250738585072014e-308, 1e-300, -1e-300, 1e-17, -1e-17,
          TWO_PI, -TWO_PI, math.pi, -math.pi, 1e300, -1e300, 1.7976931348623157e308, -1.7976931348623157e308]
    for k in list(range(-40, 41)) + [10 ** e for e in range(2, 18)] + [-(10 ** e) for e in range(2, 18)] + [2 ** 52, 2 ** 53]:
        c = k * TWO_PI
        xs += [c, np.nextafter(c, np.inf), np.nextafter(c, -np.inf)]
    for e in range(0, 301, 7):
        xs += [10.0 ** e, -(10.0 ** e), 3.7 * 10.0 ** e, -3.7 * 10.0 ** e]
    rng = np.random.default_rng(20261017)
    xs += list(rng.uniform(-1e3, 1e3, 2000)) + list(rng.uniform(-1e16, 1e16, 500))
    xs += list(np.ldexp(rng.uniform(-1, 1, 1000), rng.integers(-1074, 1023, 1000)))
    return np.array(xs, dtype=np.float64)


def reduce(x):
    y = np.ascontiguousarray(x, dtype=np.float64).copy()
    hb.callback.reduce_angles(y)
    return y


def test_reduction_range_and_bits():
    xs = hard_inputs()
    r = reduce(xs)
    assert np.all(np.isfinite(r))
    assert np.all((r >= 0.0) & (r < TWO_PI)), xs[~((r >= 0.0) & (r < TWO_PI))]
    ref = np.array([ref_reduce(x) for x in xs])
    assert np.array_equal(r.view(np.uint64), ref.view(np.uint64))
    # Values already in [0, 2pi), -0. included, are returned as they are.
    inside = (xs >= 0.0) & (xs < TWO_PI)
    assert np.array_equal(r[inside].view(np.uint64), xs[inside].view(np.uint64))


def test_reduction_congruence():
    mp.mp.prec = 2200  # exact for every double and the products involved
    tp = mp.mpf(TWO_PI)
    xs = hard_inputs()
    r = reduce(xs)
    for x, y in zip(xs.tolist(), r.tolist()):
        d = mp.mpf(x) - mp.mpf(y)
        k = mp.nint(d / tp)
        err = abs(d - k * tp)
        # Each pass's product k * fl(2pi) is rounded once: the result is congruent to x modulo fl(2pi) within a few
        # units in the last place of x (of 2pi for small x).
        bound = 4 * mp.mpf(math.ulp(max(abs(x), TWO_PI)))
        assert err <= bound, (x, y, err)


def test_non_finite_left_alone():
    xs = np.array([np.inf, -np.inf, np.nan])
    r = reduce(xs)
    assert np.isposinf(r[0]) and np.isneginf(r[1]) and np.isnan(r[2])


def test_constructor_errors():
    x, v = hb.make_vars("x", "v")
    with pytest.raises(ValueError, match="cannot be empty"):
        hb.callback.angle_reducer([])
    for bad in (x + v, hb.sin(x), hb.par[0], hb.expression(1.5), hb.time):
        with pytest.raises(ValueError, match="only variables"):
            hb.callback.angle_reducer([bad])
    ar = hb.callback.angle_reducer([x, v, x])
    assert [repr(e) for e in ar.vars] == ["x", "v"]


def _pendulum_with_event(state, batch):
    x, v = hb.make_vars("x", "v")
    sys = [(x, v), (v, -9.8 * hb.sin(x))]
    # A non-terminal event that never fires: the oracle serves integrators with events (the host loop).
    ev = hb.nt_event_batch(v - 1e6, lambda ta, t, d, i: None)
    return oracle.OracleEventIntegrator(sys, state, batch, nt_events=[ev]), x, v


def _numpy_cb(rows):
    def cb(ta):
        for i in rows:
            ta.state[i] = [ref_reduce(s) for s in ta.state[i]]
        return True
    return cb


@pytest.mark.parametrize("direction", [1.0, -1.0])
def test_front_end_host_loop_bitwise(direction):
    # Rotating pendulum above the separatrix (|v| > 2 sqrt(9.8)): the angle grows without bound.
    batch = 3
    st = np.array([[0.1, -2.0, 6.0], [7.0, -6.5, 8.0]])
    runs = []
    for cb_kind in ("reducer", "numpy"):
        ta, x, v = _pendulum_with_event(st.ravel(), batch)
        cb = hb.callback.angle_reducer([x]) if cb_kind == "reducer" else _numpy_cb([0])
        ta.propagate_until(direction * 3.0, callback=cb)
        runs.append((ta.state.copy(), ta.time.copy(), ta.last_h.copy(), list(ta.propagate_res)))
    (s0, t0, h0, p0), (s1, t1, h1, p1) = runs
    assert np.array_equal(s0.view(np.uint64), s1.view(np.uint64))
    assert np.array_equal(t0, t1) and np.array_equal(h0, h1) and p0 == p1
    assert np.all((s0[0] >= 0) & (s0[0] < TWO_PI))
    # Without the reducer the angle left [0, 2pi) (so the reduction did something).
    ta, _, _ = _pendulum_with_event(st.ravel(), batch)
    ta.propagate_until(direction * 3.0)
    assert np.any(ta.state[0] >= TWO_PI) or np.any(ta.state[0] < 0)
    k = (ta.state[0] - s0[0]) / TWO_PI
    assert np.allclose(k, np.round(k), atol=1e-9)


def test_front_end_not_a_state_variable():
    ta, x, _ = _pendulum_with_event([0.1, 7.0], 1)
    z = hb.make_vars("z")[0]
    before = ta.state.copy()
    with pytest.raises(ValueError, match="'z'.*not a state variable"):
        ta.propagate_until(1.0, callback=hb.callback.angle_reducer([x, z]))
    assert np.array_equal(ta.state, before) and ta.time[0] == 0.0
    with pytest.raises(ValueError, match="'z'.*not a state variable"):
        ta.propagate_grid([0.0, 1.0], callback=hb.callback.angle_reducer([z]))


def test_reducer_called_directly():
    ta, x, _ = _pendulum_with_event([20.0, 7.0], 1)
    assert hb.callback.angle_reducer([x])(ta) is True
    assert ta.state[0, 0] == ref_reduce(20.0) and ta.state[1, 0] == 7.0
