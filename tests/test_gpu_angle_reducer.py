"""The angle reducer on the device (hy_batch_set_angles(): k_coop / k_hbm reduce inside the propagation loops) against
the host loop (the reducer wrapped in a function, an ordinary step callback), bit for bit: state, time, last_h,
propagate_res, tc. Also the C++ test (tests/cpp/test_angle_reducer.cpp)."""
import os
import subprocess

import numpy as np
import pytest

import heyoka_b200 as hb

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "build", "test_angle_reducer")
TWO_PI = 6.283185307179586
TAPES = ["auto", "smem", "global", "global-cta", "hbm"]


def _build_cpp():
    src = os.path.join(ROOT, "tests", "cpp", "test_angle_reducer.cpp")
    lib = os.path.join(ROOT, "heyoka_b200", "lib")
    os.makedirs(os.path.dirname(EXE), exist_ok=True)
    if not os.path.exists(EXE) or os.path.getmtime(EXE) < max(os.path.getmtime(src), os.path.getmtime(
            os.path.join(lib, "libheyoka_b200.so"))):
        subprocess.run(["g++", "-std=c++17", "-O1", "-I" + os.path.join(ROOT, "include"), src, "-o", EXE, "-L" + lib,
                        "-lheyoka_b200", "-Wl,-rpath," + lib], check=True)
    return EXE


def test_cpp_angle_reducer_cpu():
    res = subprocess.run([_build_cpp(), "cpu"], capture_output=True, text=True)
    assert res.returncode == 0 and "ALL PASSED (cpu)" in res.stdout, res.stdout + res.stderr


@pytest.mark.gpu
def test_cpp_angle_reducer_gpu():
    res = subprocess.run([_build_cpp(), "gpu"], capture_output=True, text=True, timeout=900)
    assert res.returncode == 0 and "ALL PASSED (gpu)" in res.stdout, res.stdout[-3000:] + res.stderr[-2000:]


def pendulum(tape, batch=37, **kw):
    x, v = hb.make_vars("x", "v")
    sys = [(x, v), (v, -9.8 * hb.sin(x))]
    rng = np.random.default_rng(5)
    # Rotating above the separatrix (|v| > 2 sqrt(9.8)) in both senses, plus a few librating lanes.
    v0 = np.where(np.arange(batch) % 3 == 0, 1.5, 6.3 + 3 * rng.random(batch)) * np.where(np.arange(batch) % 2, -1, 1)
    st = np.concatenate([rng.uniform(-10, 10, batch), v0])
    ta = hb.taylor_adaptive_batch(sys, st, batch, kernel=None if tape == "auto" else {"tape": tape}, **kw)
    return ta, [0]


def forced(tape, batch=19):
    x, v = hb.make_vars("x", "v")
    sys = [(x, v), (v, -hb.par[0] * hb.sin(x) + 0.3 * hb.cos(hb.time))]
    rng = np.random.default_rng(7)
    st = np.concatenate([rng.uniform(-3, 3, batch), 7 + rng.random(batch)])
    ta = hb.taylor_adaptive_batch(sys, st, batch, pars=rng.uniform(5, 10, batch),
                                  kernel=None if tape == "auto" else {"tape": tape})
    return ta, [0]


def variational(tape, batch=11):
    x, v = hb.make_vars("x", "v")
    vs = hb.var_ode_sys([(x, v), (v, -9.8 * hb.sin(x))], hb.var_args.vars)
    rng = np.random.default_rng(9)
    st = np.concatenate([rng.uniform(-3, 3, batch), 7 + rng.random(batch)])
    ta = hb.taylor_adaptive_batch(vs, st, batch, kernel=None if tape == "auto" else {"tape": tape})
    return ta, [0]


SYSTEMS = {"pendulum": pendulum, "forced": forced, "variational": variational}


def launches(ta):
    return ta._b.launch_count()


def run(make, tape, device, call):
    ta, rows = make(tape)
    x = hb.expression(ta._sv_names[rows[0]])
    ar = hb.callback.angle_reducer([x])
    cb = ar if device else (lambda t: ar(t))
    l0 = launches(ta)
    out = call(ta, cb)
    return ta, out, launches(ta) - l0, rows


def same(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return a.shape == b.shape and np.array_equal(a.view(np.uint64), b.view(np.uint64))


def check_pair(d, h, check_tc=True, in_range=True):
    """Device path d against host path h, bit for bit. in_range: the listed rows are in [0, 2pi) where finite (not after
    an iteration that ended non-finite, which the reference does not reduce)."""
    (td, od, ld, rows), (th, oh, lh, _) = d, h
    assert same(td.state, th.state)
    assert same(td.time, th.time) and same(td.dtime[1], th.dtime[1])
    assert same(td.last_h, th.last_h)
    assert td.propagate_res == th.propagate_res
    if check_tc:
        assert same(td.tc, th.tc)
    if in_range:
        fin = np.isfinite(td.state[rows])
        assert np.all((td.state[rows][fin] >= 0) & (td.state[rows][fin] < TWO_PI))
    steps = max(r[3] for r in th.propagate_res)
    assert lh >= steps
    return od, oh, ld, steps


CALLS = {
    "until": lambda ta, cb: ta.propagate_until(3.0, callback=cb, write_tc=True),
    "until_back": lambda ta, cb: ta.propagate_until(-3.0, callback=cb, write_tc=True),
    "for": lambda ta, cb: ta.propagate_for(2.5, callback=cb, write_tc=True),
    "mdt": lambda ta, cb: ta.propagate_until(2.0, callback=cb, max_delta_t=0.05, write_tc=True),
    "max_steps": lambda ta, cb: ta.propagate_until(50.0, callback=cb, max_steps=9, write_tc=True),
}


@pytest.mark.gpu
@pytest.mark.parametrize("tape", TAPES)
@pytest.mark.parametrize("system", list(SYSTEMS))
@pytest.mark.parametrize("path", list(CALLS))
def test_propagate_device_vs_host(tape, system, path):
    d = run(SYSTEMS[system], tape, True, CALLS[path])
    h = run(SYSTEMS[system], tape, False, CALLS[path])
    _, _, ld, steps = check_pair(d, h)
    assert steps > 8 and ld <= 8  # the device path's launches do not grow with the steps


@pytest.mark.gpu
@pytest.mark.parametrize("tape", TAPES)
def test_unreduced_differs_by_turns(tape):
    ta, _, _, _ = run(pendulum, tape, True, CALLS["until"])
    tu, _ = pendulum(tape)
    tu.propagate_until(3.0)
    k = (tu.state[0] - ta.state[0]) / TWO_PI
    assert np.any(np.abs(k) >= 1)
    assert np.allclose(k, np.round(k), atol=1e-6)
    assert np.allclose(tu.state[1], ta.state[1], rtol=1e-8, atol=1e-8)


def blowup(tape, batch=64):
    """A pendulum whose lane 5 gains a v^2 term and blows up near t = 0.45, after about 180 shrinking steps, while the
    other lanes rotate fast (|v| around 7) towards a final time far beyond: in the iteration that ends non-finite some
    of them cross 0 or 2pi, so reducing that iteration or not shows in the bits."""
    x, v = hb.make_vars("x", "v")
    sys = [(x, v), (v, -9.8 * hb.sin(x) + hb.par[0] * v * v)]
    rng = np.random.default_rng(11)
    xs, vs = rng.uniform(-7, 7, batch), (6.5 + rng.random(batch)) * np.where(np.arange(batch) % 2, -1, 1)
    p = np.zeros(batch)
    xs[5], vs[5], p[5] = -np.pi / 2, 1.0, 1.0
    ta = hb.taylor_adaptive_batch(sys, np.concatenate([xs, vs]), batch, pars=p,
                                  kernel=None if tape == "auto" else {"tape": tape})
    return ta, [0]


def check_nonfinite_exit(d, h):
    """The run ended non-finite, and the host path left some finite angle of another lane outside [0, 2pi): the last
    iteration was not reduced, and the device path matched that."""
    td, th = d[0], h[0]
    assert any(r[0] == hb.taylor_outcome.err_nf_state for r in td.propagate_res)
    x = np.delete(th.state[0], 5)
    assert np.any(np.isfinite(x) & ((x < 0) | (x >= TWO_PI)))


@pytest.mark.gpu
@pytest.mark.parametrize("tape", TAPES)
def test_nonfinite_lane(tape):
    def make(t):
        x, v = hb.make_vars("x", "v")
        # v' = v^2: v = v0 / (1 - v0 t) blows up at t = 1 / v0 in the lane with v0 = 3.
        sys = [(x, v), (v, v * v + 0.0 * x)]
        n = 9
        st = np.concatenate([np.linspace(-20, 20, n), np.where(np.arange(n) == 4, 3.0, 0.01)])
        return hb.taylor_adaptive_batch(sys, st, n, kernel=None if t == "auto" else {"tape": t}), [0]

    def call(ta, cb):
        return ta.propagate_until(5.0, callback=cb, write_tc=True)
    d, h = run(make, tape, True, call), run(make, tape, False, call)
    check_pair(d, h)
    assert any(r[0] == hb.taylor_outcome.err_nf_state for r in d[0].propagate_res)


@pytest.mark.gpu
@pytest.mark.parametrize("tape", TAPES)
@pytest.mark.parametrize("path", ["until", "grid", "c_output"])
def test_nonfinite_exit_with_rotating_lanes(tape, path):
    def call(ta, cb):
        if path == "until":
            return ta.propagate_until(100.0, callback=cb, write_tc=True)
        if path == "grid":
            return ta.propagate_grid(ta.time[None, :] + np.linspace(0, 100, 13)[:, None], callback=cb)
        return ta.propagate_until(100.0, callback=cb, c_output=True)
    d, h = run(blowup, tape, True, call), run(blowup, tape, False, call)
    od, oh, _, _ = check_pair(d, h, check_tc=path != "grid", in_range=False)
    check_nonfinite_exit(d, h)
    if path == "grid":
        assert same(od, oh)
    elif path == "c_output":
        assert same(od.get_times(), oh.get_times()) and same(od.get_tcs(), oh.get_tcs())


@pytest.mark.gpu
@pytest.mark.parametrize("tape", TAPES)
@pytest.mark.parametrize("system", list(SYSTEMS))
def test_grid_device_vs_host(tape, system):
    def call(ta, cb):
        g = ta.time[None, :] + np.linspace(0, 3, 13)[:, None]
        return ta.propagate_grid(g, callback=cb)
    d, h = run(SYSTEMS[system], tape, True, call), run(SYSTEMS[system], tape, False, call)
    od, oh, _, _ = check_pair(d, h, check_tc=False)
    assert same(od, oh)


@pytest.mark.gpu
@pytest.mark.parametrize("tape", TAPES)
def test_c_output_device_vs_host(tape):
    def call(ta, cb):
        return ta.propagate_until(3.0, callback=cb, c_output=True)
    d, h = run(pendulum, tape, True, call), run(pendulum, tape, False, call)
    cd, ch, _, _ = check_pair(d, h)
    assert same(cd.get_times(), ch.get_times()) and same(cd.get_tcs(), ch.get_tcs())
    tm = np.full(d[0].get_batch_size(), 1.234)
    assert same(cd(tm), ch(tm))


@pytest.mark.gpu
def test_sharded_vs_single():
    def make_dev(devs):
        def make(tape):
            ta, rows = pendulum(tape, device=devs)
            return ta, rows
        return make
    s = run(make_dev(-1), "auto", True, CALLS["until"])
    m = run(make_dev([0, 0, 0]), "auto", True, CALLS["until"])
    assert m[0]._b.n_shards == 3
    assert same(s[0].state, m[0].state) and same(s[0].time, m[0].time) and s[0].propagate_res == m[0].propagate_res


@pytest.mark.gpu
def test_step_does_not_reduce():
    ta, _ = pendulum("auto")
    ta.state[0] = 50.0
    ta._push()
    ta._b.set_angles([0])
    ta._b.step()
    st, _, _, _ = ta._b.download()
    ta._b.set_angles([])
    assert np.all(st[0] > TWO_PI)


@pytest.mark.gpu
def test_nbody_takes_host_path():
    sys = hb.model.nbody(2)
    x0 = sys[0][0]
    # Two unit masses one unit apart on a bound orbit (per body: x, y, z, vx, vy, vz).
    st = np.array([0, 0, 0, 0, -0.5, 0, 1, 0, 0, 0, 0.5, 0], dtype=float)
    b = 4
    state = np.repeat(st[:, None], b, axis=1) * (1 + 0.01 * np.arange(b))
    runs = []
    for wrap in (False, True):
        ta = hb.taylor_adaptive_batch(sys, state.ravel(), b)
        assert ta._b.kernel_info()["tape"].startswith("nbody")
        ar = hb.callback.angle_reducer([x0])
        l0 = launches(ta)
        ta.propagate_until(4.0, callback=(lambda t: ar(t)) if wrap else ar)
        runs.append((ta, launches(ta) - l0))
    (a, la), (c, lc) = runs
    assert same(a.state, c.state) and a.propagate_res == c.propagate_res
    steps = max(r[3] for r in a.propagate_res)
    assert la >= steps and lc >= steps
    assert np.all((a.state[0] >= 0) & (a.state[0] < TWO_PI))
    # The C ABI refuses the list on the N-body kernel.
    a._b.set_angles([0])
    with pytest.raises(NotImplementedError):
        a._b.propagate_until(np.full(b, 5.0))
    a._b.set_angles([])


@pytest.mark.gpu
def test_errors():
    ta, _ = pendulum("auto")
    z = hb.make_vars("z")[0]
    with pytest.raises(ValueError, match="'z'"):
        ta.propagate_until(1.0, callback=hb.callback.angle_reducer([z]))
    assert np.all(ta.time == 0)
    for bad in ([2], [0, 0], [5, 0]):
        with pytest.raises(ValueError):
            ta._b.set_angles(bad)


@pytest.mark.gpu
def test_events_with_reducer_against_oracle():
    import oracle
    x, v = hb.make_vars("x", "v")
    sys = [(x, v), (v, -9.8 * hb.sin(x))]
    st = [0.1, -2.0, 6.0, 7.0, -6.5, 8.0]
    res = []
    for mk in (hb.taylor_adaptive_batch, oracle.OracleEventIntegrator):
        hits = []
        ev = hb.nt_event_batch(v - 7.5, lambda ta, t, d, i: hits.append((i, t)))
        ta = mk(sys, st, 3, nt_events=[ev])
        ta.propagate_until(3.0, callback=hb.callback.angle_reducer([x]))
        res.append((ta.state.copy(), ta.time.copy(), sorted(hits)))
    # (Events run the host loop on both; the device jet and the oracle's agree to a few ulp, not always to the bit.)
    assert np.allclose(res[0][0], res[1][0], rtol=1e-11, atol=1e-11) and same(res[0][1], res[1][1])
    assert [i for i, _ in res[0][2]] == [i for i, _ in res[1][2]]
    assert np.allclose([t for _, t in res[0][2]], [t for _, t in res[1][2]], rtol=1e-12)
    assert np.all((res[0][0][0] >= 0) & (res[0][0][0] < TWO_PI))
