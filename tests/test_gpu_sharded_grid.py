"""propagate_grid() of a batch sharded over several devices (hy_batch_create_multi()) on the device: the shards run the
grid loop in lock-step and must give, bit for bit, what the single-device batch gives: the grid output (NaN positions
included), state, times, last_h, Taylor coefficients and propagate_res. Also: the front ends take the device path
(plain grid, events without a step callback, the angle reducer), the C ABI on a sharded batch and the C++ test
(tests/cpp/test_sharded_grid.cpp)."""
import os
import subprocess

import numpy as np
import pytest

import heyoka_b200 as hb
from common import outer_ss_batch_state, sys_outer_ss, sys_tutorial
from test_gpu_event_propagate import VARIANTS, check_same, run

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TWO_PI = 6.283185307179586
BLOW = 20  # the lane that goes non-finite: in the middle shard of [0, 0, 0]


def _device_lists():
    n = hb.lib.hy_device_count()
    lists = [[0, 0, 0]]  # three shards on one GPU, uneven blocks of 37 lanes
    if n > 1:
        lists.append(list(range(n)))
    return lists


def same(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return a.shape == b.shape and np.array_equal(a.view(np.uint64), b.view(np.uint64))


def check_equal(one, many, a, b):
    assert same(a, b)
    assert same(one.state, many.state)
    assert same(one.dtime[0], many.dtime[0]) and same(one.dtime[1], many.dtime[1])
    assert same(one.last_h, many.last_h)
    assert same(one.tc, many.tc)
    assert one.propagate_res == many.propagate_res


# ---- systems: (integrator factory, time scale of the grid) ----
def nbody(n, device, blow):
    st = outer_ss_batch_state(n)
    if blow == "first":
        st[6:9, BLOW] = st[0:3, BLOW]  # Jupiter at the Sun's position
    return hb.taylor_adaptive_batch(sys_outer_ss(), st, n, high_accuracy=True, device=device), 20.0


def pendulum(tape):
    def make(n, device, blow):
        # x' = v, v' = -9.8 sin(x) + p0 v^2: p0 = 1 and v0 = 3 make a lane blow up near t = 1/3.
        x, v = hb.make_vars("x", "v")
        sys = [(x, v), (v, -9.8 * hb.sin(x) + hb.par[0] * v * v)]
        rng = np.random.default_rng(5)
        st = np.vstack([rng.uniform(-1, 1, n), rng.uniform(-2, 2, n)])
        pars = np.zeros((1, n))
        if blow == "loop":
            st[:, BLOW], pars[0, BLOW] = (0.0, 3.0), 1.0
        elif blow == "first":
            st[1, BLOW], pars[0, BLOW] = 1e200, 1.0  # v' overflows
        return hb.taylor_adaptive_batch(sys, st, n, pars=pars, device=device, kernel={"tape": tape}), 5.0
    return make


def tutorial(n, device, blow):
    rng = np.random.default_rng(3)
    st = rng.uniform(-1, 1, (2, n))
    pars = rng.uniform(0.05, 0.3, (1, n))
    if blow == "first":
        st[1, BLOW], pars[0, BLOW] = 1e300, 1e10  # v' overflows
    return hb.taylor_adaptive_batch(sys_tutorial(), st, n, pars=pars, time=rng.uniform(0, 2, n), device=device), 5.0


SYSTEMS = {"nbody": nbody, "smem": pendulum("smem"), "global": pendulum("global"), "hbm": pendulum("hbm"),
           "tutorial": tutorial}

# case: (grid from (start times, scale), propagate_grid() keywords, blow-up)
CASES = {
    "forward": (lambda t0, T: t0 + np.linspace(0, T, 20)[:, None], {}, None),
    "backward": (lambda t0, T: t0 - np.linspace(0, T, 20)[:, None], {}, None),
    "per_lane": (lambda t0, T: t0 + np.linspace(0, T, 17)[:, None] * np.linspace(1, 1.3, t0.size), {}, None),
    "one_point": (lambda t0, T: t0[None, :], {}, None),
    "max_delta_t": (lambda t0, T: t0 + np.linspace(0, T, 20)[:, None], {"max_delta_t": "T/40"}, None),
    "max_steps_loop": (lambda t0, T: t0 + np.linspace(0, T, 20)[:, None], {"max_steps": 3}, None),
    "max_steps_first": (lambda t0, T: t0 + np.linspace(0, T, 20)[:, None], {"max_steps": 1}, None),
    "nonfinite_loop": (lambda t0, T: t0 + np.linspace(0, T, 20)[:, None], {}, "loop"),
    "nonfinite_first": (lambda t0, T: t0 + np.linspace(0, T, 20)[:, None], {}, "first"),
}


def grid_pair(system, case, n, devs):
    make, (gf, kw, blow) = SYSTEMS[system], CASES[case]
    (one, T), (many, _) = make(n, -1, blow), make(n, devs, blow)
    kw = {k: (T / 40 if v == "T/40" else v) for k, v in kw.items()}
    g = gf(one.time.copy(), T)
    return one, many, one.propagate_grid(g, **kw), many.propagate_grid(g, **kw)


@pytest.mark.parametrize("devs", _device_lists())
@pytest.mark.parametrize("system,case", [(s, c) for s in SYSTEMS for c in CASES
                                         if c != "nonfinite_loop" or s not in ("nbody", "tutorial")])
def test_sharded_equals_single_device(system, case, devs):
    # (No lane of the 6-body or the tutorial system goes non-finite inside the loop.)
    one, many, a, b = grid_pair(system, case, 37, devs)
    assert many._b.n_shards == min(len(devs), 37)
    if system == "nbody":
        assert one._b.kernel_info()["tape"] == many._b.kernel_info()["tape"] == "nbody"
    check_equal(one, many, a, b)
    oc = [r[0] for r in one.propagate_res]
    TO = hb.taylor_outcome
    if case == "nonfinite_loop":
        assert oc[BLOW] == TO.err_nf_state and not np.isnan(a[1]).any() and np.isnan(a[-1, :, BLOW]).all()
    elif case == "nonfinite_first":
        assert oc[BLOW] != TO.time_limit and np.isnan(a).all()
    elif case.startswith("max_steps"):
        assert set(oc) == {TO.step_limit} and np.isnan(a[-1]).all()
    else:
        assert not np.isnan(a).any()


def test_fewer_lanes_than_devices():
    one, many, a, b = grid_pair("smem", "per_lane", 2, [0, 0, 0])
    assert many._b.n_shards == 2
    check_equal(one, many, a, b)


def test_device_path_is_taken(monkeypatch):
    """No sharded grid runs the front end's host loop, and the transfers of a call do not grow with its iterations."""
    def refuse(*a, **k):
        raise AssertionError("host loop")
    monkeypatch.setattr(hb.taylor_adaptive_batch, "_propagate_grid_host", refuse)
    downloads = [0]
    orig = hb.Batch.download

    def counted(self, *a, **k):
        downloads[0] += 1
        return orig(self, *a, **k)
    monkeypatch.setattr(hb.Batch, "download", counted)

    counts = []
    for T in (1.0, 8.0):
        downloads[0] = 0
        ta, _ = pendulum("hbm")(37, [0, 0, 0], None)
        ta.propagate_grid(np.linspace(0, T, 30)[:, None] + ta.time)
        counts.append((downloads[0], max(r[3] for r in ta.propagate_res)))
    assert counts[0][0] == counts[1][0] and counts[1][1] > 2 * counts[0][1]

    # Events without a step callback.
    d = run(VARIANTS["basic"], "grid", 37, False, device=[0, 0, 0])
    assert d[1] is None and len(d[3]) > 0

    # The angle reducer.
    ta, _ = pendulum("smem")(37, [0, 0, 0], None)
    x = hb.expression(ta._sv_names[0])
    ta.propagate_grid(np.linspace(0, 3, 13)[:, None] + ta.time, callback=hb.callback.angle_reducer([x]))
    assert np.all((ta.state[0] >= 0) & (ta.state[0] < TWO_PI))


EV_VARIANTS = ["basic", "backward", "max_delta_t", "max_steps", "nonfinite", "stop_one_lane", "stop_no_callback",
               "damped", "writes_state", "cooldown", "raise_two", "raise_first_step"]


@pytest.mark.parametrize("variant", EV_VARIANTS)
def test_events_sharded_equals_single_device_and_host_loop(variant):
    spec = VARIANTS[variant]
    many = run(spec, "grid", 37, False, device=[0, 0, 0])
    check_same(many, run(spec, "grid", 37, False))
    check_same(many, run(spec, "grid", 37, True, device=[0, 0, 0]))


def rotating_blowup(n, device, tape):
    """A pendulum whose lane 5 gains a v^2 term and blows up near t = 0.45 while the other lanes rotate fast (|v|
    around 7): in the iteration that ends non-finite, lanes of every shard cross 0 or 2pi."""
    x, v = hb.make_vars("x", "v")
    sys = [(x, v), (v, -9.8 * hb.sin(x) + hb.par[0] * v * v)]
    rng = np.random.default_rng(11)
    xs, vs = rng.uniform(-7, 7, n), (6.5 + rng.random(n)) * np.where(np.arange(n) % 2, -1, 1)
    p = np.zeros(n)
    xs[5], vs[5], p[5] = -np.pi / 2, 1.0, 1.0
    return hb.taylor_adaptive_batch(sys, np.concatenate([xs, vs]), n, pars=p, device=device,
                                    kernel={"tape": tape})


@pytest.mark.parametrize("devs", _device_lists())
@pytest.mark.parametrize("tape", ["smem", "global", "hbm"])
def test_angle_reducer(tape, devs):
    n = 96
    res = []
    for dev in (-1, devs):
        ta = rotating_blowup(n, dev, tape)
        x = hb.expression(ta._sv_names[0])
        out = ta.propagate_grid(ta.time[None, :] + np.linspace(0, 100, 13)[:, None],
                                callback=hb.callback.angle_reducer([x]))
        res.append((ta, out))
    (one, a), (many, b) = res
    check_equal(one, many, a, b)
    assert one.propagate_res[5][0] == hb.taylor_outcome.err_nf_state
    # The last iteration was not reduced in any shard: lanes far from lane 5's shard were left outside [0, 2pi).
    xo = many.state[0, n // 2:]
    assert np.any(np.isfinite(xo) & ((xo < 0) | (xo >= TWO_PI)))


def test_nbody_refuses_angles_on_a_sharded_batch():
    ta, _ = nbody(37, [0, 0, 0], None)
    ta._push()
    ta._b.set_angles([0])
    n0 = ta._b.launch_count()
    with pytest.raises(NotImplementedError, match="N-body"):
        ta._b.propagate_grid(np.vstack([ta.time, ta.time + 1.0]))
    assert ta._b.launch_count() == n0
    ta._b.set_angles([])


def _c_abi_batch(devs, events):
    x, v = hb.make_vars("x", "v")
    n = 37
    P = hb.Program([(x, v), (v, -9.8 * hb.sin(x))], events=[v] if events else ())
    b = hb.Batch(P, n, device=devs)
    if events:
        b.set_events(1, [0], [-1.0], 2.2e-16)
    b.upload(np.vstack([np.linspace(0.1, 1.5, n), np.zeros(n)]), None, np.zeros(n), np.zeros(n))
    return b


@pytest.mark.parametrize("events", [False, True])
def test_c_abi(events):
    n = 37
    grid = np.linspace(0, 4, 30)[:, None] * np.linspace(1, 1.5, n)
    logs, outs, batches = [], [], []
    for devs in (-1, [0, 0, 0]):
        b = _c_abi_batch(devs, events)
        if events:
            log = []

            def on_events(evs, th, tl, cont, log=log):
                log.append((list(evs), list(th[:len(evs)]), list(tl[:len(evs)])))
                for m in range(len(evs)):
                    cont[m] = 1
            out, err = b.propagate_grid_ev(grid, None, 0, on_events)
            assert err is None
            logs.append(log)
        else:
            out = b.propagate_grid(grid)
        outs.append(out)
        batches.append(b)
    assert same(outs[0], outs[1])
    one, many = batches
    for p, q in zip(one.download(), many.download()):
        assert same(p, q)
    for p, q in zip(one.prop_res(), many.prop_res()):
        assert np.array_equal(p, q)
    assert same(one.tc(), many.tc())
    if events:
        assert logs[0] == logs[1] and len(logs[0]) > 0

    # A bad argument: the single-device message, before any launch.
    never = lambda evs, th, tl, cont: pytest.fail("called back")  # noqa: E731
    t = one.download()[1]
    for bad, msg in ((np.vstack([t + 0.5, t + 1.0]), "must match the current time"),
                     (np.vstack([t, t + 1.0, t + 1.0]), "non-monotonic")):
        for b in batches:
            n0 = b.launch_count()
            with pytest.raises(ValueError, match=msg):
                b.propagate_grid_ev(bad, None, 0, never) if events else b.propagate_grid(bad)
            assert b.launch_count() == n0


def test_cpp_sharded_grid():
    lib = os.path.join(ROOT, "heyoka_b200", "lib")
    exe = os.path.join(ROOT, "build", "test_sharded_grid")
    os.makedirs(os.path.dirname(exe), exist_ok=True)
    subprocess.run(["g++", "-std=c++17", "-O1", "-I" + os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "cpp", "test_sharded_grid.cpp"), "-o", exe, "-L" + lib,
                    "-lheyoka_b200", "-Wl,-rpath," + lib], check=True)
    res = subprocess.run([exe, "gpu"], capture_output=True, text=True, timeout=900)
    assert res.returncode == 0 and "ALL PASSED (gpu)" in res.stdout, res.stdout[-3000:] + res.stderr[-2000:]
