"""propagate_until() / propagate_for() / propagate_grid() / continuous output of integrators with events, run on the
device (hy_batch_propagate_until_ev() / hy_batch_propagate_grid_ev()), against the front end's host lock-step loop,
bit for bit. The host loop is forced by a step callback that returns True and touches nothing; with no step callback
the front end takes the device loop. Also: sharded batches, the CPU oracle, the transfers of a call and the C ABI."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import heyoka_b200 as hb
from heyoka_b200 import _capi
import oracle

pytestmark = pytest.mark.gpu

TO = hb.taylor_outcome


class Spec:
    """A pendulum x' = v, v' = -9.8 sin(x) - p0 v + p1 v^2 with a non-terminal event at every zero of x and a terminal
    event at every zero of v, and what its callbacks do."""

    def __init__(self, backward=False, mdt=None, max_steps=0, blowup=False, stop_lane=None, damped=False, write=False,
                 cooldown=-1.0, raise_lanes=(), alter_lane=None, no_te_cb=False, tf=6.0, raise_at=2, early=False):
        self.backward, self.mdt, self.max_steps, self.blowup = backward, mdt, max_steps, blowup
        self.stop_lane, self.damped, self.write, self.cooldown = stop_lane, damped, write, cooldown
        self.raise_lanes, self.alter_lane, self.no_te_cb, self.tf = raise_lanes, alter_lane, no_te_cb, tf
        self.raise_at, self.early = raise_at, early  # early: the raising lanes start next to a zero of x


VARIANTS = {
    "basic": Spec(),
    "backward": Spec(backward=True),
    "max_delta_t": Spec(mdt=0.05),
    "max_steps": Spec(max_steps=7),
    "nonfinite": Spec(blowup=True),
    "stop_one_lane": Spec(stop_lane=3),
    "stop_no_callback": Spec(no_te_cb=True),
    "damped": Spec(damped=True),
    "writes_state": Spec(write=True),
    "cooldown": Spec(cooldown=0.3, mdt=0.02, tf=2.0),
    "raise_one": Spec(raise_lanes=(2,)),
    "raise_two": Spec(raise_lanes=(2, 7)),
    "alters_time": Spec(alter_lane=4),
    "raise_first_step": Spec(raise_lanes=(2,), raise_at=1, early=True),
}


def make(spec, n, log, device=-1, seed=1, ctor=None):
    x, v = hb.make_vars("x", "v")
    sys = [(x, v), (v, -9.8 * hb.sin(x) - hb.par[0] * v + hb.par[1] * v * v)]
    rng = np.random.default_rng(seed)
    st = np.vstack([0.05 + 0.5 * rng.random(n), 0.2 * rng.random(n) - 0.1])
    pars = np.zeros((2, n))
    if spec.blowup:
        st[:, 5], pars[1, 5] = (0.0, 3.0), 1.0  # v' ~ v^2: non-finite near t = 1/3
    if spec.early:
        for i in spec.raise_lanes:
            st[:, i] = (1e-3, -0.5)
    count = {}

    def ncb(ta, t, d_sgn, i):
        log.append(("nt", i, t, d_sgn))
        k = count[("nt", i)] = count.get(("nt", i), 0) + 1
        if i in spec.raise_lanes and k == spec.raise_at:
            raise ValueError("lane %d refuses" % i)
        if spec.write:
            ta.state[1, i] *= 0.999

    def tcb(ta, d_sgn, i):
        hi, lo = ta.dtime
        log.append(("te", i, float(hi[i]), float(lo[i]), d_sgn))
        k = count[("te", i)] = count.get(("te", i), 0) + 1
        if spec.damped:
            ta.pars[0, i] = 0.5 if ta.pars[0, i] == 0 else 0.
        if spec.alter_lane == i and k == 2:
            ta.time[i] += 1.0
        return not (i == spec.stop_lane and k == 3)

    te = hb.t_event_batch(v, callback=None if spec.no_te_cb else tcb, cooldown=spec.cooldown)
    if ctor is None:
        return hb.taylor_adaptive_batch(sys, st, n, pars=pars, device=device, t_events=[te],
                                        nt_events=[hb.nt_event_batch(x, ncb)])
    return ctor(sys, st, n, pars=pars, t_events=[te], nt_events=[hb.nt_event_batch(x, ncb)])


def snapshot(ta, n_ev=2):
    cd = ta.te_cooldowns
    return dict(state=ta.state.copy(), t_hi=ta.dtime[0].copy(), t_lo=ta.dtime[1].copy(), last_h=ta.last_h.copy(),
                tc=ta.tc.copy(), tc_ev=ta._b.tc_events(n_ev), step_res=list(ta.step_res), prop_res=list(ta.propagate_res),
                pars=ta.pars.copy(), cooldowns=cd)


def same(a, b):
    if isinstance(a, np.ndarray):
        return a.shape == b.shape and np.array_equal(a.view(np.int64), b.view(np.int64))
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(same(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(same(p, q) for p, q in zip(a, b))
    if isinstance(a, float):
        return np.float64(a).view(np.int64) == np.float64(b).view(np.int64)
    return a == b


def run(spec, mode, n, host, device=-1):
    """One call on a fresh integrator; returns (result, exception, snapshot, callback log)."""
    log = []
    ta = make(spec, n, log, device=device)
    kw = dict(max_steps=spec.max_steps, max_delta_t=spec.mdt)
    if host:
        kw["callback"] = lambda ta: True
    tf = -spec.tf if spec.backward else spec.tf
    res = exc = None
    try:
        if mode == "until":
            res = ta.propagate_until(tf, **kw)
        elif mode == "for":
            res = ta.propagate_for(tf, **kw)
        elif mode == "cout":
            co = ta.propagate_until(tf, c_output=True, **kw)
            res = None if co is None else (co.get_times(), co.get_tcs())
        else:
            grid = np.repeat(np.linspace(0., tf, 25)[:, None], n, axis=1)
            res = ta.propagate_grid(grid, **kw)
    except Exception as e:  # noqa: BLE001 - compared below
        exc = e
    return res, exc, snapshot(ta), log


def check_same(d, h):
    rd, ed, sd, ld = d
    rh, eh, sh, lh = h
    assert (type(ed), str(ed)) == (type(eh), str(eh))
    assert same(ld, lh)
    for k in sd:
        assert same(sd[k], sh[k]), k
    assert (rd is None) == (rh is None)
    if rd is not None:
        assert same(list(rd) if isinstance(rd, tuple) else rd, list(rh) if isinstance(rh, tuple) else rh)


@pytest.mark.parametrize("mode", ["until", "for", "grid", "cout"])
@pytest.mark.parametrize("variant", sorted(VARIANTS))
def test_device_loop_equals_host_loop(variant, mode):
    spec = VARIANTS[variant]
    d, h = run(spec, mode, 37, False), run(spec, mode, 37, True)
    check_same(d, h)
    n_te = sum(1 for e in d[3] if e[0] == "te")
    assert n_te > 0 or variant in ("stop_no_callback", "nonfinite", "max_steps")
    if variant == "nonfinite":
        assert any(r[0] == TO.err_nf_state for r in d[2]["prop_res"]) or mode == "grid"
    if variant in ("raise_one", "raise_two", "alters_time", "raise_first_step"):
        assert d[1] is not None


def test_device_loop_equals_host_loop_65536_lanes():
    # (The host grid loop's own propagate_until() to grid[0] has no step callback: it takes the device loop. It is a
    # zero-length step, as the grid starts at the current time.)
    for spec in (Spec(tf=0.6), Spec(tf=0.6, raise_lanes=(40000,), raise_at=1)):
        for mode in ("until", "grid"):
            d, h = run(spec, mode, 1 << 16, False), run(spec, mode, 1 << 16, True)
            check_same(d, h)
            assert (d[1] is not None) == bool(spec.raise_lanes)


def test_six_body_close_approach():
    """The 6-body system (the N-body kernel's program; an event batch runs its steps on k_ev_jet) with a terminal event
    at a close approach of Jupiter and Saturn whose callback continues, device loop against host loop."""
    from common import outer_ss_batch_state, sys_outer_ss
    sys = sys_outer_ss()
    xs = [lhs for lhs, _ in sys]
    d2 = hb.sum([(xs[6 + k] - xs[12 + k]) * (xs[6 + k] - xs[12 + k]) for k in range(3)])
    res = []
    for host in (False, True):
        log = []

        def cb(ta, d_sgn, i, log=log):
            log.append((i, float(ta.time[i]), d_sgn))
            return True
        ta = hb.taylor_adaptive_batch(sys, outer_ss_batch_state(40), 40, high_accuracy=True,
                                      t_events=[hb.t_event_batch(d2 - 49.0, callback=cb)])
        ta.propagate_until(30.0, **({"callback": lambda ta: True} if host else {}))
        res.append((None, None, snapshot(ta, n_ev=1), log))
    check_same(res[0], res[1])
    assert len(res[0][3]) >= 40


def test_continuous_output_on_non_current_device():
    if hb.lib.hy_device_count() < 2:
        pytest.skip("needs a second GPU")
    spec = VARIANTS["basic"]
    log_a, log_b = [], []
    a, b = make(spec, 37, log_a, device=1), make(spec, 37, log_b, device=0)
    ca, cb = a.propagate_until(spec.tf, c_output=True), b.propagate_until(spec.tf, c_output=True)
    assert same(ca.get_tcs(), cb.get_tcs()) and same(ca(3.0).copy(), cb(3.0).copy())


def test_cpp_event_propagate():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    lib = os.path.join(root, "heyoka_b200", "lib")
    exe = os.path.join(root, "build", "test_event_propagate")
    os.makedirs(os.path.dirname(exe), exist_ok=True)
    subprocess.run(["g++", "-std=c++17", "-O1", "-I" + os.path.join(root, "include"),
                    os.path.join(root, "tests", "cpp", "test_event_propagate.cpp"), "-o", exe, "-L" + lib,
                    "-lheyoka_b200", "-Wl,-rpath," + lib], check=True)
    res = subprocess.run([exe, "gpu"], capture_output=True, text=True, timeout=900)
    assert res.returncode == 0 and "ALL PASSED (gpu)" in res.stdout, res.stdout[-3000:] + res.stderr[-2000:]


@pytest.mark.parametrize("variant", ["basic", "nonfinite", "stop_one_lane", "max_steps", "raise_two", "damped"])
@pytest.mark.parametrize("mode", ["until", "for"])
def test_sharded_equals_single_device(variant, mode):
    spec = VARIANTS[variant]
    check_same(run(spec, mode, 37, False, device=[0, 0, 0]), run(spec, mode, 37, False))


def test_device_loop_vs_oracle():
    spec = Spec(tf=10.0)
    lg, lo = [], []
    g = make(spec, 16, lg)
    o = make(spec, 16, lo, ctor=oracle.OracleEventIntegrator)
    g.propagate_until(spec.tf)
    o.propagate_until(spec.tf)
    assert [e[:2] + e[-1:] for e in lg] == [e[:2] + e[-1:] for e in lo]
    for a, b in zip(lg, lo):
        assert abs(a[2] - b[2]) <= 1e-11 * max(1.0, abs(b[2]))
    assert [r[0] for r in g.propagate_res] == [r[0] for r in o.propagate_res]
    assert np.max(np.abs(g.state - o.state)) < 1e-11
    assert np.max(np.abs(g.time - o.time)) < 1e-12


def test_transfers(monkeypatch):
    calls = {"download": 0, "tc": 0}
    for name in calls:
        orig = getattr(hb.Batch, name)

        def counted(self, *a, _orig=orig, _name=name, **k):
            calls[_name] += 1
            return _orig(self, *a, **k)
        monkeypatch.setattr(hb.Batch, name, counted)
    x, v = hb.make_vars("x", "v")
    sys = [(x, v), (v, -9.8 * hb.sin(x))]
    st = np.vstack([np.linspace(0.1, 0.5, 40), np.zeros(40)])
    seen = []
    ta = hb.taylor_adaptive_batch(sys, st, 40, nt_events=[hb.nt_event_batch(v, lambda ta, t, s, i: seen.append(i))])
    ta.propagate_until(20.0)
    assert len(seen) > 100
    assert calls == {"download": 1, "tc": 1}
    th = hb.taylor_adaptive_batch(sys, st, 40, nt_events=[hb.nt_event_batch(v, lambda ta, t, s, i: None)])
    calls.update(download=0, tc=0)
    th.propagate_until(20.0, callback=lambda ta: True)
    iters = calls["download"]
    assert iters > 10 and calls["tc"] == iters
    assert same(ta.state, th.state)

    # A callback that reads the state sees the values of the host loop.
    def reader(out):
        return lambda ta, t, s, i: out.append(ta.state[:, i].copy())
    rd, rh = [], []
    a = hb.taylor_adaptive_batch(sys, st, 40, nt_events=[hb.nt_event_batch(v, reader(rd))])
    b = hb.taylor_adaptive_batch(sys, st, 40, nt_events=[hb.nt_event_batch(v, reader(rh))])
    a.propagate_until(5.0)
    b.propagate_until(5.0, callback=lambda ta: True)
    assert len(rd) == len(rh) > 0 and all(same(p, q) for p, q in zip(rd, rh))


def test_c_abi_checks():
    x, v = hb.make_vars("x", "v")
    P = hb.Program([(x, v), (v, -9.8 * hb.sin(x))], events=[v])
    b = hb.Batch(P, 8)
    b.set_events(1, [0], [-1.0], 2.2e-16)
    b.upload(np.vstack([np.full(8, 0.1), np.zeros(8)]), None, np.zeros(8), np.zeros(8))
    lib = _capi.lib
    tf = np.full(8, 1.0)
    dp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))  # noqa: E731
    # The device-resident propagations still refuse a batch with event equations.
    st = lib.hy_batch_propagate_until(b._h, dp(tf), None, None, 0, 0)
    assert st == _capi.HY_ERR_NOT_IMPLEMENTED and "lock-step" in _capi.last_error()
    out = np.empty((2, 2, 8))
    grid = np.vstack([np.zeros(8), tf])
    assert lib.hy_batch_propagate_grid(b._h, dp(grid), 2, None, 0, dp(out)) == _capi.HY_ERR_NOT_IMPLEMENTED
    # The new ones check their arguments, with the messages of propagate_until(), before any step.
    n0 = b.launch_count()
    never = lambda evs, th, tl, cont: pytest.fail("called back")  # noqa: E731
    for bad, msg in ((dict(t_hi=np.full(8, np.nan)), "A non-finite time was passed"),
                     (dict(max_delta_t=np.full(8, -1.0)), "A non-positive max_delta_t"),
                     (dict(max_delta_t=np.full(8, np.nan)), "A nan max_delta_t")):
        with pytest.raises(ValueError, match=msg):
            b.propagate_until_ev(bad.get("t_hi", tf), None, bad.get("max_delta_t"), 0, never)
    with pytest.raises(ValueError, match="must match the current time"):
        b.propagate_grid_ev(np.vstack([np.full(8, 0.5), tf]), None, 0, never)
    assert b.launch_count() == n0
    st = lib.hy_batch_propagate_until_ev(b._h, dp(tf), None, None, 0, None, None, None)
    assert st == _capi.HY_ERR_INVALID_ARG and "Null pointer" in _capi.last_error()
    plain = hb.Batch(hb.Program([(x, v), (v, -9.8 * hb.sin(x))]), 8)
    with pytest.raises(ValueError, match="needs a batch with event equations"):
        plain.propagate_until_ev(tf, None, None, 0, never)
