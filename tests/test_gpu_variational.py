"""Variational integrators on the GPU: the augmented systems on every kernel shape (bit for bit against the HBM-tape
kernel, and against the oracle), the closed form and det(Phi) on the device, automatic kernel selection for the
variational 6-body system, and the device Taylor map (k_taylor_map) against a numpy restatement of its fixed
summation order, against propagations from perturbed states, and on a sharded batch."""
import numpy as np
import pytest

import heyoka_b200 as hb
import oracle
from common import outer_ss_batch_state, sys_outer_ss, sys_two_body, two_body_batch_state
from test_variational_cpu import osc_closed_form, osc_state, three_body_state

pytestmark = pytest.mark.gpu

SHAPES = [dict(tape="auto"), dict(tape="hbm"), dict(tape="smem"), dict(tape="global"), dict(tape="global-cta")]
LANES = 5


def case(name):
    """(variational system, original state [n, LANES], pars or None, final time)."""
    if name == "pendulum":
        vs = hb.var_ode_sys(hb.model.pendulum(), hb.var_args.vars)
        return vs, np.stack([np.linspace(0.2, 1.2, LANES), np.linspace(-0.3, 0.3, LANES)]), None, 4.0
    if name == "oscillator":
        x, v = hb.make_vars("x", "v")
        vs = hb.var_ode_sys([(x, v), (v, -hb.par[0] ** 2 * x)], [x, v, hb.par[0]])
        x0, v0, w = osc_state(LANES)
        return vs, np.stack([x0, v0]), w[None, :], 3.0
    if name == "two-body":
        return hb.var_ode_sys(sys_two_body(), hb.var_args.vars), two_body_batch_state(LANES), None, 2.0
    if name == "3-body":
        return hb.var_ode_sys(hb.model.nbody(3), hb.var_args.vars), three_body_state(LANES), None, 1.0
    raise KeyError(name)


CASES = ["pendulum", "oscillator", "two-body", "3-body"]


def make(vs, x0, pars, kernel):
    return hb.taylor_adaptive_batch(vs, x0, x0.shape[1], pars=pars, kernel=kernel)


def run(vs, x0, pars, tf, kernel):
    ta = make(vs, x0, pars, kernel)
    ta.step(write_tc=True)
    first = (ta.state.copy(), ta.tc.copy(), ta.last_h.copy())
    ta.propagate_until(tf)
    return first, ta.state.copy(), [r[3] for r in ta.propagate_res], ta._b.kernel_info()


@pytest.mark.parametrize("name", CASES)
def test_every_shape_bitwise_and_against_oracle(name):
    vs, x0, pars, tf = case(name)
    P = hb.Program(vs)
    full = hb._var_initial_state(vs, x0, LANES)
    ref = run(vs, x0, pars, tf, dict(tape="hbm"))
    o = oracle.OracleIntegrator(P, full, LANES, pars=pars, mode=oracle.FMA)
    o.step(write_tc=True)
    w = np.abs(o.last_h)[None, None, :] ** np.arange(P.order + 1)[None, :, None]
    scale = np.maximum(np.max(np.abs(o.tc[:, 0, :]), axis=0), 1.0)[None, None, :]
    assert np.max(np.abs(ref[0][1] - o.tc) * w / scale) < 1e-12
    assert np.max(np.abs(ref[0][2] / o.last_h - 1)) < 1e-10
    o.propagate_until(tf)
    assert ref[2] == [int(s) for s in o.n_steps], (ref[2], o.n_steps)
    assert np.max(np.abs(ref[1] - o.state) / np.maximum(np.abs(o.state), 1.0)) < 1e-11
    ran = []
    for kernel in SHAPES:
        try:
            got = run(vs, x0, pars, tf, kernel)
        except ValueError as e:
            # The shared-memory tape is refused when the plan does not fit an SM.
            assert kernel["tape"] == "smem", (kernel, e)
            continue
        ran.append(got[3]["tape"])
        for a, b in zip(got[0], ref[0]):
            assert np.array_equal(a, b), (name, kernel)
        assert np.array_equal(got[1], ref[1]) and got[2] == ref[2], (name, kernel)
    assert {"hbm", "global", "global-cta"} <= set(ran), ran
    if name in ("pendulum", "oscillator"):
        assert "smem" in ran


def test_oscillator_closed_form_on_device():
    vs, x0, pars, tf = case("oscillator")
    ta = make(vs, x0, pars, None)
    ta.propagate_until(tf)
    for lane in range(LANES):
        xs, phi = osc_closed_form(x0[0, lane], x0[1, lane], pars[0, lane], tf)
        assert np.allclose(ta.state[:2, lane], xs, rtol=1e-12, atol=1e-12)
        assert np.allclose(ta.state[ta.get_vslice(1), lane].reshape(2, 3), phi, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("name", ["pendulum", "two-body", "3-body"])
def test_det_phi_on_device(name):
    vs, x0, pars, tf = case(name)
    n = vs.n_orig_sv
    ta = make(vs, x0, pars, None)
    ta.propagate_until(tf)
    for lane in range(LANES):
        assert abs(np.linalg.det(ta.state[n:, lane].reshape(n, n)) - 1.0) < 1e-9


def test_variational_six_body_selection_and_oracle():
    vs = hb.var_ode_sys(sys_outer_ss(), hb.var_args.vars)
    assert len(vs.sys) == 1332
    x0 = outer_ss_batch_state(4)
    ta = make(vs, x0, None, None)
    ki = ta._b.kernel_info()
    # Not N-body-shaped any more: the cooperative kernel (shared-memory tape if the plan fits, else global tape).
    assert ki["tape"] in ("smem", "global", "global-cta"), ki
    with pytest.raises(ValueError, match="The N-body kernel cannot run this program"):
        make(vs, x0, None, dict(tape="nbody"))
    P = hb.Program(vs)
    o = oracle.OracleIntegrator(P, hb._var_initial_state(vs, x0, 4), 4, mode=oracle.FMA)
    for _ in range(3):
        ta.step()
        o.step()
    assert np.max(np.abs(ta.last_h / o.last_h - 1)) < 1e-10
    assert np.max(np.abs(ta.state - o.state) / np.maximum(np.abs(o.state), 1.0)) < 1e-11


# ---- the Taylor map -----------------------------------------------------------------------------------------------
def taylor_map_np(state, n, m, dx):
    """k_taylor_map's arithmetic: acc = x_i, then acc = acc + Phi_ij * dx_j for j = 0 .. m - 1, each rounded."""
    acc = state[:n].copy()
    phi = state[n:].reshape(n, m, -1)
    for j in range(m):
        acc = acc + phi[:, j, :] * dx[j][None, :]
    return acc


def random_phi_batch(vs, batch, seed):
    """A Batch of the variational program holding a random state (the map does not care where the state came from)."""
    rng = np.random.default_rng(seed)
    P = hb.Program(vs)
    b = hb.Batch(P, batch)
    st = rng.uniform(-2, 2, (P.n_eq, batch))
    b.upload(st, None, np.zeros(batch), np.zeros(batch))
    return b, st, rng


@pytest.mark.parametrize("batch", [1, 31, 33, 2 ** 16 + 3])
def test_taylor_map_bitwise_host_and_device(batch):
    import torch
    vs = hb.var_ode_sys(hb.model.nbody(2), hb.var_args.vars)  # 12 x 12 STM
    n, m = vs.n_orig_sv, len(vs.vargs)
    b, st, rng = random_phi_batch(vs, batch, batch)
    dx = rng.uniform(-1e-3, 1e-3, (m, batch))
    want = taylor_map_np(st, n, m, dx)
    got = b.eval_taylor_map(n, dx)
    assert np.array_equal(got, want)
    d_dx = torch.from_numpy(dx).cuda()
    d_out = torch.empty((n, batch), dtype=torch.float64, device="cuda")
    b.eval_taylor_map_dev(n, m, d_dx.data_ptr(), d_out.data_ptr())
    b.sync()
    assert np.array_equal(d_out.cpu().numpy(), want)


def test_taylor_map_more_arguments_than_one_chunk():
    """45 arguments: the kernel works through two chunks of dx with the partial sums in `out`."""
    x = hb.make_vars(*["x%d" % i for i in range(3)])
    sys_ = [(x[0], x[1]), (x[1], x[2]), (x[2], -x[0] * sum(hb.par[k] for k in range(42)))]
    vs = hb.var_ode_sys(sys_, hb.var_args.vars | hb.var_args.params)
    assert len(vs.vargs) == 45
    b, st, rng = random_phi_batch(vs, 97, 3)
    dx = rng.uniform(-1, 1, (45, 97))
    assert np.array_equal(b.eval_taylor_map(3, dx), taylor_map_np(st, 3, 45, dx))


def test_taylor_map_size_checks():
    vs, x0, pars, tf = case("oscillator")
    ta = make(vs, x0, pars, None)
    with pytest.raises(ValueError):
        ta.eval_taylor_map(np.zeros((2, LANES)))
    with pytest.raises(ValueError):
        ta._b.eval_taylor_map(3, np.zeros((2, LANES)))
    plain = hb.taylor_adaptive_batch(hb.model.pendulum(), np.zeros((2, 2)), 2)
    assert not plain.is_variational and plain.n_orig_sv == 2 and plain.vorder == 0
    with pytest.raises(ValueError):
        plain.eval_taylor_map(np.zeros((2, 2)))


def test_taylor_map_against_perturbed_propagations():
    """x(tf; x0 + dx) - TaylorMap(dx) = O(|dx|^2): the residual falls by ~4 when dx is halved."""
    vs, x0, pars, tf = case("pendulum")
    ta = make(vs, x0, pars, None)
    ta.propagate_until(tf)
    assert ta.is_variational and ta.vorder == 1 and ta.n_orig_sv == 2
    res = []
    for eps in (1e-3, 5e-4):
        dx = eps * np.stack([np.ones(LANES), -np.ones(LANES)])
        tm = ta.eval_taylor_map(dx).copy()
        assert tm is not None and np.array_equal(ta.tstate, tm)
        pt = hb.taylor_adaptive_batch(hb.model.pendulum(), x0 + dx, LANES)
        pt.propagate_until(tf)
        res.append(np.max(np.abs(pt.state - tm)))
    assert res[0] < 1e-4 and 3.0 < res[0] / res[1] < 5.0, res


def test_taylor_map_sharded_equals_single_device():
    vs, x0, pars, tf = case("3-body")
    x0 = three_body_state(37)
    single = make(vs, x0, None, None)
    shard = hb.taylor_adaptive_batch(vs, x0, 37, device=[0, 0])
    assert shard._b.n_shards == 2
    single.propagate_until(tf)
    shard.propagate_until(tf)
    assert np.array_equal(single.state, shard.state)
    dx = np.random.default_rng(9).uniform(-1e-4, 1e-4, (18, 37))
    assert np.array_equal(single.eval_taylor_map(dx), shard.eval_taylor_map(dx))


def test_variational_members():
    vs, x0, pars, tf = case("oscillator")
    ta = make(vs, x0, pars, None)
    assert [repr(a) for a in ta.vargs] == ["x", "v", "p0"]
    assert ta.get_vslice(0) == slice(0, 2) and ta.get_vslice(1) == slice(2, 8)
    assert ta.get_vslice(1, component=1) == slice(5, 8) and ta.get_vslice(0, component=1) == slice(1, 2)
    assert ta.get_mindex(1) == [1, 0, 0, 0] and ta.get_mindex(6) == [1, 0, 1, 0]
    with pytest.raises(ValueError):
        ta.get_vslice(2)
    # The constructor filled the STM (identity block for x, v; zero column for the parameter).
    phi = ta.state[2:].reshape(2, 3, LANES)
    assert np.array_equal(phi[:, :, 0], [[1, 0, 0], [0, 1, 0]])
    # Later writes to the state are taken as given, the variational rows included.
    ta.state[:2] = 0.5
    ta.state[2:] = np.arange(6 * LANES).reshape(6, LANES) / 7.0
    dx = np.ones((3, LANES))
    assert np.array_equal(ta.eval_taylor_map(dx), taylor_map_np(ta.state, 2, 3, dx))


def test_propagate_grid_and_continuous_output_against_oracle():
    vs, x0, pars, tf = case("pendulum")
    P = hb.Program(vs)
    full = hb._var_initial_state(vs, x0, LANES)
    grid = np.repeat(np.linspace(0.0, tf, 9)[:, None], LANES, axis=1)
    ta = make(vs, x0, pars, None)
    out = ta.propagate_grid(grid)
    o = oracle.OracleIntegrator(P, full, LANES, mode=oracle.FMA)
    want = o.propagate_grid(grid)
    assert np.max(np.abs(out - want) / np.maximum(np.abs(want), 1.0)) < 1e-11
    ta2 = make(vs, x0, pars, None)
    co = ta2.propagate_until(tf, c_output=True)
    o2 = oracle.OracleIntegrator(P, full, LANES, mode=oracle.FMA)
    oc = o2.propagate_until_cout(tf)
    for t in (0.3, 1.7, 3.9):
        assert np.max(np.abs(co(t) - oc(t)) / np.maximum(np.abs(oc(t)), 1.0)) < 1e-11
