"""GPU parity tests: the CUDA path (through the C ABI) against the CPU oracle on the same seeded inputs.

Tolerances. All arithmetic of the jet is + - * / sqrt and explicit fma in the same order on both sides
(oracle mode FMA), so the Taylor coefficients of N-body systems agree to the last bit or two; the
differences come from the math library (pow in the step-size estimate, sin/cos/tanh/exp/log at order 0:
CUDA libdevice vs glibc, both <= 2 ulp). Stated bounds: one step 1e-13 relative (100-1000 eps, like
test/taylor_adaptive_batch.cpp:143), long propagations 1e-12 relative on the final state with IDENTICAL
step counts (BASELINE.json north_star).
"""
import numpy as np
import pytest

import heyoka_b200 as hb
import oracle
from common import (OUTER_SS_G, OUTER_SS_MASSES, approx, decimals_equal, golden, nbody_rel_err, outer_ss_batch_state, outer_ss_ic,
                    sig_digits_equal, sys_outer_ss, sys_pendulum, sys_tutorial, sys_two_body, two_body_batch_state)

pytestmark = pytest.mark.gpu

OC = {"success": hb.taylor_outcome.success, "time_limit": hb.taylor_outcome.time_limit}

# Every parity test runs on both tape strategies and a few cooperative-kernel shapes (see kernels.cuh).
KERNELS = {
    "hbm": dict(tape="hbm"),
    "global": dict(tape="global"),  # the cooperative kernel with the tape in global memory
    "global-cta": dict(tape="global-cta"),  # idem, a whole CTA per chunk of lanes
    "smem-auto": dict(tape="smem"),
    "smem-notmem": dict(tape="smem-notmem"),  # (the same kernel as "smem": the API keeps the name)
    "smem-L8N2": dict(tape="smem", lanes_per_warp=8, lanes_per_thread=2),
    "smem-L2N1": dict(tape="smem", lanes_per_warp=2, lanes_per_thread=1, block_threads=64),
    "smem-L2N2": dict(tape="smem", lanes_per_warp=2, lanes_per_thread=2),
    "smem-L4N4": dict(tape="smem", lanes_per_warp=4, lanes_per_thread=4, block_threads=32),
    # The dedicated N-body kernel (nb_kernel.cuh; N-body-shaped programs only, on the others the tests check that it is
    # refused, see _refused()): default / with lanes_per_thread given (ignored) / 12 warps per CTA (168 registers per
    # thread) / one lane per team.
    "nbody": dict(tape="nbody"),
    "nbody-smem": dict(tape="nbody", lanes_per_thread=2),
    "nbody-384": dict(tape="nbody", lanes_per_thread=1, block_threads=384),
    "nbody-L1": dict(tape="nbody", lanes_per_warp=1, block_threads=128),
    # One thread per lane (nb1_kernel.cuh; programs with ONE pair interaction only): default / lanes_per_thread given.
    "nbody-lane": dict(tape="nbody-lane"),
    "nbody-lane-smem": dict(tape="nbody-lane", lanes_per_thread=2),
}


@pytest.fixture(params=list(KERNELS), scope="module")
def kernel(request):
    return KERNELS[request.param]


def _refused(kernel, sys, **program_kw):
    """The dedicated N-body kernels run N-body-shaped programs only (nb_plan.hpp; the one-thread-per-lane form: one pair
    interaction). Forcing one of them on another program must fail with the documented error, never fall back to another
    kernel: for those (kernel, program) combinations that refusal is what the test checks, and it returns True. False:
    the kernel runs the program (and the test goes on with it)."""
    if not kernel["tape"].startswith("nbody"):
        return False
    b = hb.Batch(hb.Program(sys, **program_kw), 1)
    try:
        b.set_kernel(**kernel)
    except ValueError as e:
        assert "The N-body kernel cannot run this program" in str(e), str(e)
        return True
    assert b.kernel_info()["tape"] == kernel["tape"]
    return False


def rel_err(a, b, floor=1e-6):
    """Component-wise relative error (with an absolute floor)."""
    a, b = np.asarray(a), np.asarray(b)
    return np.max(np.abs(a - b) / np.maximum(np.abs(b), floor))


def lane_err(a, b):
    """Lane-wise norm error of a state array [n_eq, batch]: max |a - b| over the variables of a lane, relative to
    the largest |b| of that lane (components that pass through zero have no meaningful relative error)."""
    a, b = np.asarray(a), np.asarray(b)
    return float(np.max(np.max(np.abs(a - b), axis=0) / np.maximum(np.max(np.abs(b), axis=0), 1e-3)))


def tc_err(tc_a, tc_b, h):
    """Error of the Taylor coefficients weighted by their contribution to the state: |d tc[o]| |h|^o relative
    to the state's magnitude. (High-order coefficients are tiny and the result of cancelling sums: their
    component-wise relative accuracy is ~1e-9 in the reference too, while their weight in the step is < 1 ulp.)"""
    order = tc_a.shape[1] - 1
    w = np.abs(h)[None, None, :] ** np.arange(order + 1)[None, :, None]
    scale = np.maximum(np.max(np.abs(tc_b[:, 0, :]), axis=0), 1e-3)[None, None, :]
    return np.max(np.abs(tc_a - tc_b) * w / scale)


def test_tutorial_batch_mode_gpu(kernel):
    """doc/tut_batch_mode.rst end to end on the GPU (same fixture that pins the oracle)."""
    if _refused(kernel, sys_tutorial()):
        return
    g = golden("tut_batch_mode.json")
    ta = hb.taylor_adaptive_batch(sys_tutorial(), [g["x0"], g["v0"]], 4, pars=[g["alpha"]], kernel=kernel)
    assert ta.get_order() == 20

    ta.step()
    assert [r[0] for r in ta.step_res] == [OC[r["outcome"]] for r in g["first_step"]]
    assert sig_digits_equal([r[1] for r in ta.step_res], [r["h"] for r in g["first_step"]])
    assert decimals_equal(ta.state, g["states"][0])
    assert decimals_equal(ta.time, g["times"][0])

    ta.step(g["clamped_step_limits"])
    assert [r[0] for r in ta.step_res] == [OC[r["outcome"]] for r in g["clamped_step"]]
    assert [r[1] for r in ta.step_res] == g["clamped_step_limits"]
    assert decimals_equal(ta.state, g["states"][1])

    ta.propagate_for(g["propagate_for"]["delta_ts"])
    res = g["propagate_for"]["res"]
    assert [r[0] for r in ta.propagate_res] == [OC[r["outcome"]] for r in res]
    assert [r[3] for r in ta.propagate_res] == [r["n_steps"] for r in res]
    assert sig_digits_equal([r[1] for r in ta.propagate_res], [r["min_h"] for r in res])
    assert sig_digits_equal([r[2] for r in ta.propagate_res], [r["max_h"] for r in res])
    assert decimals_equal(ta.state, g["states"][2])
    assert decimals_equal(ta.time, g["times"][2])

    ta.propagate_until(g["propagate_until"]["ts"])
    res = g["propagate_until"]["res"]
    assert [r[3] for r in ta.propagate_res] == [r["n_steps"] for r in res]
    assert decimals_equal(ta.state, g["states"][3])
    assert np.all(ta.time == np.array(g["propagate_until"]["ts"]))

    ta.step(write_tc=True)
    assert sig_digits_equal(ta.tc, g["tc_after_final_step"], 7)


def _step_parity(kernel, sys, state, batch, pars=None, time=0.0, ha=False, n_steps=3, tol=1e-13, max_delta_t=None):
    if _refused(kernel, sys, high_accuracy=ha):
        return
    P = hb.Program(sys, high_accuracy=ha)
    o = oracle.OracleIntegrator(P, state, batch, pars=pars, time=time, mode=oracle.FMA)
    ta = hb.taylor_adaptive_batch(sys, state, batch, pars=pars, time=time, high_accuracy=ha, kernel=kernel)
    for _ in range(n_steps):
        o.step(max_delta_t, write_tc=True)
        ta.step(max_delta_t, write_tc=True)
        assert rel_err(ta.last_h, o.last_h) < tol
        assert lane_err(ta.state, o.state) < tol
        assert tc_err(ta.tc, o.tc, o.last_h) < tol
        assert np.array_equal([r[0] for r in ta.step_res], o.step_outcome)
        assert rel_err(ta.time, o.t_hi) < tol
        # keep the two sides on the same trajectory: identical inputs for the next step
        ta._state[:] = o.state
        ta._t_hi[:] = o.t_hi
        ta._t_lo[:] = o.t_lo


@pytest.mark.parametrize("ha", [False, True])
@pytest.mark.parametrize("batch", [1, 4, 33, 70])
def test_step_parity_pendulum(kernel, ha, batch):
    rng = np.random.default_rng(1)
    st = np.stack([rng.uniform(-1, 1, batch), rng.uniform(-1, 1, batch)])
    _step_parity(kernel, sys_pendulum(), st, batch, ha=ha)


@pytest.mark.parametrize("ha", [False, True])
def test_step_parity_tutorial_system(kernel, ha):
    rng = np.random.default_rng(2)
    batch = 37
    st = np.stack([rng.uniform(-1, 1, batch), rng.uniform(1, 2, batch)])
    pars = rng.uniform(0.05, 0.2, (1, batch))
    tm = rng.uniform(0, 10, batch)
    _step_parity(kernel, sys_tutorial(), st, batch, pars=pars, time=tm, ha=ha)


@pytest.mark.parametrize("ha", [False, True])
def test_step_parity_two_body(kernel, ha):
    _step_parity(kernel, sys_two_body(), two_body_batch_state(50), 50, ha=ha)


@pytest.mark.parametrize("ha", [False, True])
@pytest.mark.parametrize("masses", [[1., 0.3], [0.7, 1.1], [0., 2.]])
def test_step_parity_two_massive_bodies(kernel, ha, masses):
    """Two bodies that both pull (pair outputs m_k and the rescaled n_k), and the massless body first."""
    rng = np.random.default_rng(3)
    batch = 77
    st = two_body_batch_state(batch) + 0.05 * rng.standard_normal((12, batch))
    _step_parity(kernel, hb.model.nbody(2, masses=masses), st, batch, ha=ha)


@pytest.mark.parametrize("ha", [False, True])
@pytest.mark.parametrize("batch", [3, 45])
def test_step_parity_outer_ss(kernel, ha, batch):
    _step_parity(kernel, sys_outer_ss(), outer_ss_batch_state(batch), batch, ha=ha, n_steps=2)


def test_step_backward_and_limits(kernel):
    if _refused(kernel, sys_outer_ss()):
        return
    st = outer_ss_batch_state(8)
    P = hb.Program(sys_outer_ss())
    o = oracle.OracleIntegrator(P, st, 8, mode=oracle.FMA)
    ta = hb.taylor_adaptive_batch(sys_outer_ss(), st, 8, kernel=kernel)
    o.step(backward=True)
    ta.step_backward()
    assert np.all(ta.last_h < 0)
    assert rel_err(ta.last_h, o.last_h) < 1e-13 and rel_err(ta.state, o.state) < 1e-13
    lim = np.array([1e-3, -1e-3, 0.0, 1e3, -1e3, 2e-3, 5e-4, -5e-4])
    o.step(lim)
    ta.step(lim)
    assert np.array_equal([r[0] for r in ta.step_res], o.step_outcome)
    assert rel_err(ta.state, o.state) < 1e-13
    assert np.all(ta.last_h[[0, 1, 2, 5, 6, 7]] == lim[[0, 1, 2, 5, 6, 7]])


@pytest.mark.parametrize("ha", [False, True])
def test_propagate_parity_outer_ss(kernel, ha):
    """100 years of the perturbed outer Solar System: identical step counts, final state to 1e-12."""
    if _refused(kernel, sys_outer_ss(), high_accuracy=ha):
        return
    batch = 40
    st = outer_ss_batch_state(batch)
    P = hb.Program(sys_outer_ss(), high_accuracy=ha)
    o = oracle.OracleIntegrator(P, st, batch, mode=oracle.FMA)
    ta = hb.taylor_adaptive_batch(sys_outer_ss(), st, batch, high_accuracy=ha, kernel=kernel)
    o.propagate_until(100.)
    ta.propagate_until(100.)
    assert np.all(ta.time == 100.)
    assert np.array_equal([r[3] for r in ta.propagate_res], o.n_steps)
    assert np.all(np.array([r[0] for r in ta.propagate_res]) == hb.taylor_outcome.time_limit)
    assert nbody_rel_err(ta.state, o.state) < 1e-12
    assert rel_err([r[1] for r in ta.propagate_res], o.min_h) < 1e-12
    assert rel_err([r[2] for r in ta.propagate_res], o.max_h) < 1e-12
    # backwards to where we started: test/back_and_forth.cpp style round trip.
    ta.propagate_until(0.)
    assert np.all(ta.time == 0.)
    assert nbody_rel_err(ta.state, st) < 1e-11


@pytest.mark.parametrize("mode", ["pairwise", "seq"])
def test_propagate_parity_reference_default_mode(mode):
    """The reference's DEFAULT (non-compact) mode sums pairwise, its compact mode sequentially without contraction; the
    kernels sum sequentially with fused multiply-adds (the third oracle mode, which every other test compares against).
    Here the GPU meets the other two restatements directly: 64 lanes of the perturbed outer Solar System over 100 years
    and the two-body problem over 40 time units - identical step counts, final states to 1e-11 (a few hundred steps of
    reordered sums: the reference's own compact-vs-default tests use 100-1000 eps per step)."""
    m = oracle.PAIRWISE if mode == "pairwise" else oracle.SEQ
    for sys_, st, tf, ha in ((sys_outer_ss(), outer_ss_batch_state(64, seed=9), 100., True),
                             (sys_two_body(), two_body_batch_state(64, seed=3), 40., False)):
        P = hb.Program(sys_, high_accuracy=ha)
        o = oracle.OracleIntegrator(P, st, 64, mode=m)
        ta = hb.taylor_adaptive_batch(sys_, st, 64, high_accuracy=ha)
        o.propagate_until(tf, lockstep=False)
        ta.propagate_until(tf)
        assert [r[3] for r in ta.propagate_res] == [int(x) for x in o.n_steps]
        assert lane_err(ta.state, o.state) < 1e-11


def test_propagate_exact_step_counts_gpu(kernel):
    """test/taylor_adaptive_batch.cpp:586-598 on the GPU."""
    if _refused(kernel, sys_pendulum()):
        return
    ta = hb.taylor_adaptive_batch(sys_pendulum(), [[0.05, 0.06], [0.025, 0.026]], 2, kernel=kernel)
    ta2 = hb.taylor_adaptive_batch(sys_pendulum(), [[0.05, 0.06], [0.025, 0.026]], 2, kernel=kernel)
    ta.propagate_until([10., 11.], max_delta_t=[1e-4, 5e-5])
    ta2.propagate_until([10., 11.])
    assert np.all(ta.time == [10., 11.])
    assert [r[3] for r in ta.propagate_res] == [100000, 220000]
    assert all(r[0] == hb.taylor_outcome.time_limit for r in ta.propagate_res)
    assert approx(ta.state, ta2.state, 1000.)
    # backwards with propagate_for (:640-652)
    ta.propagate_for([-10., -11.], max_delta_t=[1e-4, 5e-5])
    assert np.all(ta.time == [0., 0.])
    assert [r[3] for r in ta.propagate_res] == [100000, 220000]


def test_propagate_per_lane_times_and_dfloat(kernel):
    if _refused(kernel, sys_pendulum()):
        return
    batch = 35
    rng = np.random.default_rng(5)
    st = np.stack([rng.uniform(-1, 1, batch), rng.uniform(-1, 1, batch)])
    t0 = rng.uniform(-5, 5, batch)
    tf = t0 + rng.uniform(-20, 20, batch)
    tf[3] = t0[3]  # zero-length propagation
    P = hb.Program(sys_pendulum())
    o = oracle.OracleIntegrator(P, st, batch, time=t0, mode=oracle.FMA)
    ta = hb.taylor_adaptive_batch(sys_pendulum(), st, batch, time=t0, kernel=kernel)
    o.propagate_until(tf)
    ta.propagate_until(tf)
    assert np.array_equal(ta.time, tf) and np.array_equal(o.t_hi, tf)
    assert np.array_equal([r[3] for r in ta.propagate_res], o.n_steps)
    assert ta.propagate_res[3][3] == 0
    assert rel_err(ta.state, o.state) < 1e-12


def test_global_exits_match_reference_semantics(kernel):
    """max_steps counts iterations and turns EVERY outcome into step_limit; a non-finite lane stops EVERY
    lane at that iteration (src/taylor_adaptive_batch.cpp:1462-1467, :1516-1526). Checked against the
    oracle's lock-step loop."""
    if _refused(kernel, sys_outer_ss()):
        return
    batch = 6
    st = outer_ss_batch_state(batch)
    P = hb.Program(sys_outer_ss())

    # iteration limit
    o = oracle.OracleIntegrator(P, st, batch, mode=oracle.FMA)
    ta = hb.taylor_adaptive_batch(sys_outer_ss(), st, batch, kernel=kernel)
    tf = np.array([0.5, 100., 100., 2.0, 100., 100.])
    o.propagate_until(tf, max_steps=7)
    ta.propagate_until(tf, max_steps=7)
    assert np.all(o.prop_outcome == hb.taylor_outcome.step_limit)
    assert [r[0] for r in ta.propagate_res] == [hb.taylor_outcome.step_limit] * batch
    assert np.array_equal([r[3] for r in ta.propagate_res], o.n_steps)
    assert rel_err(ta.time, o.t_hi) < 1e-13 and rel_err(ta.state, o.state) < 1e-12

    # non-finite state: put two bodies of lane 2 on top of each other after a few steps' worth of time by
    # making lane 2 start from a collision configuration (distance 0 -> r^-3 = inf -> NaN).
    st2 = st.copy()
    st2[6:9, 2] = st2[0:3, 2]
    o = oracle.OracleIntegrator(P, st2, batch, mode=oracle.FMA)
    ta = hb.taylor_adaptive_batch(sys_outer_ss(), st2, batch, kernel=kernel)
    o.propagate_until(100.)
    ta.propagate_until(100.)
    assert int(o.prop_outcome[2]) == hb.taylor_outcome.err_nf_state
    assert np.array_equal([r[0] for r in ta.propagate_res], o.prop_outcome)
    assert np.array_equal([r[3] for r in ta.propagate_res], o.n_steps)
    ok = [0, 1, 3, 4, 5]
    assert rel_err(ta.state[:, ok], o.state[:, ok]) < 1e-12
    assert rel_err(ta.time[ok], o.t_hi[ok]) < 1e-13


def test_dense_output(kernel):
    if _refused(kernel, sys_outer_ss(), high_accuracy=True):
        return
    batch = 9
    st = outer_ss_batch_state(batch)
    P = hb.Program(sys_outer_ss(), high_accuracy=True)
    o = oracle.OracleIntegrator(P, st, batch, mode=oracle.FMA)
    ta = hb.taylor_adaptive_batch(sys_outer_ss(), st, batch, high_accuracy=True, kernel=kernel)
    o.step(write_tc=True)
    ta.step(write_tc=True)
    tau = 0.37 * o.last_h
    ref = o.d_output(tau)
    # rel_time is relative to the CURRENT time (src/taylor_adaptive_batch.cpp:2276-2280): the polynomial, expanded about
    # the start of the last step, is evaluated at last_h + t.
    got = ta.update_d_output(tau - ta.last_h, rel_time=True)
    assert rel_err(got, ref) < 1e-13
    got_abs = ta.update_d_output(ta.time - ta.last_h + tau)
    assert rel_err(got_abs, ref) < 1e-12
    # rel_time = 0 reproduces the current state, rel_time = -last_h the state before the step
    assert rel_err(ta.update_d_output(0., rel_time=True), ta.state) < 1e-13
    assert rel_err(ta.update_d_output(-ta.last_h, rel_time=True), st) < 1e-15


def test_propagate_early_lanes_last_h_and_tc(kernel):
    """Lanes that reach their final time before the slowest lane take zero-length steps in the reference's lock-step
    loop (src/taylor_adaptive_batch.cpp:1372-1397): on return last_h = 0 and, with write_tc, the Taylor coefficients
    are re-expanded about the final state. The device-resident loop reproduces both (one masked zero-length step);
    compared against the oracle's lock-step loop, then through update_d_output()."""
    if _refused(kernel, sys_outer_ss(), high_accuracy=True):
        return
    batch = 10
    st = outer_ss_batch_state(batch)
    tf = np.linspace(2.0, 11.0, batch)  # different numbers of steps per lane
    P = hb.Program(sys_outer_ss(), high_accuracy=True)
    for wtc in (True, False):
        o = oracle.OracleIntegrator(P, st, batch, mode=oracle.FMA)
        ta = hb.taylor_adaptive_batch(sys_outer_ss(), st, batch, high_accuracy=True, kernel=kernel)
        o.propagate_until(tf, write_tc=wtc)
        ta.propagate_until(tf, write_tc=wtc)
        assert [r[3] for r in ta.propagate_res] == [int(x) for x in o.n_steps]
        assert np.count_nonzero(o.last_h == 0.) >= batch - 3          # most lanes finished early
        assert np.array_equal(ta.last_h == 0., o.last_h == 0.)
        assert rel_err(ta.last_h, o.last_h, floor=1e-3) < 1e-11
        assert lane_err(ta.state, o.state) < 1e-12
        if wtc:
            assert tc_err(ta.tc, o.tc, np.maximum(np.abs(o.last_h), 0.3)) < 1e-11
            # Dense output at the current time reproduces the state for every lane (early ones included).
            assert rel_err(ta.update_d_output(0., rel_time=True), ta.state) < 1e-13
            assert rel_err(ta.update_d_output(tf), ta.state) < 1e-13


@pytest.mark.parametrize("masses", [[1., 0.], [1., 0.4]])
def test_two_body_lane_kernel(masses):
    """The one-thread-per-lane N-body kernel (k_nb1, nb1_kernel.cuh): selected automatically for systems with one pair
    interaction; bit-identical to k_nb with 32 lanes per warp (same arithmetic, same order) for steps with and without
    the public Taylor coefficients, propagate_until() with lanes that finish early, and a masked re-expansion; against
    the oracle: identical step counts over 40 time units, states to 2e-11."""
    sys_ = hb.model.nbody(2, masses=masses)
    batch = 1000  # (not a multiple of 32; several warps and CTAs)
    rng = np.random.default_rng(11)
    st = two_body_batch_state(batch) + 0.02 * rng.standard_normal((12, batch))
    lane = hb.taylor_adaptive_batch(sys_, st, batch)
    assert lane._b.kernel_info()["tape"] == "nbody-lane" and lane._b.kernel_info()["lanes_per_warp"] == 32
    team = hb.taylor_adaptive_batch(sys_, st, batch, kernel=dict(tape="nbody"))
    assert team._b.kernel_info()["tape"] == "nbody" and team._b.kernel_info()["lanes_per_warp"] == 32
    for wtc in (False, True, False):
        lane.step(write_tc=wtc)
        team.step(write_tc=wtc)
        assert np.array_equal(lane.state, team.state) and np.array_equal(lane.last_h, team.last_h)
        assert np.array_equal(lane.time, team.time)
        assert [r[0] for r in lane.step_res] == [r[0] for r in team.step_res]
        if wtc:
            assert np.array_equal(lane.tc, team.tc)
    lim = np.where(np.arange(batch) % 3 == 0, 1e-3, -2e-3)
    lane.step(lim)
    team.step(lim)
    assert np.array_equal(lane.state, team.state) and np.array_equal(lane.last_h, lim)
    tf = lane.time + np.linspace(5., 40., batch)
    for wtc in (False, True):
        lane.propagate_until(tf if not wtc else tf + 3., write_tc=wtc)
        team.propagate_until(tf if not wtc else tf + 3., write_tc=wtc)
        assert lane.propagate_res == team.propagate_res
        assert np.array_equal(lane.state, team.state) and np.array_equal(lane.last_h, team.last_h)
        assert np.array_equal(lane.time, team.time)
        if wtc:
            assert np.array_equal(lane.tc, team.tc)
    # Against the oracle, from the initial conditions.
    P = hb.Program(sys_)
    idx = rng.choice(batch, 96, replace=False)
    o = oracle.OracleIntegrator(P, st[:, idx], len(idx), mode=oracle.FMA)
    ta = hb.taylor_adaptive_batch(sys_, st, batch)
    o.propagate_until(40., lockstep=False)
    ta.propagate_until(40.)
    assert [ta.propagate_res[i][3] for i in idx] == [int(x) for x in o.n_steps]
    assert lane_err(ta.state[:, idx], o.state) < 2e-11  # (~150 steps of ulp-level differences in pow)
    # A non-finite lane stops alone and is reported (global exit handled by the host replay).
    bad = st.copy()
    bad[0:3, 5] = bad[6:9, 5] = 0.  # one body on top of the other: r = 0
    ta = hb.taylor_adaptive_batch(sys_, bad, batch)
    ta.step()
    assert ta.step_res[5][0] == hb.taylor_outcome.err_nf_state
    assert all(r[0] == hb.taylor_outcome.success for i, r in enumerate(ta.step_res) if i != 5)


def test_raw_program_interface_matches():
    """hy_program_create() from raw arrays gives the same results as the symbolic path."""
    P = hb.Program(sys_two_body())
    d = P.desc
    import ctypes as C
    n_ops = P.n_uvars - P.n_eq
    args = np.ctypeslib.as_array(C.cast(d.args, C.POINTER(C.c_uint32)), shape=(max(d.n_args, 1),))[:d.n_args]
    consts = np.ctypeslib.as_array(C.cast(d.consts, C.POINTER(C.c_double)), shape=(max(d.n_consts, 1),))[:d.n_consts]
    sv = np.ctypeslib.as_array(C.cast(d.sv_defs, C.POINTER(C.c_uint32)), shape=(P.n_eq,))
    P2 = hb.Program.from_arrays(P.n_eq, P.n_uvars, P.n_pars, P.order, P.ops_array(), args, consts, sv)
    st = two_body_batch_state(10)
    res = []
    for prog in (P, P2):
        b = hb.Batch(prog, 10)
        b.upload(st, None, np.zeros(10), np.zeros(10))
        b.step()
        res.append(b.download()[0])
    assert np.array_equal(res[0], res[1])
    assert n_ops == 21 - 12


def test_kernel_selection_info():
    """Automatic selection: the dedicated N-body kernel for N-body-shaped programs (warp teams for the 6-body system,
    CTA teams for 32 bodies), the shared-memory tape otherwise; every strategy can be forced."""
    b = hb.Batch(hb.Program(sys_outer_ss(), high_accuracy=True), 64)
    ki = b.kernel_info()
    # 15 pair interactions x 2 lanes, one per thread, every private row in shared memory: 7 warps of 2 lanes fit in the
    # 227 KB of an H100 SM.
    assert ki["tape"] == "nbody" and ki["lanes_per_warp"] == 2 and ki["tmem_cols_per_warp"] == 0
    assert ki["block_threads"] == 224 and ki["smem_bytes"] <= 227 * 1024
    b.set_kernel("nbody", lanes_per_thread=2)
    ki = b.kernel_info()
    assert ki["tape"] == "nbody" and ki["tmem_cols_per_warp"] == 0
    b.set_kernel("smem")
    ki = b.kernel_info()
    assert ki["tape"] == "smem" and ki["tape_slots_per_lane"] < 234 * 21 / 2
    assert ki["smem_bytes"] <= 227 * 1024
    # The generic cooperative kernel: 8 warps of 2 lanes, two per thread, in shared memory.
    assert ki["tmem_cols_per_warp"] == 0 and ki["block_threads"] == 256 and ki["lanes_per_thread"] == 2
    b.set_kernel("smem", lanes_per_warp=2, lanes_per_thread=2)
    ki = b.kernel_info()
    assert ki["tmem_cols_per_warp"] == 0 and ki["block_threads"] == 256
    b.set_kernel("smem-notmem")
    ki = b.kernel_info()
    assert ki["tmem_cols_per_warp"] == 0 and ki["block_threads"] == 256
    b.set_kernel("hbm")
    assert b.kernel_info()["tape"] == "hbm"
    from common import sys_nbody32
    big = hb.Batch(hb.Program(sys_nbody32()), 32)
    assert big.kernel_info()["tape"] == "nbody-cta"  # 496 pair interactions: one lane per CTA of 512 threads
    big.set_kernel("global-cta")
    assert big.kernel_info()["tape"] == "global-cta"
    big.set_kernel("hbm")
    assert big.kernel_info()["tape"] == "hbm"
    with pytest.raises(ValueError, match="does not fit in shared memory"):
        big.set_kernel("smem")
    pend = hb.Batch(hb.Program(sys_pendulum()), 8)
    assert pend.kernel_info()["tape"] == "smem"
    with pytest.raises(ValueError, match="The N-body kernel cannot run this program"):
        pend.set_kernel("nbody")


def _closed_form_cases():
    from closed_form_cases import CASES
    from common import golden
    g = golden("closed_form_jets.json")
    return list(zip(CASES, g["cases"]))


@pytest.mark.gpu
@pytest.mark.parametrize("case,gold", _closed_form_cases(), ids=lambda v: v[0] if isinstance(v, tuple) else "")
def test_closed_form_jets_gpu(case, gold, kernel):
    """The reference's closed-form jet blocks (test/taylor_*.cpp, see tests/closed_form_cases.py) on the GPU:
    one step with write_tc, jets against the symbolic closed forms to the reference's tolerance."""
    from closed_form_cases import EPS_MUL, ORDER, TOL, batch_of, hb_system
    from test_oracle_golden import approximately
    if _refused(kernel, hb_system(hb, case), tol=TOL):
        return
    BATCH = batch_of(case)
    ta = hb.taylor_adaptive_batch(hb_system(hb, case), np.array(gold["state"], dtype=float).reshape(2, BATCH), BATCH,
                                  time=gold["time"] if gold["time"] else 0.0, tol=TOL, kernel=kernel)
    assert ta.get_order() == ORDER
    ta.step(write_tc=True)
    assert approximately(ta.tc, gold["tc"], EPS_MUL.get(case[0], 100.0)), (case[0], ta.tc, gold["tc"])


# ---- propagate_grid (src/taylor_adaptive_batch.cpp:1545-2055) ----

@pytest.mark.gpu
def test_propagate_grid_oscillator_gpu(kernel):
    """test/taylor_adaptive_batch.cpp:269-385: regular and random grids, forward and backward, against the closed
    form (the reference's tolerances) and against the oracle's restatement (step counts, outcomes, values)."""
    from test_oracle_golden import OSC_STATE, approximately, grid_fixtures, sys_oscillator
    if _refused(kernel, sys_oscillator()):
        return
    for name, grid, tol in grid_fixtures():
        ta = hb.taylor_adaptive_batch(sys_oscillator(), OSC_STATE, 4, kernel=kernel)
        ret = ta.propagate_grid(grid)
        assert ret.shape == (1000, 2, 4)
        assert [r[0] for r in ta.propagate_res] == [hb.taylor_outcome.time_limit] * 4
        assert np.array_equal(ta.time, grid[-1])
        amp = 1.0 + np.arange(4) / 10.0
        assert approximately(ret[:, 0, :], amp * np.sin(grid), tol), name
        assert approximately(ret[:, 1, :], amp * np.cos(grid), tol), name
        o = oracle.OracleIntegrator(hb.Program(sys_oscillator()), OSC_STATE, 4, mode=oracle.FMA)
        oret = o.propagate_grid(grid)
        assert np.max(np.abs(ret - oret)) < 1e-13, name
        assert [r[3] for r in ta.propagate_res] == [int(s) for s in o.n_steps], name
        assert np.allclose([r[1] for r in ta.propagate_res], o.min_h, rtol=1e-9)
        assert np.allclose([r[2] for r in ta.propagate_res], o.max_h, rtol=1e-9)
        assert lane_err(ta.state, o.state) < 1e-12


@pytest.mark.gpu
def test_propagate_grid_errors_and_trivial_cases():
    """test/taylor_adaptive_batch.cpp:162-268: argument checks (the reference's messages), a non-finite state, a
    grid made of the current time only."""
    st = np.array([0.05, 0.025, 0.051, 0.0251, 0.052, 0.0252, 0.053, 0.0253]).reshape(2, 4)
    ta = hb.taylor_adaptive_batch(sys_pendulum(), st, 4)
    inf = float("inf")
    with pytest.raises(ValueError, match="if the time grid is empty"):
        ta.propagate_grid([])
    for bad in ([1.0], [1.0, 2.0], [1.0, 2.0, 3.0, 4.0, 5.0]):
        with pytest.raises(ValueError, match=r"the grid has a size of %d, which is not a multiple of the batch size \(4\)"
                           % len(bad)):
            ta.propagate_grid(bad)
    with pytest.raises(ValueError, match="the first element of the time grid at batch index 2 has a value of 1, while "
                                         "the current time coordinate is 0"):
        ta.propagate_grid([0.0, 0.0, 1.0, 4.0])
    ta.set_time([0.0, 0.0, inf, 0.0])
    with pytest.raises(ValueError, match="if the current time is not finite"):
        ta.propagate_grid([0.0, 0.0, 0.0, 0.0])
    ta.set_time([0.0, 0.0, 0.0, 0.0])
    nf = "A non-finite time value was passed to propagate_grid"
    nm = "A non-monotonic time grid was passed to propagate_grid"
    for grid, msg in (([0, 0, inf, 0], nf), ([0, 0, 0, 0, 0, inf, 0, 0], nf), ([0, 0, 0, 0, 1, 1, -1, 1], nm),
                      ([0, 0, 0, 0, 1, 1, 1, 1, 0, 0, 0, inf], nf), ([0, 0, 0, 0, 1, 1, 1, 1, 2, 0, 0, 2], nm),
                      ([0, 0, 0, 0, 0, 1, 1, 1, 2, 2, 2, 2], nm), ([0, 0, 0, 0, 1, 0, 1, 1, 2, 2, 2, 2], nm),
                      ([0, 0, 0, 0, 1, 1, 1, 0, 2, 2, 2, 2], nm), ([0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 1, 2], nm)):
        with pytest.raises(ValueError, match=msg):
            ta.propagate_grid(np.array(grid, dtype=float))
    with pytest.raises(ValueError, match="A non-positive max_delta_t was passed to the propagate_grid"):
        ta.propagate_grid([0.0] * 4 + [1.0] * 4, max_delta_t=[1.0, 0.0, 1.0, 1.0])

    # An infinity in the state: lane 0 fails, the output stays NaN.
    ta = hb.taylor_adaptive_batch(sys_pendulum(), st, 4)
    ta.state[0, 0] = inf  # (like the reference's ta.get_state_data()[0] = inf)
    ret = ta.propagate_grid([0.0, 0.0, 0.0, 0.0])
    assert ret.shape == (1, 2, 4) and np.all(np.isnan(ret))
    assert [r[0] for r in ta.propagate_res] == [hb.taylor_outcome.err_nf_state] + [hb.taylor_outcome.time_limit] * 3

    # Propagate to the initial time.
    ta = hb.taylor_adaptive_batch(sys_pendulum(), st, 4)
    ret = ta.propagate_grid([0.0, 0.0, 0.0, 0.0])
    assert np.array_equal(ret[0], st)
    for oc, min_h, max_h, nsteps in ta.propagate_res:
        assert (oc, min_h, max_h, nsteps) == (hb.taylor_outcome.time_limit, inf, 0.0, 0)


@pytest.mark.gpu
def test_propagate_grid_limits_match_oracle(kernel):
    """max_delta_t and max_steps (early exit: remaining rows NaN, every outcome step_limit), 6-body system."""
    if _refused(kernel, sys_outer_ss(), high_accuracy=True):
        return
    st = outer_ss_batch_state(5, perturb=1e-3, seed=3)
    grid = np.linspace(0.0, 4.0, 41)[:, None] * np.array([1.0, 1.1, 0.9, 1.05, 0.95])[None, :]
    for kw in (dict(max_delta_t=[0.05, 0.2, 0.3, 0.11, 1.0]), dict(max_steps=5), dict()):
        ta = hb.taylor_adaptive_batch(sys_outer_ss(), st, 5, high_accuracy=True, kernel=kernel)
        o = oracle.OracleIntegrator(hb.Program(sys_outer_ss(), high_accuracy=True), st, 5, mode=oracle.FMA)
        ret = ta.propagate_grid(grid, **kw)
        oret = o.propagate_grid(grid, **kw)
        assert np.array_equal(np.isnan(ret), np.isnan(oret)), kw
        if "max_steps" in kw:
            assert np.isnan(ret).any() and not np.isnan(ret[:2]).any()
        m = ~np.isnan(oret)
        scale = np.max(np.abs(oret[m]))
        assert np.max(np.abs(ret[m] - oret[m])) < 1e-12 * scale, kw
        assert [r[0] for r in ta.propagate_res] == [int(x) for x in o.prop_outcome], kw
        assert [r[3] for r in ta.propagate_res] == [int(x) for x in o.n_steps], kw
        assert np.array_equal(ta.time, o.t_hi)


# ---- BASELINE.json configs[2] and [4] at oracle-sized batches (the tape of these systems lives in HBM) ----

@pytest.mark.gpu
@pytest.mark.parametrize("tape", ["nbody-cta", "global-cta"])
def test_nbody32_parity(tape):
    """model::nbody N = 32 (496 pair interactions, ~0.5 MB of tape per lane): a step and a short propagation
    against the oracle; identical step counts. Automatic selection = the N-body kernel with CTA teams."""
    from common import nbody32_batch_state, sys_nbody32
    batch = 8
    st = nbody32_batch_state(batch)
    P = hb.Program(sys_nbody32(), high_accuracy=False)
    assert (P.n_eq, P.order) == (192, 20)
    ta = hb.taylor_adaptive_batch(sys_nbody32(), st, batch)
    assert ta._b.kernel_info()["tape"] == "nbody-cta"
    ta._b.set_kernel(tape)
    assert ta._b.kernel_info()["tape"] == tape
    o = oracle.OracleIntegrator(P, st, batch, mode=oracle.FMA)
    ta.step(write_tc=True)
    o.step(write_tc=True)
    assert np.max(np.abs(ta.last_h / o.last_h - 1)) < 1e-12
    assert lane_err(ta.state, o.state) < 1e-13
    assert tc_err(ta.tc, o.tc, o.last_h) < 1e-12
    ta.propagate_until(1.5)
    o.propagate_until(1.5)
    assert [r[3] for r in ta.propagate_res] == [int(s) for s in o.n_steps]
    assert np.array_equal(ta.time, o.t_hi)
    assert lane_err(ta.state, o.state) < 1e-12


@pytest.mark.gpu
@pytest.mark.parametrize("tape", ["nn", "global-cta"])
def test_ffnn_parity(tape):
    """model::ffnn right-hand side (3 x 64 tanh, order 15): 10476 u variables per lane, sums of 64 products, tanh
    recurrences; a step and propagate_until(1) against the oracle; identical step counts. Automatic selection = the
    dense-network kernel: its layers are matrix products on the FP64 tensor cores, which sum the same 64 products of a
    neuron in another association (fused) than the reference's nested 8-term sums (src/math/sum.cpp:185-238) - the
    tolerances below (the ones of the generic kernel) bound that difference."""
    from common import FFNN_TOL, ffnn_batch_state, sys_ffnn
    batch = 17  # (odd: the last CTA of the dense-network kernel owns one lane only)
    st = ffnn_batch_state(batch)
    P = hb.Program(sys_ffnn(), tol=FFNN_TOL)
    assert (P.n_eq, P.order) == (4, 15)
    ta = hb.taylor_adaptive_batch(sys_ffnn(), st, batch, tol=FFNN_TOL)
    assert ta._b.kernel_info()["tape"] == "nn"
    ta._b.set_kernel(tape)
    assert ta._b.kernel_info()["tape"] == tape
    o = oracle.OracleIntegrator(P, st, batch, mode=oracle.FMA)
    ta.step(write_tc=True)
    o.step(write_tc=True)
    assert np.max(np.abs(ta.last_h / o.last_h - 1)) < 1e-11
    assert lane_err(ta.state, o.state) < 1e-13
    assert tc_err(ta.tc, o.tc, o.last_h) < 1e-12
    ta.propagate_until(1.0)
    o.propagate_until(1.0)
    assert [r[3] for r in ta.propagate_res] == [int(s) for s in o.n_steps]
    assert lane_err(ta.state, o.state) < 1e-12


# ---- continuous output (include/heyoka/continuous_output.hpp, producer src/taylor_adaptive_batch.cpp:1246-1346) ----

@pytest.mark.gpu
def test_continuous_output_gpu(kernel):
    """The batch block of test/c_output.cpp:289-420: the continuous output of propagate_until() against a grid
    propagation of the same integrator (100 eps), the closed form, and the oracle's restatement (same number of
    recorded iterations, same values)."""
    from test_oracle_golden import approximately, cout_fixture, sys_oscillator
    if _refused(kernel, sys_oscillator()):
        return
    ic, final_tm, grid = cout_fixture()
    for ha in (False, True):
        ta = hb.taylor_adaptive_batch(sys_oscillator(), ic, 4, high_accuracy=ha, kernel=kernel)
        co = ta.propagate_until(final_tm, c_output=True)
        assert co is not None and np.array_equal(ta.time, final_tm)
        assert [r[0] for r in ta.propagate_res] == [hb.taylor_outcome.time_limit] * 4
        lb, ub = co.get_bounds()
        assert np.all(lb == 0) and np.array_equal(ub, final_tm)
        ta2 = hb.taylor_adaptive_batch(sys_oscillator(), ic, 4, high_accuracy=ha, kernel=kernel)
        grid_out = ta2.propagate_grid(grid)
        o = oracle.OracleIntegrator(hb.Program(sys_oscillator(), high_accuracy=ha), ic, 4, mode=oracle.FMA)
        oco = o.propagate_until_cout(final_tm)
        assert co.get_n_steps() == oco.get_n_steps()
        assert [r[3] for r in ta.propagate_res] == [int(s) for s in o.n_steps]
        for k in range(grid.shape[0]):
            s = co(grid[k]).copy()
            assert approximately(s, grid_out[k], 100.0)
            assert np.max(np.abs(s - oco(grid[k]))) < 1e-13
        for tval in (0.0, 3.3, 9.99, -0.5, 11.0):  # the same time for every lane, also outside the bounds
            s = co(tval).copy()
            assert np.max(np.abs(s - oco(tval))) < 1e-12
        with pytest.raises(ValueError, match="at the non-finite time"):
            co([0.0, float("inf"), 0.0, 0.0])
    # max_steps: the recording stops with the loop, outcomes step_limit.
    ta = hb.taylor_adaptive_batch(sys_oscillator(), ic, 4, kernel=kernel)
    co = ta.propagate_until(final_tm, c_output=True, max_steps=3)
    assert co.get_n_steps() == 3 and [r[0] for r in ta.propagate_res] == [hb.taylor_outcome.step_limit] * 4
    # Non-finite state at the first step: no continuous output.
    ta = hb.taylor_adaptive_batch(sys_oscillator(), ic, 4, kernel=kernel)
    ta.state[0, 1] = float("inf")
    assert ta.propagate_until(final_tm, c_output=True) is None
    assert ta.propagate_res[1][0] == hb.taylor_outcome.err_nf_state
    # Continuous output TOGETHER with a step callback (src/taylor_adaptive_batch.cpp:1476-1500, hy_batch_propagate_until_
    # cout_cb): called after every recorded iteration, same recording; False stops with cb_stop and keeps what was
    # recorded; exceptions and alterations of the time come back to the caller.
    ref = hb.taylor_adaptive_batch(sys_oscillator(), ic, 4, kernel=kernel)
    co_ref = ref.propagate_until(final_tm, c_output=True)
    seen = []
    ta = hb.taylor_adaptive_batch(sys_oscillator(), ic, 4, kernel=kernel)
    co = ta.propagate_until(final_tm, c_output=True, callback=lambda t: seen.append(t.time.copy()) or True)
    assert len(seen) == co_ref.get_n_steps() == co.get_n_steps() and np.array_equal(seen[-1], final_tm)
    assert np.array_equal(ta.state, ref.state) and np.array_equal(co(3.3), co_ref(3.3))
    ta = hb.taylor_adaptive_batch(sys_oscillator(), ic, 4, kernel=kernel)
    count = []
    co = ta.propagate_until(final_tm, c_output=True, callback=lambda t: count.append(1) or len(count) < 3)
    assert co.get_n_steps() == 3 and [r[0] for r in ta.propagate_res] == [hb.taylor_outcome.cb_stop] * 4
    ta = hb.taylor_adaptive_batch(sys_oscillator(), ic, 4, kernel=kernel)

    def bad(t):
        raise KeyError("from the callback")
    with pytest.raises(KeyError, match="from the callback"):
        ta.propagate_until(final_tm, c_output=True, callback=bad)


@pytest.mark.gpu
def test_two_body_kepler_conservation_gpu(kernel):
    """test/two_body_batch.cpp:60-190 on the GPU: 200 steps of the hand-written equal-mass two-body system; every
    step agrees with a one-lane integrator taking the same step, and the Keplerian elements of both bodies are
    conserved to 1e4 epsilon."""
    from common import check_kepler_conservation, sys_two_body_symmetric, two_body_kepler_fixture
    if _refused(kernel, sys_two_body_symmetric()):
        return
    from test_oracle_golden import approximately
    kep, st = two_body_kepler_fixture()
    ta = hb.taylor_adaptive_batch(sys_two_body_symmetric(), st, 4, kernel=kernel)
    one = [hb.taylor_adaptive_batch(sys_two_body_symmetric(), st[:, i:i + 1], 1, kernel=kernel) for i in range(4)]
    for _ in range(200):
        prev, t_prev = ta.state.copy(), np.array(ta.time)
        ta.step()
        for i in range(4):
            one[i].state[:] = prev[:, i:i + 1]
            one[i].set_time([t_prev[i]])
            one[i].step()
            assert one[i].step_res[0][0] == ta.step_res[i][0]
            assert approximately(one[i].step_res[0][1], ta.step_res[i][1], 1e4)
            assert approximately(one[i].state[:, 0], ta.state[:, i], 1e5)
        check_kepler_conservation(ta.state, kep, approximately)


@pytest.mark.gpu
def test_lean_division_is_ieee():
    """The N-body kernel's own correctly-rounded division (nb_core.hpp div_rn: reciprocal seed + Newton + Markstein)
    returns the bits of the IEEE division on 2^30 pseudo-random pairs (fast path and out-of-line path)."""
    import ctypes as C
    bad = C.c_uint64(123)
    hb.check(hb.lib.hy_selftest_div(1 << 30, 20260924, C.byref(bad)))
    assert bad.value == 0
