"""The oracle's jets of the opcode systems of series_ref.py against the 50-digit series reference, at orders 3 to 40 and
in the oracle's three summation modes (CPU only). Every coefficient of every state variable counts, normalised by
E(v, o) = max over lanes |c_ref[v, o]| with no |h|^o weight, so that a wrong high-order coefficient cannot hide behind
a small step. The same systems run on the device in test_gpu_coop_shapes.py, bit for bit against the oracle's FMA mode,
so this pins the device's jets to the reference as well.

The bound, SERIES_BOUND = 5e-12, was calibrated on an x86-64 CPU: the oracle's worst normalised error over all
systems, orders and modes was 5.8e-13 (sigmoid: its recurrence subtracts sigmoid^2 from sigmoid, which cancels; every
other system stays below 5e-14), so the bound is about 9 times above it. A wrong
convolution bound, history row or quotient moves a coefficient by far more (O(1) in these units)."""
import numpy as np
import pytest

import oracle
import series_ref as sr

ORDERS = (3, 4, 8, 9, 20, 33, 40)
MODES = {"pairwise": oracle.PAIRWISE, "seq": oracle.SEQ, "fma": oracle.FMA}
BATCH = 3
SERIES_BOUND = 5e-12


def reference(sysdef, order, centred=False, batch=BATCH, seed=1):
    st = sysdef.state(batch, centred=centred, seed=seed)
    pars, t0 = sysdef.pars(batch), sysdef.t0(batch)
    return st, pars, t0, sr.series_jets(sysdef, st, pars, t0, order)


@pytest.mark.parametrize("name", [s.name for s in sr.SYSTEMS])
def test_system_lowers_to_its_opcodes(name):
    s = sr.SYSTEMS_BY_NAME[name]
    got = sr.coop_opcodes(s.program(8))
    assert s.ops <= got, (name, s.ops - got)


def test_every_opcode_is_covered():
    """The systems together contain every opcode and every order-0 algorithm of pow by a number."""
    seen = set()
    for s in sr.SYSTEMS:
        seen |= sr.coop_opcodes(s.program(8))
    assert set(sr.OPNAMES) <= seen, set(sr.OPNAMES) - seen
    assert {("POW_VN", a) for a in range(5)} <= seen


def test_series_class_against_closed_forms():
    """The series arithmetic itself, on functions whose Taylor coefficients are known in closed form."""
    D = 12
    t = sr.Series([sr.mpf(0), sr.mpf(1)] + [sr.mpf(0)] * (D - 1))  # the series of t
    fact = [sr.mp.factorial(k) for k in range(D + 1)]
    e = sr.s_exp(t)
    s, c = sr.s_sincos(t)
    lg = sr.s_log(1 + t)
    q = 1 / (1 - t)
    sq = sr.s_sqrt(1 + t)
    for k in range(D + 1):
        assert abs(e.c[k] - 1 / fact[k]) < 1e-45
        assert abs(s.c[k] - ((-1) ** (k // 2) / fact[k] if k % 2 else 0)) < 1e-45
        assert abs(c.c[k] - (0 if k % 2 else (-1) ** (k // 2) / fact[k])) < 1e-45
        assert abs(lg.c[k] - (0 if k == 0 else sr.mpf((-1) ** (k + 1)) / k)) < 1e-45
        assert abs(q.c[k] - 1) < 1e-45
        assert abs(sq.c[k] - sr.mp.binomial(0.5, k)) < 1e-45
    th = sr.s_tanh(t)
    assert abs(th.c[3] + sr.mpf(1) / 3) < 1e-45 and abs(th.c[5] - sr.mpf(2) / 15) < 1e-45
    sg = sr.s_sigmoid(t)
    assert abs(sg.c[0] - 0.5) < 1e-45 and abs(sg.c[1] - 0.25) < 1e-45 and abs(sg.c[3] + sr.mpf(1) / 48) < 1e-45
    p = sr.s_pow(1 + t, sr.mpf(-1.5))
    for k in range(D + 1):
        assert abs(p.c[k] - sr.mp.binomial(-1.5, k)) < 1e-45
    # The jet of x' = x, x(0) = 1 is 1 / k!.
    jet = sr.series_jet(lambda m, x: [x[0]], [1.], [], 0., D)
    assert all(abs(jet[0][k] - 1 / fact[k]) < 1e-45 for k in range(D + 1))


@pytest.mark.parametrize("name", [s.name for s in sr.SYSTEMS])
def test_oracle_against_series(name):
    s = sr.SYSTEMS_BY_NAME[name]
    st, pars, t0, ref = reference(s, max(ORDERS))
    worst = 0.
    for order in ORDERS:
        P = s.program(order)
        for mode in MODES.values():
            o = oracle.OracleIntegrator(P, st, BATCH, pars=pars, mode=mode)
            o.t_hi[:] = t0
            o.step(write_tc=True)
            err = sr.normalised_err(o.tc, ref[:, :order + 1])
            worst = max(worst, err)
            assert err < SERIES_BOUND, (name, order, mode, err)
    print("%s: worst normalised error %.3g" % (name, worst))
