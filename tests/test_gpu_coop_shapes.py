"""Every compiled shape of the cooperative kernel (k_coop, kernels.cuh) on the device, opcode by opcode and at high
orders: bit for bit against the oracle, against the HBM-tape kernel k_hbm, and within the series reference's bound.

Why bit for bit. Every k_coop shape and k_hbm run the same diff_op(), pow_eval(), step-size and double-length time
code with the same libdevice functions, compiled with -fmad=false: they must agree to the bit on any program, for free
steps and propagations alike. k_hbm keeps every u variable at every order, so it is a device reference that does not
depend on the residency plan (smem_plan.cpp: which rows keep their history). Against the oracle's FMA mode the only
differences are libdevice vs glibc at order 0 of the transcendental ops, and pow() in the step size. "Centred" initial
conditions (every transcendental's argument exactly 0 at order 0, exactly 1 for log and general pow) remove the first;
a step clamped by max_delta_t removes the second. No exception to exactness is needed.

What kernel_info() reports is checked against coop_expected(), which restates setup_coop() / setup_coop_global()
(batch.cu) from the plan's sizes (tests/cpp/nb_emul.cpp: coop_emul_plan()); test_every_instantiation_is_launched()
then checks without a GPU that the cases launch all 70 compiled entries of coop_inst.cu and both k_hbm kernels:

| variant (L, N, MAXT, MODE) | case that launches it |
|---|---|
| MODE 1, every (L, N), MAXT 256 | `rand3@4`, forced shape, 64 threads |
| MODE 1, every (L, N), MAXT 512 | `tanh_exp_log@3`, forced shape, 288 threads |
| MODE 0, every (L, N), MAXT 256 / 512 | `nbody3@9` / `nbody3_m1@3`, `tape="smem"`, 64 / 288 threads |
| MODE 4: (1,1) (2,1) (4,1) (2,2) (4,2) (8,2) | `rand0@20`, `tape="global"` |
| MODE 5: (1,1) (2,1) (2,2) (4,2) | `rand0@20`, `tape="global-cta"` |
| k_hbm step / propagate | every case's reference run |

Requests that cannot run (a shape that is not compiled, a table that does not fit) must raise the documented
ValueError instead of running another kernel."""
import ctypes as C
import functools

import numpy as np
import pytest

import heyoka_b200 as hb
import oracle
import series_ref as sr
from test_nb_plan import _emul, nb_lane_states, nb_order_program, nb_order_tol, nb_system
from test_series_reference import SERIES_BOUND

SMEM_OPTIN = 227 * 1024    # cudaDeviceProp::sharedMemPerBlockOptin of an H100
SMEM_PER_SM = 228 * 1024   # cudaDeviceProp::sharedMemPerMultiprocessor
RESERVE = 1024             # setup_coop()'s per-block margin
H100_SMS = 132

SMEM_LN = [(1, 1), (2, 1), (4, 1), (8, 1), (16, 1), (32, 1), (2, 2), (4, 2), (8, 2), (16, 2), (32, 2), (4, 4), (8, 4),
           (16, 4), (32, 4)]
GLOBAL_LN = {4: [(1, 1), (2, 1), (4, 1), (2, 2), (4, 2), (8, 2)], 5: [(1, 1), (2, 1), (2, 2), (4, 2)]}
COMPILED = ({(L, N, mt, md) for L, N in SMEM_LN for mt in (256, 512) for md in (0, 1)}
            | {(L, N, 512, md) for md, lns in GLOBAL_LN.items() for L, N in lns})
assert len(COMPILED) == 70

_lib = functools.cache(_emul)


@functools.cache
def _coop_plan(P, fuse=True, fuse_sv=True, spill=False):
    out = (C.c_uint32 * 6)()
    assert _lib().coop_emul_plan(P._h, int(fuse), int(fuse_sv), int(spill), out) == 0
    return dict(zip(("n_slots", "n_gslots", "n_items", "n_segments", "elementary", "blob_bytes"), out))


def _cwb(n_slots, L):
    return (n_slots * L + 2 * L + (L + 1) // 2 + 1) // 2 * 2 * 8


def coop_expected(P, batch, tape="smem", lanes_per_warp=0, lanes_per_thread=0, block_threads=0, fuse=True,
                  fuse_sv=True, spill=False):
    """What hy_batch::configure() (batch.cu) chooses for a program that is neither N-body- nor network-shaped, or
    for any program with tape "smem" / "global" / "global-cta": ("refused", message) or a dict of kernel_info()'s
    fields and the compiled variant (L, N, MAXT, MODE). Restates setup_coop() / setup_coop_global() line by line; the
    grid of the shared-memory kernel depends on the occupancy the driver reports, so it is given as a function of
    kernel_info()'s blocks_per_sm."""
    L, N, threads = lanes_per_warp, lanes_per_thread, block_threads
    pl = _coop_plan(P, fuse, fuse_sv, spill)
    if tape in ("auto", "smem"):
        if N == 0:
            N = 2 if (L == 0 or L >= 2) else 1
        blob, ns = pl["blob_bytes"], pl["n_slots"]
        fits = True
        if L == 0:
            avg = pl["n_items"] / max(1, pl["n_segments"])
            for cand in (1, 2, 4, 8, 16, 32):
                if cand < N:
                    continue
                b = _cwb(ns, cand)
                if blob + b + RESERVE > SMEM_OPTIN or (SMEM_PER_SM - blob) // b < 4:
                    break
                L = cand
                if avg * cand / N >= 12.:
                    break
            if L == 0:
                if blob + _cwb(ns, N) + RESERVE > SMEM_OPTIN:
                    fits = False
                L = N
        wb = _cwb(ns, L)
        if fits and (blob > 24 * 1024 or blob + wb + RESERVE > SMEM_OPTIN):
            fits = False
        if fits:
            if threads == 0:
                threads = 32 * max(min((SMEM_OPTIN - RESERVE - blob) // wb, 16), 1)
            if threads % 32 or threads > 512:
                return ("refused", "Invalid number of threads")
            maxt = 256 if threads <= 256 else 512
            if (L, N) not in SMEM_LN:
                return ("refused", "Unsupported cooperative kernel configuration")
            smem = blob + threads // 32 * wb
            if smem + RESERVE <= SMEM_OPTIN:
                lpb = L * threads // 32
                return dict(tape="smem", lanes_per_warp=L, lanes_per_thread=N, block_threads=threads, smem_bytes=smem,
                            grid=lambda occ: max(1, min(H100_SMS * occ, -(-batch // lpb))),
                            variant=(L, N, maxt, pl["elementary"]))
        if tape == "smem":
            return ("refused", "does not fit in shared memory")
        L, N, threads, cta = 0, 0, 0, -1
    else:
        cta = 1 if tape == "global-cta" else 0
    # setup_coop_global() (the planner runs without the overflow tape there).
    pl = _coop_plan(P, fuse, fuse_sv, False)
    if N == 0:
        N = 2 if (L == 0 or L >= 2) else 1
    threads = threads or 512
    if threads % 32 or threads > 512:
        return ("refused", "Invalid number of threads")
    warps = threads // 32
    if cta < 0:
        avg = pl["n_items"] / max(1, pl["n_segments"])
        cta = 1 if (avg >= 128. and -(-batch // N) < 8 * H100_SMS * warps) else 0
    if L == 0:
        L = N
        while cta == 0 and 2 * L <= 8 and batch // (2 * L) >= H100_SMS * 16:
            L *= 2
    mode = 5 if cta else 4
    if (L, N) not in GLOBAL_LN[mode]:
        return ("refused", "Unsupported cooperative kernel configuration \\(global tape\\)")
    teams = 1 if cta else warps
    return dict(tape="global-cta" if cta else "global", lanes_per_warp=L, lanes_per_thread=N, block_threads=threads,
                smem_bytes=0, grid=lambda occ: max(1, min(H100_SMS, -(-batch // (L * teams)))),
                variant=(L, N, 512, mode))


# ---- programs ------------------------------------------------------------------------------------------------------

class RandomDAG:
    """A seeded random system with 4 to 8 equations: a pool of shared subexpressions built level by level (depth 4 to
    5) over the state variables, 3 parameters and time; each right-hand side sums several pool entries, one of them
    more than 8 terms (split into partial sums), and one equation sums 40 products of state variables (a segment of
    more than 32 independent items). Bounded functions keep every argument inside its domain."""

    def __init__(self, seed):
        self.seed = seed
        rng = np.random.default_rng(500 + seed)
        self.n_eq = int(rng.integers(4, 9))
        self.depth = int(rng.integers(4, 6))
        self.n_pars = 3
        self._rng_state = rng.bit_generator.state

    def rhs(self, m, x):
        rng = np.random.default_rng()
        rng.bit_generator.state = self._rng_state
        pool = list(x) + [m.p(i) * x[i % len(x)] for i in range(self.n_pars)] + [m.t() * x[0]]
        for _ in range(self.depth):
            new = []
            for _ in range(6):
                a, b = (pool[int(k)] for k in rng.integers(len(pool), size=2))
                kind = int(rng.integers(9))
                new.append([a + b, a * b, a - m.c(0.75) * b, m.sin(a) * b, m.cos(a + b),
                            m.tanh(a), a / (m.c(2.5) + m.sin(b)), m.exp(m.tanh(a)) - b,
                            m.sqrt(m.c(3.) + m.cos(a)) + m.log(m.c(2.) + m.sin(b))][kind])
            pool += new
        out = []
        for i in range(len(x)):
            k = 12 if i == 0 else int(rng.integers(2, 5))
            terms = [pool[int(j)] for j in rng.integers(len(x), len(pool), size=k)]
            out.append(m.c(0.1) * m.sum(terms) - x[i])
        out[1] = out[1] + m.c(0.01) * m.sum([x[i % len(x)] * x[(i * 7 + 3) % len(x)] * m.c(1. + 0.01 * i)
                                             for i in range(40)])
        return out

    def hb_sys(self):
        xs = hb.make_vars(*["x%d" % i for i in range(self.n_eq)])
        return [(v, r) for v, r in zip(xs, self.rhs(sr.hb_backend(), list(xs)))]

    def program(self, order):
        P = hb.Program(self.hb_sys(), tol=sr.order_tol(order))
        assert P.order == order
        return P

    def state(self, batch, centred=False, seed=0):
        return np.random.default_rng(seed + 77).uniform(-1., 1., (self.n_eq, batch))

    def pars(self, batch):
        return np.random.default_rng(self.seed).uniform(-1., 1., (self.n_pars, batch))

    def t0(self, batch):
        return np.linspace(-1., 1., batch)


class NBody:
    """model::nbody (test_nb_plan.NB_SYSTEMS) on the cooperative kernel: with superinstructions only (MODE 0)."""

    def __init__(self, name):
        self.name = name

    def hb_sys(self):
        return nb_system(self.name)

    def program(self, order):
        return nb_order_program(self.name, order)

    def state(self, batch, centred=False, seed=0):
        return nb_lane_states(self.name, batch, seed=seed)

    def pars(self, batch):
        return None

    def t0(self, batch):
        return np.zeros(batch)


def system(key):
    if key.startswith("rand"):
        return RandomDAG(int(key[4:]))
    if key.startswith("nbody") or key.startswith("two_body"):
        return NBody(key)
    return sr.SYSTEMS_BY_NAME[key]


@functools.cache
def program(key, order):
    return system(key).program(order)


def make_ta(key, order, st, kernel, pars=None, t0=0.):
    s = system(key)
    if getattr(s, "arrays", None) is not None:
        return _ArrayBatch(program(key, order), st, kernel, pars, t0)
    tol = nb_order_tol(order) if isinstance(s, NBody) else sr.order_tol(order)
    return hb.taylor_adaptive_batch(s.hb_sys(), st, st.shape[1], tol=tol, pars=pars, time=t0, kernel=kernel)


class _ArrayBatch:
    """The part of taylor_adaptive_batch these tests use, over a program built from raw arrays (hb.Batch)."""

    def __init__(self, P, st, kernel, pars, t0):
        self.P, self.n = P, st.shape[1]
        self._b = hb.Batch(P, self.n)
        if kernel is not None:
            self._b.set_kernel(**kernel)
        self.state = np.array(st, dtype=np.float64)
        self.pars = np.zeros((max(P.n_pars, 1), self.n)) if pars is None else np.array(pars, dtype=np.float64)
        self.set_time(t0)
        self.last_h = np.zeros(self.n)

    def set_time(self, t):
        self.dtime = (np.array(np.broadcast_to(t, (self.n,)), dtype=np.float64), np.zeros(self.n))

    def _push(self):
        self._b.upload(self.state, self.pars[:self.P.n_pars] if self.P.n_pars else None, *self.dtime)

    def _pull(self, wtc):
        self.state, t_hi, t_lo, self.last_h = self._b.download()
        self.dtime = (t_hi, t_lo)
        self.tc = self._b.tc() if wtc else None

    def step(self, max_delta_ts=None, write_tc=False):
        self._push()
        self._b.step(None if max_delta_ts is None else np.ascontiguousarray(np.broadcast_to(max_delta_ts, (self.n,)),
                                                                          dtype=np.float64), write_tc=write_tc)
        self._pull(write_tc)
        oc, h = self._b.step_res()
        self.step_res = [(int(o), float(v)) for o, v in zip(oc, h)]

    def propagate_until(self, ts, max_delta_t=None, write_tc=False):
        self._push()
        self._b.propagate_until(np.ascontiguousarray(np.broadcast_to(ts, (self.n,)), dtype=np.float64),
                                max_delta_t=None if max_delta_t is None else np.ascontiguousarray(max_delta_t),
                                write_tc=write_tc)
        self._pull(write_tc)
        oc, mn, mx, ns = self._b.prop_res()
        self.propagate_res = [(int(a), float(b), float(c), int(d)) for a, b, c, d in zip(oc, mn, mx, ns)]


def _ki_check(ta, P, batch, kw, **opts):
    e = coop_expected(P, batch, **kw, **opts)
    assert isinstance(e, dict), (kw, e)
    ki = ta._b.kernel_info()
    got = {k: ki[k] for k in ("tape", "lanes_per_warp", "lanes_per_thread", "block_threads", "smem_bytes")}
    assert got == {k: e[k] for k in got}, (kw, got, e)
    assert ki["grid"] == e["grid"](ki["blocks_per_sm"]), (kw, ki)
    return e


# ---- coverage (no GPU) ---------------------------------------------------------------------------------------------

BATCH = 37  # odd, > 32: partial last warp / CTA for every shape


def shape_requests():
    """Every compiled (L, N) with 64 threads (MAXT 256) and 288 threads (MAXT 512: 9 warps fit where 16 do not), the
    automatic shape of the shared-memory kernel, every global-tape shape; and requests that must be refused."""
    out = [dict(tape="smem", lanes_per_warp=L, lanes_per_thread=N, block_threads=bt) for L, N in SMEM_LN
           for bt in (64, 288)]
    out += [dict(tape="smem"), dict(tape="smem", block_threads=512)]
    out += [dict(tape="global" if md == 4 else "global-cta", lanes_per_warp=L, lanes_per_thread=N)
            for md, lns in GLOBAL_LN.items() for L, N in lns]
    out += [dict(tape="smem", lanes_per_warp=3), dict(tape="smem", lanes_per_warp=1, lanes_per_thread=2),
            dict(tape="smem", lanes_per_warp=2, lanes_per_thread=4), dict(tape="global", lanes_per_warp=16),
            dict(tape="global-cta", lanes_per_warp=8, lanes_per_thread=2)]
    return out


# (system, order) of the cross-kernel identity: random DAGs at the default order and at orders 9 and 33, N-body programs
# on the shared-memory kernel (superinstructions only: MODE 0), at low orders where 288 threads of 32 lanes fit.
SHAPE_CASES = [("rand0", 20), ("rand0", 9), ("rand1", 20), ("rand2", 33), ("rand3", 4), ("nbody3", 9),
               ("nbody3_m1", 3), ("two_body_m10", 20), ("tanh_exp_log", 3)]


def test_every_instantiation_is_launched():
    """(No GPU needed.) The shape cases launch every compiled cooperative variant; coop_expected() of each request is
    what the GPU tests check kernel_info() against."""
    seen = set()
    for key, order in SHAPE_CASES:
        P = program(key, order)
        for kw in shape_requests():
            e = coop_expected(P, BATCH, **kw)
            if isinstance(e, dict):
                seen.add(e["variant"])
    assert seen == COMPILED, sorted(COMPILED - seen)
    # The requests that must be refused are refused, for the documented reason.
    P = program("rand0", 20)
    for kw in shape_requests()[-5:]:
        assert coop_expected(P, BATCH, **kw)[0] == "refused", kw
    # The opcode systems run on the shared-memory kernel in MODE 1 at every order of the exactness test.
    for s in sr.SYSTEMS:
        for order in EXACT_ORDERS:
            e = coop_expected(program(s.name, order), 5, tape="auto")
            assert e["tape"] == "smem" and e["variant"][3] == 1, (s.name, order, e)


# ---- opcode systems against the oracle, bit for bit ----------------------------------------------------------------

EXACT_ORDERS = (3, 4, 8, 9, 20, 33) + tuple(range(64, 72))
EXACT_CASES = [(s.name, o) for s in sr.SYSTEMS for o in EXACT_ORDERS]
OBATCH = 5


def _snap(ta, tc=True):
    return dict(state=ta.state.copy(), t_hi=ta.dtime[0].copy(), t_lo=ta.dtime[1].copy(), last_h=ta.last_h.copy(),
                tc=ta.tc.copy() if tc else None)


def _ulps(a, b):
    return np.max(np.where(a == b, 0., np.abs(a - b) / np.spacing(np.abs(b))))


@pytest.mark.gpu
@pytest.mark.parametrize("name,order", EXACT_CASES, ids=["%s@%d" % c for c in EXACT_CASES])
def test_opcode_systems_match_oracle_bit_for_bit(name, order):
    """Centred initial conditions, the automatic kernel: one free step (coefficients and outcomes exactly, the step
    size within 4 ulps: libdevice pow() within 2, glibc's within 1, then one rounded product); clamped steps forward and
    backward (state, double-length time, step size, coefficients exactly); an all-clamped propagate_until() exactly
    for the systems whose order-0 values need no libm."""
    s = sr.SYSTEMS_BY_NAME[name]
    P = program(name, order)
    st, pars, t0 = s.state(OBATCH, centred=True), s.pars(OBATCH), s.t0(OBATCH)

    def orc():
        o = oracle.OracleIntegrator(P, st, OBATCH, pars=pars, mode=oracle.FMA)
        o.t_hi[:] = t0
        return o

    def dev():
        ta = make_ta(name, order, st, dict(tape="auto"), pars, t0)
        _ki_check(ta, P, OBATCH, dict(tape="auto"))
        return ta

    o = orc()
    o.step(write_tc=True)
    ta = dev()
    ta.step(write_tc=True)
    assert np.array_equal(ta.tc, o.tc), np.argwhere(ta.tc != o.tc)[:5]
    assert [r[0] for r in ta.step_res] == [int(x) for x in o.step_outcome]
    assert _ulps(ta.last_h, o.last_h) <= 4.
    h_nat = o.last_h.copy()
    assert np.all(np.isfinite(h_nat))
    for sign in (1., -1.):
        lim = 0.5 * sign * np.abs(h_nat)
        o = orc()
        o.step(lim, write_tc=True)
        ta = dev()
        ta.step(lim, write_tc=True)
        assert np.array_equal(o.last_h, lim) and np.array_equal(ta.last_h, lim)
        for k, v in (("state", o.state), ("t_hi", o.t_hi), ("t_lo", o.t_lo), ("tc", o.tc)):
            assert np.array_equal(_snap(ta)[k], v), (sign, k)
        assert [r[0] for r in ta.step_res] == [int(x) for x in o.step_outcome]
    if not s.transcendental:
        # (5 to 12 steps of a tenth of the first free step: none of them free, also where a relu switches.)
        tf = t0 + np.linspace(0.5, 1.2, OBATCH) * np.abs(h_nat)
        mdt = 0.1 * np.abs(h_nat)
        o = orc()
        o.propagate_until(tf, max_delta_t=mdt)
        assert np.all(o.max_h == 0.)  # (no free step: no step size went through pow())
        ta = dev()
        ta.propagate_until(tf, max_delta_t=mdt)
        for k, v in (("state", o.state), ("t_hi", o.t_hi), ("t_lo", o.t_lo), ("last_h", o.last_h)):
            assert np.array_equal(_snap(ta, tc=False)[k], v), k
        assert [r[0] for r in ta.propagate_res] == [int(x) for x in o.prop_outcome]
        assert [r[3] for r in ta.propagate_res] == [int(x) for x in o.n_steps]


@pytest.mark.gpu
@pytest.mark.parametrize("name", [s.name for s in sr.SYSTEMS])
def test_opcode_systems_against_series(name):
    """Non-centred initial conditions (order-0 values through libdevice): the device's coefficients within the series
    reference's bound (test_series_reference.py), at orders 8 and 40."""
    s = sr.SYSTEMS_BY_NAME[name]
    st, pars, t0 = s.state(OBATCH, centred=False, seed=3), s.pars(OBATCH), s.t0(OBATCH)
    ref = sr.series_jets(s, st, pars, t0, 40)
    for order in (8, 40):
        ta = make_ta(name, order, st, dict(tape="auto"), pars, t0)
        ta.step(write_tc=True)
        err = sr.normalised_err(ta.tc, ref[:, :order + 1])
        assert err < SERIES_BOUND, (name, order, err)


# ---- every shape against k_hbm -------------------------------------------------------------------------------------

def _run_seq(key, order, st, kernel, pars, t0, tf, grid, check=None):
    """step(write_tc), propagate_until() to per-lane final times with and without write_tc, propagate_grid()."""
    ta = make_ta(key, order, st, kernel, pars, t0)
    if check is not None:
        check(ta)
    out = {}
    ta.step(write_tc=True)
    out["step"] = _snap(ta) | {"res": list(ta.step_res)}
    for wtc in (True, False):
        ta.state[:] = st
        ta.set_time(t0)
        ta.propagate_until(tf, write_tc=wtc)
        out["prop%d" % wtc] = _snap(ta, tc=wtc) | {"res": list(ta.propagate_res)}
    if grid is not None:
        ta.state[:] = st
        ta.set_time(t0)
        out["grid"] = {"ret": ta.propagate_grid(grid), "res": list(ta.propagate_res)}
    return out


def _assert_same(ref, got, what):
    for phase, d in ref.items():
        for k, v in d.items():
            if v is None:
                continue
            if isinstance(v, np.ndarray):
                assert np.array_equal(v, got[phase][k], equal_nan=True), (what, phase, k)
            else:
                assert v == got[phase][k], (what, phase, k)


def _times(key, order, st, pars, t0):
    """Per-lane final times of 2 to 6 first steps (most lanes finish before the slowest one: masked zero-length steps
    and re-expansion), and a grid over the first 4."""
    ta = make_ta(key, order, st, dict(tape="hbm"), pars, t0)
    ta.step()
    h = np.abs(ta.last_h)
    n = st.shape[1]
    tf = t0 + np.linspace(2., 6., n) * h
    grid = t0[None, :] + np.linspace(0., 4., 9)[:, None] * h[None, :]
    return tf, grid


@pytest.mark.gpu
@pytest.mark.parametrize("key,order", SHAPE_CASES, ids=["%s@%d" % c for c in SHAPE_CASES])
def test_shapes_match_hbm_bit_for_bit(key, order):
    """Every forced shape, the automatic one, "global" and "global-cta": the bits of k_hbm for step(write_tc=True),
    propagate_until() to per-lane final times with and without write_tc, and propagate_grid(). A request that cannot
    run is refused with the documented error."""
    s = system(key)
    P = program(key, order)
    st, pars, t0 = s.state(BATCH, seed=order), s.pars(BATCH), s.t0(BATCH)
    tf, grid = _times(key, order, st, pars, t0)
    def is_hbm(ta):
        assert ta._b.kernel_info()["tape"] == "hbm"

    ref = _run_seq(key, order, st, dict(tape="hbm"), pars, t0, tf, grid, check=is_hbm)
    assert np.count_nonzero(ref["prop1"]["last_h"] == 0.) >= 1  # lanes that finished early
    ran = set()
    for kw in shape_requests():
        e = coop_expected(P, BATCH, **kw)
        if isinstance(e, dict):
            got = _run_seq(key, order, st, kw, pars, t0, tf, grid, check=lambda ta: _ki_check(ta, P, BATCH, kw))
            _assert_same(ref, got, kw)
            ran.add(e["variant"])
        else:
            ta = make_ta(key, order, st, None, pars, t0)
            with pytest.raises(ValueError, match=e[1]):
                ta._b.set_kernel(**kw)
    assert ran


# ---- plan options --------------------------------------------------------------------------------------------------

OPTION_CASES = [("rand0", 20), ("rand2", 33), ("trig", 20), ("pow", 9), ("relu", 20), ("nbody3", 20), ("nbody4", 9),
                ("two_body_m10", 20)]
OPTIONS = [("HEYOKA_B200_FUSE", "0", dict(fuse=False)), ("HEYOKA_B200_FUSE_SV", "0", dict(fuse_sv=False)),
           ("HEYOKA_B200_SPILL", "1", dict(spill=True))]


@pytest.mark.gpu
@pytest.mark.parametrize("key,order", OPTION_CASES, ids=["%s@%d" % c for c in OPTION_CASES])
def test_plan_options_give_the_same_bits(key, order, monkeypatch):
    """HEYOKA_B200_FUSE=0 (no superinstructions: N-body programs run in MODE 1), HEYOKA_B200_FUSE_SV=0 (the generic
    state-variable pass instead of the fused propagation) and HEYOKA_B200_SPILL=1 (the overflow tape in global memory)
    give the bits of the default plan, on the automatic and two forced shared-memory shapes."""
    s = system(key)
    P = program(key, order)
    st, pars, t0 = s.state(BATCH, seed=5), s.pars(BATCH), s.t0(BATCH)
    tf, grid = _times(key, order, st, pars, t0)
    kws = [dict(tape="smem"), dict(tape="smem", lanes_per_warp=4, lanes_per_thread=1, block_threads=64),
           dict(tape="smem", lanes_per_warp=8, lanes_per_thread=2, block_threads=288)]
    for kw in kws:
        if not isinstance(coop_expected(P, BATCH, **kw), dict):
            continue
        ref = _run_seq(key, order, st, kw, pars, t0, tf, grid, check=lambda ta: _ki_check(ta, P, BATCH, kw))
        for var, val, opts in OPTIONS:
            e = coop_expected(P, BATCH, **kw, **opts)
            if not isinstance(e, dict):
                continue
            with monkeypatch.context() as mc:
                mc.setenv(var, val)
                got = _run_seq(key, order, st, kw, pars, t0, tf, grid,
                               check=lambda ta: _ki_check(ta, P, BATCH, kw, **opts))
            if var == "HEYOKA_B200_FUSE" and isinstance(s, NBody):
                assert e["variant"][3] == 1
            if var == "HEYOKA_B200_SPILL" and isinstance(s, NBody):
                assert _coop_plan(P, spill=True)["n_gslots"] > 0
            _assert_same(ref, got, (kw, var))


# ---- batch tails ---------------------------------------------------------------------------------------------------

TAIL_CASES = [("rand1", 20, dict(tape="smem", lanes_per_warp=8, lanes_per_thread=2, block_threads=64)),
              ("rand3", 4, dict(tape="smem", lanes_per_warp=32, lanes_per_thread=4, block_threads=64)),
              ("trig", 20, dict(tape="auto")), ("nbody3", 9, dict(tape="smem", lanes_per_warp=4, lanes_per_thread=1,
                                                                  block_threads=64)),
              ("rand1", 20, dict(tape="global", lanes_per_warp=8, lanes_per_thread=2)),
              ("rand1", 20, dict(tape="global-cta", lanes_per_warp=4, lanes_per_thread=2))]
N_BASE = 7


@pytest.mark.gpu
@pytest.mark.parametrize("key,order,kw", TAIL_CASES, ids=["%s@%d-%s-%d" % (k, o, w["tape"], w.get("lanes_per_warp", 0))
                                                          for k, o, w in TAIL_CASES])
def test_batch_tails(key, order, kw):
    """Batch sizes 1, L - 1, 3 L + 1 and one larger than grid x warps x L: every lane gives the bits of the same lane
    run alone (a step with write_tc, propagate_until())."""
    s = system(key)
    P = program(key, order)
    assert isinstance(coop_expected(P, 1, **kw), dict)
    base, bpars = s.state(N_BASE, seed=11), s.pars(N_BASE)

    def run(idx):
        st = np.ascontiguousarray(base[:, idx])
        pars = None if bpars is None else np.ascontiguousarray(bpars[:, idx])
        t0 = s.t0(N_BASE)[idx]
        ta = make_ta(key, order, st, kw, pars, t0)
        e = _ki_check(ta, P, len(idx), kw)
        ta.step(write_tc=True)
        r = {"step": _snap(ta) | {"res": list(ta.step_res)}}
        ta.state[:] = st
        ta.set_time(t0)
        ta.propagate_until(t0 + 0.05 * (1 + np.arange(N_BASE)[idx] % 3))
        r["prop"] = _snap(ta, tc=False) | {"res": list(ta.propagate_res)}
        return r, e, ta._b.kernel_info()

    alone = [run(np.array([i]))[0] for i in range(N_BASE)]
    _, e, ki = run(np.arange(N_BASE))
    L = e["lanes_per_warp"]
    teams = 1 if ki["tape"] == "global-cta" else ki["block_threads"] // 32
    big = ki["n_sms"] * max(ki["blocks_per_sm"], 1) * teams * L + 3
    for batch in sorted({1, max(L - 1, 1), 3 * L + 1, big}):
        idx = np.arange(batch) % N_BASE
        r, _, ki = run(idx)
        assert batch != big or batch > ki["grid"] * teams * L
        for phase in ("step", "prop"):
            for k in ("state", "t_hi", "t_lo", "tc", "last_h"):
                if alone[0][phase][k] is None or (phase == "prop" and k == "last_h"):
                    continue
                exp = np.stack([alone[i][phase][k][..., 0] for i in range(N_BASE)], axis=-1)[..., idx]
                assert np.array_equal(r[phase][k], exp), (batch, phase, k)
            assert r[phase]["res"] == [alone[i][phase]["res"][0] for i in idx], (batch, phase)
