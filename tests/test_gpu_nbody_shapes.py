"""Every compiled shape of the N-body kernels (k_nb, nb_kernel.cuh; k_nb1, nb1_kernel.cuh) on the device, bit for bit
against the oracle, across body counts, orders, team shapes and batch tails.

Why bit for bit. For model::nbody programs (r^-3/2: HY_POW_NEG_SMALL_HALF) the order-0 power is 1 / sqrt(x)^3 in IEEE
operations and every division of the jet is correctly rounded (div_rn, div_si), so the device's Taylor coefficients
equal the oracle's FMA mode exactly; tests/test_nb_plan.py shows it for the same systems, orders and team shapes on the
host emulation of nb_core.hpp, so a failure here is in the device code. The one difference is the step size, which goes
through libdevice pow() on the device and glibc pow() in the oracle (<= 1 ulp each). A step whose size is set by
max_delta_t takes the pow out: it and every propagation whose steps are all clamped are bit-identical as well.

What is asserted for each shape: what kernel_info() reports equals what setup_nb() (batch.cu) must choose, recomputed
here from its shared-memory arithmetic (nb_expected()), so that no case silently runs another kernel;
test_every_instantiation_is_launched() then checks, without a GPU, that the cases below launch every entry of the
nb_inst.cu / nb1_inst.cu families.

No compiled variant is unreachable. The role table is read from global memory (roles_in_smem = 0) only by CTA teams
whose private rows and role table do not fit in shared memory together: model::nbody with 12 bodies at orders 9 and 10
(rows on chip), with 9 bodies at order 25 (rows off chip); _cases() finds those orders with nb_expected() and runs them."""
import ctypes as C
import functools

import numpy as np
import pytest

import heyoka_b200 as hb
import oracle
from test_gpu_parity import lane_err, tc_err
from test_nb_plan import NB_SYSTEMS, _emul, _plan, nb_lane_states, nb_order_program, nb_order_tol, nb_system

SMEM_OPTIN = 227 * 1024  # shared memory per block an H100 kernel can opt in to (cudaDeviceProp::sharedMemPerBlockOptin)
H100_SMS = 132
RESERVE = 1024           # setup_nb()'s margin

# The compiled instantiations (nb_inst.cu families lt{1,2,4,8,16,32}_cta0 and lt1_cta1, nb1_inst.cu):
# (LT, CTA, OFFCHIP, MAXT, one thread per lane). Each has a step and a propagate kernel; both run in every case.
COMPILED = ({(lt, False, False, mt, False) for lt in (1, 2, 4, 8, 16, 32) for mt in (256, 384, 512)}
            | {(1, True, False, 512, False), (1, True, True, 512, False)}
            | {(32, False, False, mt, True) for mt in (256, 384, 512)})

NF = hb.taylor_outcome.err_nf_state


# ---- setup_nb()'s choice, restated ---------------------------------------------------------------------------------

_lib = functools.cache(_emul)


def _roles(P, tt, lt, nl):
    out = (C.c_uint32 * 4)()
    assert _lib().nb_emul_roles(P._h, C.c_uint32(tt), C.c_uint32(lt), C.c_uint32(nl), out) == 0
    return list(out)


def _coop_warp_bytes(slots, lt):
    return (slots * lt + 2 * lt + (lt + 1) // 2 + 1) // 2 * 2 * 8


def nb_expected(P, batch, tape="auto", lanes_per_warp=0, block_threads=0, n_sms=H100_SMS):
    """What hy_batch::configure() / setup_nb() (batch.cu) choose for an N-body-shaped program on an H100: None if the
    request is refused, else kernel_info()'s tape, lanes_per_warp, block_threads, smem_bytes and grid, and the compiled
    variant that runs. Restates the code line by line; the one-thread-per-lane test of make_nb1_tab() is reduced to what
    decides it for the two-body systems of NB_SYSTEMS (one pair interaction, order >= 4)."""
    ok, n_pairs, n_pos, n_out = _plan(_lib(), P)[0][:4]
    assert ok
    order, npp = P.order, (P.order + 1) // 2
    LT, want_cta, want_lane = {"auto": (0, -1, -1), "nbody": (lanes_per_warp, 0, 0), "nbody-cta": (lanes_per_warp, 1, 0),
                               "nbody-lane": (32, 0, 1)}[tape]
    cta = want_cta > 0 or (want_cta < 0 and n_pairs > 32)
    if not cta and n_pairs > 32:
        return None
    if LT == 0:
        LT = 1
        while not cta and 2 * LT * n_pairs <= 32:
            LT *= 2
    if (cta and (LT != 1 or n_pairs > 512)) or (not cta and (LT < 1 or LT > 32 or LT & (LT - 1) or LT * n_pairs > 32)):
        return None
    lane = want_lane != 0 and not cta and LT == 32 and n_pairs == 1 and order >= 4
    if want_lane > 0 and not lane:
        return None
    TT, NL = (512 if cta else 32), (2 if LT >= 2 else 1)
    n_rounds, n_records, n_consts, fac_stride = _roles(P, TT, LT, NL)
    assert n_out * LT < 0xffff and n_rounds <= 32
    if lane:
        n_records = 0
    copies = 8 if LT <= 2 else (2 if LT <= 8 else 1)  # nb_norm_copies()

    def shared_doubles(ris):
        return (order + 1) * fac_stride + ((order + 5) & ~1) + ((n_consts + 1) & ~1) + (n_records * 4 if ris else 0)

    def team_slots(off):
        d = (0 if lane else (n_pos + n_out) * LT * 2) + (2 if off else 5) * npp * TT * 2 + (3 * copies + 16) * LT
        return (d + LT - 1) // LT

    def fit(off):
        warps, ris_pick = 0, False
        for ris in (True, False):
            sh, tb = shared_doubles(ris) * 8, _coop_warp_bytes(team_slots(off), LT)
            if sh + tb + RESERVE > SMEM_OPTIN:
                continue
            w = 16 if cta else min((SMEM_OPTIN - RESERVE - sh) // tb, 16)
            if w > warps:
                warps, ris_pick = w, ris
            if w:
                break
        return warps, ris_pick

    off = False
    warps, ris = fit(False)
    if cta and warps == 0:
        off = True
        warps, ris = fit(True)
    if warps == 0:
        return None
    threads = block_threads or 32 * (warps if cta else min(warps, 12))
    if not cta:
        threads = min(threads, 32 * warps)
    assert threads % 32 == 0 and (not cta or threads == 512)
    maxt = 512 if cta else (256 if threads <= 256 else (384 if threads <= 384 else 512))
    teams = 1 if cta else threads // 32
    return dict(tape="nbody-lane" if lane else ("nbody-cta" if cta else "nbody"), lanes_per_warp=LT,
                block_threads=threads,
                smem_bytes=shared_doubles(ris) * 8 + teams * _coop_warp_bytes(team_slots(off), LT),
                grid=max(1, min(n_sms, -(-batch // (LT * teams)))), variant=(LT, cta, off, maxt, lane),
                roles_in_smem=ris)


def _cta_orders(name):
    """(the highest order at which a 512-thread CTA keeps all five private rows on chip, the lowest order at which
    it reads the role table from global memory, or None) for system `name`, from nb_expected()."""
    es = {o: nb_expected(nb_order_program(name, o), 1, "nbody-cta") for o in range(2, 72)}
    on_chip = [o for o, e in es.items() if e is not None and not e["variant"][2]]
    roles_g = [o for o, e in es.items() if e is not None and not e["roles_in_smem"]]
    return max(on_chip), (min(roles_g) if roles_g else None)


# ---- the matrix ----------------------------------------------------------------------------------------------------

def _legal_lts(n_pairs):
    return [lt for lt in (1, 2, 4, 8, 16, 32) if lt * n_pairs <= 32]


def requests(name, order):
    """The kernel requests tried for a system at an order: every legal lanes_per_warp with the default CTA size and with
    384 and 512 threads (clamped by setup_nb() to the warps that fit: at high orders the same kernel as the default),
    CTA teams, one thread per lane; and requests that must be refused: a lanes_per_warp that is not a power of two, or
    whose pair threads do not fit in a warp. nb_expected() tells which is which (CTA teams do not fit at high orders,
    one thread per lane needs one pair interaction and order >= 4)."""
    lts = _legal_lts(NB_SYSTEMS[name][2])
    out = [dict(tape="nbody", lanes_per_warp=lt, block_threads=bt) for lt in lts for bt in (0, 384, 512)]
    out += [dict(tape="nbody-cta")] + [dict(tape="nbody-lane", block_threads=bt) for bt in (0, 384, 512)]
    out += [dict(tape="nbody", lanes_per_warp=3), dict(tape="nbody", lanes_per_warp=2 * lts[-1]) if lts and lts[-1] < 32
            else dict(tape="nbody")]
    return out


# (system, order): the default order everywhere; odd orders 15 and 5; 5 is also the low order where warp teams of 512
# threads fit and CTA rows stay on chip; high orders 25, 36 (fewer warps fit) and 71 (quotients by n > 64 take the true
# division); the two-body boundary of k_nb1 at 3 / 4. The CTA thresholds are added in CASES below.
_BASE_CASES = [("nbody3_m1", 20), ("nbody3_m1", 5), ("nbody3_m1", 15), ("nbody3", 20), ("nbody3", 15), ("nbody3", 36),
               ("nbody3", 71), ("nbody4", 20), ("nbody4", 5), ("nbody4_m0102", 20), ("nbody5_m1_01", 20),
               ("nbody5_m1_01", 15), ("nbody5", 20), ("nbody5", 25), ("nbody8", 20), ("nbody8", 5), ("nbody9", 20),
               ("nbody9", 5), ("nbody12", 20), ("two_body_m10", 20), ("two_body_m10", 5), ("two_body_m10", 3),
               ("two_body_m10", 4), ("two_body_m10", 71), ("two_body_m104", 20), ("two_body_m104", 4),
               ("two_body_m104", 36)]


def _cases():
    cases = list(_BASE_CASES)
    for name in ("nbody9", "nbody12"):
        hi_on, lo_roles_g = _cta_orders(name)
        cases += [(name, hi_on), (name, hi_on + 1)]
        if lo_roles_g is not None:
            cases.append((name, lo_roles_g))
    return sorted(set(cases), key=cases.index)


CASES = _cases()
BATCH = 37  # > 32 and odd: every team shape has a partial last team, and several teams claim chunks


def test_every_instantiation_is_launched():
    """(No GPU needed.) The cases of this file launch every compiled N-body variant: nb_expected() of every shape of
    every case, which the GPU tests check against kernel_info()."""
    seen = set()
    for name, order in CASES:
        P = nb_order_program(name, order)
        assert nb_expected(P, BATCH) is not None, (name, order)
        for kw in [dict(tape="auto")] + requests(name, order):
            e = nb_expected(P, BATCH, **kw)
            if e is not None:
                seen.add(e["variant"])
    assert seen == COMPILED, sorted(COMPILED - seen)
    # The CTA cases cover both storage policies and the role table in global memory.
    for name in ("nbody9", "nbody12"):
        hi_on, _ = _cta_orders(name)
        a = nb_expected(nb_order_program(name, hi_on), BATCH, "nbody-cta")
        b = nb_expected(nb_order_program(name, hi_on + 1), BATCH, "nbody-cta")
        assert not a["variant"][2] and b["variant"][2] and a["smem_bytes"] != b["smem_bytes"]
    assert any(not nb_expected(nb_order_program(n, o), BATCH, "nbody-cta")["roles_in_smem"] for n, o in CASES
               if NB_SYSTEMS[n][2] > 32)


# ---- running one shape ---------------------------------------------------------------------------------------------

def _ki_check(ta, P, batch, kw):
    e = nb_expected(P, batch, **kw)
    ki = ta._b.kernel_info()
    got = {k: ki[k] for k in ("tape", "lanes_per_warp", "block_threads", "smem_bytes", "grid")}
    assert got == {k: e[k] for k in got}, (kw, got, e)
    return e, ki


def _snap(ta, tc=True):
    return dict(state=ta.state.copy(), t_hi=ta.dtime[0].copy(), t_lo=ta.dtime[1].copy(), last_h=ta.last_h.copy(),
                tc=ta.tc.copy() if tc else None)


def _reset(ta, st, t0=0.):
    ta.state[:] = st
    ta.set_time(t0)


def _run(name, order, st, kw, lim_f, lim_b, tf, mdt_prop):
    """The sequence every shape runs: a free step with write_tc, a clamped step forward and one backward (each from the
    initial state), propagate_until() to per-lane final times with write_tc, and the same with every step clamped."""
    P = nb_order_program(name, order)
    batch = st.shape[1]
    ta = hb.taylor_adaptive_batch(nb_system(name), st, batch, tol=nb_order_tol(order), kernel=kw)
    e, _ = _ki_check(ta, P, batch, kw)
    out = {"variant": e["variant"]}
    ta.step(write_tc=True)
    out["step"] = _snap(ta) | {"res": list(ta.step_res)}
    for key, lim in (("fwd", lim_f), ("bwd", lim_b)):
        _reset(ta, st)
        ta.step(lim, write_tc=True)
        out[key] = _snap(ta) | {"res": list(ta.step_res)}
    _reset(ta, st)
    ta.propagate_until(tf, write_tc=True)
    out["prop"] = _snap(ta) | {"res": list(ta.propagate_res)}
    _reset(ta, st)
    ta.propagate_until(tf, max_delta_t=mdt_prop)
    out["prop_clamped"] = _snap(ta, tc=False) | {"res": list(ta.propagate_res)}
    return out


def _equal(a, b):
    if isinstance(a, np.ndarray):
        return np.array_equal(a, b)
    return a == b


def _assert_same(ref, got, what):
    for phase in ("step", "fwd", "bwd", "prop", "prop_clamped"):
        for k, v in ref[phase].items():
            if v is not None:
                assert _equal(v, got[phase][k]), (what, phase, k)


def _ulps(a, b):
    return np.max(np.abs(a - b) / np.spacing(np.abs(b)))


@pytest.mark.gpu
@pytest.mark.parametrize("name,order", CASES, ids=["%s@%d" % c for c in CASES])
def test_shapes_match_oracle_bit_for_bit(name, order):
    """The automatic shape against the oracle, then every forced shape against the automatic one, bit for bit."""
    P = nb_order_program(name, order)
    st = nb_lane_states(name, BATCH, seed=order)
    o = oracle.OracleIntegrator(P, st, BATCH, mode=oracle.FMA)
    o.step(write_tc=True)
    h_nat = o.last_h.copy()
    ob = oracle.OracleIntegrator(P, st, BATCH, mode=oracle.FMA)
    ob.step(backward=True)
    lim_f, lim_b = 0.5 * h_nat, 0.5 * ob.last_h
    tf = np.linspace(2., 6., BATCH) * np.abs(h_nat)  # 2-6 first steps: most lanes finish before the slowest
    op = oracle.OracleIntegrator(P, st, BATCH, mode=oracle.FMA)
    op.propagate_until(tf, write_tc=True)
    # Clamped propagation: half the smallest free step of each lane (min_h: its successful steps; a lane whose only
    # step reached tf has none).
    mdt_prop = 0.5 * np.where(np.isfinite(op.min_h), op.min_h, np.abs(h_nat))

    ref = _run(name, order, st, dict(tape="auto"), lim_f, lim_b, tf, mdt_prop)

    # 1. One free step with write_tc: the coefficients and outcomes exactly; the step size within 4 ulps (it is a pow()
    # of the norms: libdevice's is within 2 ulps, glibc's within 1, then one rounded product); the state moves by |x'|
    # times that difference (< 1e-14 of its size).
    s = ref["step"]
    assert np.array_equal(s["tc"], o.tc)
    assert [r[0] for r in s["res"]] == [int(x) for x in o.step_outcome]
    assert _ulps(s["last_h"], o.last_h) <= 4.
    assert lane_err(s["state"], o.state) < 1e-14

    # 2. Clamped steps, forward and backward: state, double-length time, step size and coefficients exactly.
    for key, lim in (("fwd", lim_f), ("bwd", lim_b)):
        oc = oracle.OracleIntegrator(P, st, BATCH, mode=oracle.FMA)
        oc.step(lim, write_tc=True)
        g = ref[key]
        assert np.array_equal(g["last_h"], lim) and np.array_equal(oc.last_h, lim), key
        for k, v in (("state", oc.state), ("t_hi", oc.t_hi), ("t_lo", oc.t_lo), ("tc", oc.tc)):
            assert np.array_equal(g[k], v), (key, k)
        assert [r[0] for r in g["res"]] == [int(x) for x in oc.step_outcome] == [hb.taylor_outcome.time_limit] * BATCH

    # 5. propagate_until() to per-lane final times (lock-step: lanes that finish early take zero-length steps): identical
    # step counts and outcomes, final states to 1e-12 (a dozen steps of 1-2 ulp differences in h), the zero pattern of
    # last_h, the coefficients re-expanded about the final state (weighted by the last step, or the smallest one of
    # the lane if it finished early, as in test_gpu_parity.py).
    g = ref["prop"]
    assert [r[3] for r in g["res"]] == [int(x) for x in op.n_steps]
    assert [r[0] for r in g["res"]] == [int(x) for x in op.prop_outcome] == [hb.taylor_outcome.time_limit] * BATCH
    assert np.count_nonzero(op.last_h == 0.) >= BATCH // 2
    assert np.array_equal(g["t_hi"], tf) and np.array_equal(g["last_h"] == 0., op.last_h == 0.)
    assert lane_err(g["state"], op.state) < 1e-12
    assert tc_err(g["tc"], op.tc, np.where(op.last_h != 0., np.abs(op.last_h), 2. * mdt_prop)) < 1e-11
    # ... and with every step clamped: the whole propagation exactly. (max_h counts the successful steps, those whose
    # size the clamp did not set: none, so no step size went through pow().)
    op = oracle.OracleIntegrator(P, st, BATCH, mode=oracle.FMA)
    op.propagate_until(tf, max_delta_t=mdt_prop)
    assert np.all(op.max_h == 0.)
    g = ref["prop_clamped"]
    for k, v in (("state", op.state), ("t_hi", op.t_hi), ("t_lo", op.t_lo), ("last_h", op.last_h)):
        assert np.array_equal(g[k], v), k
    assert [r[0] for r in g["res"]] == [int(x) for x in op.prop_outcome]
    assert [r[3] for r in g["res"]] == [int(x) for x in op.n_steps]
    assert np.array_equal([r[1] for r in g["res"]], op.min_h) and np.array_equal([r[2] for r in g["res"]], op.max_h)

    # 3. Every forced shape: the same bits as the automatic one, everywhere; a shape that cannot run is refused with
    # the documented error.
    for kw in requests(name, order):
        if nb_expected(P, BATCH, **kw) is not None:
            _assert_same(ref, _run(name, order, st, kw, lim_f, lim_b, tf, mdt_prop), kw)
        else:
            ta = hb.taylor_adaptive_batch(nb_system(name), st, BATCH, tol=nb_order_tol(order))
            with pytest.raises(ValueError, match="The N-body kernel cannot run this program"):
                ta._b.set_kernel(**kw)


# ---- batch tails and persistence -----------------------------------------------------------------------------------

# (system, order, kernel): one case per team width, plus CTA teams and the one-thread-per-lane kernel.
TAIL_CASES = [("nbody3_m1", 20, dict(tape="auto")), ("nbody3", 20, dict(tape="auto")), ("nbody4", 5, dict(tape="auto")),
              ("nbody5", 20, dict(tape="auto")), ("nbody8", 20, dict(tape="auto")), ("nbody9", 20, dict(tape="auto")),
              ("two_body_m10", 20, dict(tape="auto")), ("two_body_m104", 20, dict(tape="nbody"))]
N_BASE = 7  # base lanes, tiled: lane i of a batch starts like base lane i % 7 (7 is odd: neighbours always differ)


@pytest.mark.gpu
@pytest.mark.parametrize("name,order,kw", TAIL_CASES, ids=["%s@%d-%s" % (n, o, k["tape"]) for n, o, k in TAIL_CASES])
def test_batch_tails_and_persistence(name, order, kw):
    """Batch sizes 1, LT - 1, k LT + 1 and one larger than grid x teams x LT (every team claims more than one chunk):
    every lane gives the bits of the same lane run alone in a batch of 1 (a step with write_tc, a clamped step, and
    propagate_until(): state, time and its results)."""
    P = nb_order_program(name, order)
    base = nb_lane_states(name, N_BASE, seed=100 + order)
    tol = nb_order_tol(order)
    o = oracle.OracleIntegrator(P, base, N_BASE, mode=oracle.FMA)
    o.step()
    h_nat = np.abs(o.last_h)
    tf_base = np.linspace(3., 9., N_BASE) * h_nat
    lim_base = -0.5 * h_nat

    def run(batch):
        idx = np.arange(batch) % N_BASE
        st = base[:, idx]
        ta = hb.taylor_adaptive_batch(nb_system(name), st, batch, tol=tol, kernel=kw)
        e, ki = _ki_check(ta, P, batch, kw)
        r = {"ki": ki, "LT": e["lanes_per_warp"]}
        ta.step(write_tc=True)
        r["step"] = _snap(ta) | {"res": list(ta.step_res)}
        _reset(ta, st)
        ta.step(lim_base[idx])
        r["lim"] = _snap(ta, tc=False) | {"res": list(ta.step_res)}
        _reset(ta, st)
        ta.propagate_until(tf_base[idx])
        r["prop"] = _snap(ta, tc=False) | {"res": list(ta.propagate_res)}
        return r

    alone = [None] * N_BASE
    for i in range(N_BASE):
        ta = hb.taylor_adaptive_batch(nb_system(name), base[:, i:i + 1], 1, tol=tol, kernel=kw)
        ta.step(write_tc=True)
        s = _snap(ta) | {"res": list(ta.step_res)}
        _reset(ta, base[:, i:i + 1])
        ta.step(lim_base[i:i + 1])
        lm = _snap(ta, tc=False) | {"res": list(ta.step_res)}
        _reset(ta, base[:, i:i + 1])
        ta.propagate_until(tf_base[i:i + 1])
        alone[i] = (s, lm, _snap(ta, tc=False) | {"res": list(ta.propagate_res)})
    first = run(N_BASE)
    LT, ki = first["LT"], first["ki"]
    teams = 1 if ki["tape"] == "nbody-cta" else ki["block_threads"] // 32
    big = ki["n_sms"] * teams * LT * 2 + 3
    sizes = sorted({1, max(LT - 1, 1), 3 * LT + 1, big})
    for batch in sizes:
        r = run(batch)
        assert batch != big or batch > r["ki"]["grid"] * teams * LT
        idx = np.arange(batch) % N_BASE
        for p, phase in enumerate(("step", "lim", "prop")):
            ref = [alone[i][p] for i in range(N_BASE)]
            g = r[phase]
            for k in ("state", "t_hi", "t_lo", "tc", "last_h"):
                # (After propagate_until() a lane that finished before the slowest one of its batch has last_h = 0.)
                if ref[0][k] is not None and not (phase == "prop" and k == "last_h"):
                    exp = np.stack([a[k][..., 0] for a in ref], axis=-1)[..., idx]
                    assert np.array_equal(g[k], exp), (batch, phase, k, np.argwhere(g[k] != exp)[:4])
            assert g["res"] == [ref[i]["res"][0] for i in idx], (batch, phase)


# ---- non-finite and limit exits in a partial last team -------------------------------------------------------------

EXIT_CASES = [("nbody3_m1", 20), ("nbody3", 20), ("nbody4", 20), ("nbody9", 20)]  # LT 16, 8, 4, CTA


@pytest.mark.gpu
@pytest.mark.parametrize("name,order", EXIT_CASES, ids=["%s@%d" % c for c in EXIT_CASES])
def test_exits_in_partial_last_team(name, order):
    """A lane whose bodies 0 and 1 collide (r = 0: a non-finite jet), placed in the partial last team and not its first
    lane: step() fails that lane only and leaves the others' bits as without it; propagate_until() with max_steps and
    with the colliding lane follows the oracle's lock-step semantics (test_gpu_parity.py's
    test_global_exits_match_reference_semantics)."""
    P = nb_order_program(name, order)
    e = nb_expected(P, 1)
    LT = e["lanes_per_warp"]
    batch = 2 * LT + 3 if LT >= 4 else 7
    bad = batch - 2  # in the last (partial) team, not its lane 0
    assert LT == 1 or bad % LT != 0
    st = nb_lane_states(name, batch, seed=5)
    st2 = st.copy()
    st2[6:9, bad] = st2[0:3, bad]
    sys_, tol = nb_system(name), nb_order_tol(order)

    clean = hb.taylor_adaptive_batch(sys_, st, batch, tol=tol)
    clean.step()
    ta = hb.taylor_adaptive_batch(sys_, st2, batch, tol=tol)
    _ki_check(ta, P, batch, dict(tape="auto"))
    ta.step()
    assert [r[0] for r in ta.step_res] == [NF if i == bad else r[0] for i, r in enumerate(clean.step_res)]
    ok = np.arange(batch) != bad
    assert np.array_equal(ta.state[:, ok], clean.state[:, ok]) and np.array_equal(ta.last_h[ok], clean.last_h[ok])

    o = oracle.OracleIntegrator(P, st, batch, mode=oracle.FMA)
    o.step()
    tf = np.linspace(3., 40., batch) * np.abs(o.last_h)
    # Iteration limit: every outcome becomes step_limit, step counts and times as in the lock-step loop.
    o = oracle.OracleIntegrator(P, st, batch, mode=oracle.FMA)
    ta = hb.taylor_adaptive_batch(sys_, st, batch, tol=tol)
    o.propagate_until(tf, max_steps=7)
    ta.propagate_until(tf, max_steps=7)
    assert [r[0] for r in ta.propagate_res] == [hb.taylor_outcome.step_limit] * batch
    assert [r[3] for r in ta.propagate_res] == [int(x) for x in o.n_steps]
    # (Times and states after 7 steps of 1-2 ulp step-size differences: 1e-13 / 1e-12, as in test_gpu_parity.py.)
    assert np.max(np.abs(ta.time - o.t_hi) / np.abs(o.t_hi)) < 1e-13 and lane_err(ta.state, o.state) < 1e-12
    # A non-finite lane stops every lane at that iteration.
    o = oracle.OracleIntegrator(P, st2, batch, mode=oracle.FMA)
    ta = hb.taylor_adaptive_batch(sys_, st2, batch, tol=tol)
    o.propagate_until(tf)
    ta.propagate_until(tf)
    assert int(o.prop_outcome[bad]) == NF
    assert [r[0] for r in ta.propagate_res] == [int(x) for x in o.prop_outcome]
    assert [r[3] for r in ta.propagate_res] == [int(x) for x in o.n_steps]
    assert lane_err(ta.state[:, ok], o.state[:, ok]) < 1e-12
    assert np.max(np.abs(ta.time[ok] - o.t_hi[ok]) / np.abs(o.t_hi[ok])) < 1e-13


# ---- propagate_grid ------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("name", ["nbody3", "nbody9"])  # LT 8, CTA
def test_propagate_grid_partial_teams(name):
    """propagate_grid() (the skip-masked steps of the host loop, src/taylor_adaptive_batch.cpp:1545-2055) with partial
    teams, against the oracle: max_delta_t, max_steps and free steps (test_gpu_parity.py's
    test_propagate_grid_limits_match_oracle). Values to 1e-12 of the largest (dense output after a few steps of
    1-2 ulp step-size differences), outcomes and step counts exactly."""
    P = nb_order_program(name, 20)
    batch = 11
    st = nb_lane_states(name, batch, seed=9)
    o = oracle.OracleIntegrator(P, st, batch, mode=oracle.FMA)
    o.step()
    h = np.abs(o.last_h)
    grid = np.linspace(0., 6., 25)[:, None] * h[None, :]
    for kw in (dict(max_delta_t=0.4 * h), dict(max_steps=3), dict()):
        ta = hb.taylor_adaptive_batch(nb_system(name), st, batch)
        assert ta._b.kernel_info()["tape"] == nb_expected(P, batch)["tape"]
        o = oracle.OracleIntegrator(P, st, batch, mode=oracle.FMA)
        ret = ta.propagate_grid(grid, **kw)
        oret = o.propagate_grid(grid, **kw)
        assert np.array_equal(np.isnan(ret), np.isnan(oret)), kw
        m = ~np.isnan(oret)
        assert np.max(np.abs(ret[m] - oret[m])) < 1e-12 * np.max(np.abs(oret[m])), kw
        assert [r[0] for r in ta.propagate_res] == [int(x) for x in o.prop_outcome], kw
        assert [r[3] for r in ta.propagate_res] == [int(x) for x in o.n_steps], kw
        if "max_steps" in kw:  # (stopped after 3 free steps: 1-2 ulp step-size differences)
            assert np.max(np.abs(ta.time - o.t_hi) / np.abs(o.t_hi)) < 1e-13, kw
        else:
            assert np.array_equal(ta.time, o.t_hi), kw
