"""The N-body kernel's host logic, without a GPU: the planner (heyoka_b200/csrc/nb_plan.cpp) and the two-orders-at-a-time
arithmetic of heyoka_b200/csrc/nb_core.hpp, emulated on plain arrays (tests/cpp/nb_emul.cpp) and compared against the
oracle's one-order-at-a-time jet. The same nb_core.hpp is what k_nb (nb_kernel.cuh) runs on the device."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import heyoka_b200 as hb
import oracle
from common import (nbody32_batch_state, outer_ss_batch_state, sys_ffnn, sys_nbody32, sys_outer_ss, sys_pendulum,
                    sys_two_body, sys_two_body_symmetric, two_body_batch_state)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "heyoka_b200", "csrc")
LIBDIR = os.path.join(ROOT, "heyoka_b200", "lib")
SO = os.path.join(ROOT, "build", "libnb_emul.so")


def _emul():
    src = os.path.join(ROOT, "tests", "cpp", "nb_emul.cpp")
    deps = [src, os.path.join(CSRC, "nb_core.hpp"), os.path.join(CSRC, "nb_plan.hpp"), os.path.join(CSRC, "nb_desc.hpp"),
            os.path.join(CSRC, "nb_plan.cpp"), os.path.join(CSRC, "smem_plan.hpp"), os.path.join(CSRC, "smem_plan.cpp"),
            os.path.join(LIBDIR, "libheyoka_b200.so")]
    os.makedirs(os.path.dirname(SO), exist_ok=True)
    if not os.path.exists(SO) or os.path.getmtime(SO) < max(os.path.getmtime(d) for d in deps):
        # -ffp-contract=off: the only fused operations are the explicit fma() calls, like -fmad=false on the device.
        subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-shared", "-fPIC", "-I" + os.path.join(ROOT, "include"),
                        "-I" + CSRC, src, "-o", SO, "-L" + LIBDIR, "-lheyoka_b200", "-Wl,-rpath," + LIBDIR], check=True)
    lib = C.CDLL(SO)
    lib.nb_emul_plan.restype = C.c_int
    lib.nb_emul_jet.restype = C.c_int
    return lib


def _plan(lib, P):
    out = (C.c_uint32 * 6)()
    why = C.create_string_buffer(256)
    lib.nb_emul_plan(P._h, out, why, C.c_size_t(256))
    return list(out), why.value.decode()


def _emul_jet(lib, P, state_lanes, n_pairs, tt, lt):
    """Jets of `lt` lanes run by one emulated team of `tt` threads. state_lanes: [n_eq, lt]."""
    n_ord = 2 * ((P.order + 1) // 2)
    coef = np.zeros((lt, P.n_eq, P.order + 1))
    u_idx = np.zeros(n_pairs * 8, dtype=np.uint32)
    u_rows = np.zeros((n_pairs, lt, 8, n_ord))
    st = np.ascontiguousarray(state_lanes, dtype=np.float64)
    assert st.shape == (P.n_eq, lt)
    rc = lib.nb_emul_jet(P._h, C.c_uint32(tt), C.c_uint32(lt), st.ctypes.data_as(C.POINTER(C.c_double)),
                         coef.ctypes.data_as(C.POINTER(C.c_double)), u_idx.ctypes.data_as(C.POINTER(C.c_uint32)),
                         u_rows.ctypes.data_as(C.POINTER(C.c_double)))
    assert rc == 0, rc
    return coef, u_idx, u_rows


def test_plan_shapes():
    lib = _emul()
    # 6 bodies: 15 pair interactions, 18 positions, 45 products, 18 sums of 5 terms in one level.
    info, why = _plan(lib, hb.Program(sys_outer_ss(), high_accuracy=True))
    assert info == [1, 15, 18, 90, 18, 1], (info, why)  # outputs: m_k and the rescaled n_k of every pair
    # Two bodies, one of them massless: one pair interaction, the accelerations of the massive body are the number 0.
    info, why = _plan(lib, hb.Program(sys_two_body()))
    assert info == [1, 1, 6, 3, 6, 1], (info, why)
    # 32 bodies: 496 pair interactions; 31-term sums are nested (4 partial sums + 1 per acceleration).
    info, why = _plan(lib, hb.Program(sys_nbody32()))
    assert info[:4] == [1, 496, 96, 496 * 6 + 96 * 4] and info[4] == 96 * 5 and info[5] == 2, (info, why)
    # Programs that are not N-body-shaped are refused (they run on the generic cooperative kernel).
    for s in (sys_pendulum(), sys_ffnn(), sys_two_body_symmetric()):
        info, why = _plan(lib, hb.Program(s))
        assert info[0] == 0 and why != "", (info, why)


# ---- the systems x orders x team shapes that tests/test_gpu_nbody_shapes.py runs on the device ----
# name -> (bodies, masses, pair interactions). The comments give the automatic shape of the device kernel. (Planets of
# unequal masses: with unit masses the right-hand side simplifies to negations the planner does not take for pair
# outputs, and the program runs on the generic kernel instead.)
_PLANETS = [1.] + [1e-3 * (b + 1) for b in range(1, 12)]
NB_SYSTEMS = {
    "nbody3_m1": (3, [1.], 2),                  # LT 16: one massive body, the massless-massless pair is dropped
    "nbody3": (3, [1., 0.5, 0.2], 3),           # LT 8
    "nbody4": (4, _PLANETS[:4], 6),            # LT 4
    "nbody4_m0102": (4, [0., 1., 0., 2.], 5),   # LT 4, massless bodies first
    "nbody5_m1_01": (5, [1., 0.1], 7),          # LT 4, three massless bodies at the end
    "nbody5": (5, _PLANETS[:5], 10),           # LT 2
    "nbody8": (8, _PLANETS[:8], 28),           # LT 1, 4 idle threads per warp
    "nbody9": (9, _PLANETS[:9], 36),           # CTA teams: the first count above a warp
    "nbody12": (12, _PLANETS[:12], 66),        # CTA teams, two summation levels
    "two_body_m10": (2, [1., 0.], 1),           # k_nb1: the second body's accelerations are the number 0
    "two_body_m104": (2, [1., 0.4], 1),         # k_nb1: both bodies pull (rescaled pair outputs)
}


def nb_order_tol(order):
    """The tolerance of a given Taylor order: 0 (the default, order 20) for order 20, else exp(-2 (order - 1))
    (order = ceil(1 - ln(tol) / 2), src/taylor_00.cpp), nudged up by 0.1 % so that the rounding of the logarithm cannot
    change the order."""
    return 0. if order == 20 else float(np.exp(-2. * (order - 1)) * 1.001)


def nb_system(name):
    n, masses, _ = NB_SYSTEMS[name]
    return hb.model.nbody(n, masses=masses)


def nb_order_program(name, order):
    """The program of system `name` at the given Taylor order."""
    tol = nb_order_tol(order)
    P = hb.Program(nb_system(name)) if tol == 0. else hb.Program(nb_system(name), tol=tol)
    assert P.order == order, (name, order, P.order)
    return P


def nb_lane_states(name, batch, seed=0):
    """[6 n, batch] states of system `name` whose lanes differ by O(1): body b (b >= 1) on a near-circular orbit of
    radius 1.5 b + U(0, 0.5) with a random phase per lane and body, speeds 0.97-1.03 times the circular one about the
    mass inside it, small inclinations; body 0 near the origin. Bodies of a lane start at least 1 apart, so that no
    close approach shrinks the steps of a short propagation. A lane mix-up in a kernel then moves its results by O(1), not by a perturbation."""
    n, masses, _ = NB_SYSTEMS[name]
    masses = list(masses) + [0.] * (n - len(masses))
    rng = np.random.default_rng(seed)
    st = np.zeros((6 * n, batch))
    st[0:3] = 0.05 * rng.uniform(-1., 1., (3, batch))
    st[3:6] = 0.05 * rng.uniform(-1., 1., (3, batch))
    for b in range(1, n):
        r = 1.5 * b + rng.uniform(0., 0.5, batch)
        ph = rng.uniform(0., 2. * np.pi, batch)
        v = np.sqrt(max(sum(masses[:b]), 0.5) / r) * rng.uniform(0.97, 1.03, batch)
        st[6 * b + 0], st[6 * b + 1], st[6 * b + 2] = r * np.cos(ph), r * np.sin(ph), rng.uniform(-0.1, 0.1, batch)
        st[6 * b + 3], st[6 * b + 4], st[6 * b + 5] = -v * np.sin(ph), v * np.cos(ph), rng.uniform(-0.05, 0.05, batch)
    return st


def nb_team_shapes(n_pairs):
    """(threads per team, lanes per team) of every team shape the device kernel has: a warp with each power-of-two
    number of lanes whose pairs fit in its 32 threads, and a CTA of 512 threads with one lane."""
    return [(32, lt) for lt in (1, 2, 4, 8, 16, 32) if lt * n_pairs <= 32] + [(512, 1)]


NB_ORDERS = (20, 15, 5, 25)                   # default, odd, low (warp teams of 512 threads, CTA rows on chip), high
NB_ORDERS_EXTRA = {"nbody3": (36, 71), "two_body_m10": (2, 3, 4, 71), "two_body_m104": (3, 4, 36)}


def _sweep_cases():
    out = []
    for name, (_, _, n_pairs) in NB_SYSTEMS.items():
        for order in NB_ORDERS + NB_ORDERS_EXTRA.get(name, ()):
            out += [("%s@%d" % (name, order), tt, lt) for tt, lt in nb_team_shapes(n_pairs)]
    return out


@pytest.mark.parametrize("name,tt,lt", [("outer_ss", 32, 2), ("outer_ss", 32, 1), ("two_body", 32, 32), ("two_body", 32, 4),
                                        ("nbody32", 512, 1), ("outer_ss_odd_order", 32, 2)] + _sweep_cases())
def test_two_order_blocks_match_oracle(name, tt, lt):
    """Every coefficient the blocked evaluation produces (coordinate differences, r^2, r^alpha, products, state
    variables) equals the oracle's sequential+FMA jet bit for bit, for the team shapes the kernel uses (threads per
    team, lanes per team): the pair threads, the output-slot layout and the per-thread role table of the sums.
    "system@order": the systems and orders of tests/test_gpu_nbody_shapes.py, so that a failure there can be put on the
    device code."""
    lib = _emul()
    if "@" in name:
        sys_name, order = name.split("@")
        P = nb_order_program(sys_name, int(order))
        st = nb_lane_states(sys_name, lt, seed=lt)
    elif name == "outer_ss":
        P, st = hb.Program(sys_outer_ss(), high_accuracy=True), outer_ss_batch_state(lt)
    elif name == "outer_ss_odd_order":
        P, st = hb.Program(sys_outer_ss(), tol=1e-12), outer_ss_batch_state(lt)
        assert P.order % 2 == 1
    elif name == "two_body":
        P, st = hb.Program(sys_two_body()), two_body_batch_state(lt)
    else:
        P, st = hb.Program(sys_nbody32()), nbody32_batch_state(lt)
    info, why = _plan(lib, P)
    assert info[0] == 1, why
    if "@" in name:
        assert info[1] == NB_SYSTEMS[sys_name][2], info
    coef, u_idx, u_rows = _emul_jet(lib, P, st, info[1], tt, lt)
    for lane in range(lt):
        tape = oracle.jet(P, st, lane=lane, mode=oracle.FMA)  # [order + 1, n_uvars]; u variables: orders < order
        assert np.array_equal(coef[lane], tape[:, :P.n_eq].T), np.max(np.abs(coef[lane] - tape[:, :P.n_eq].T))
        ref = tape[:P.order, u_idx].T.reshape(info[1], 8, P.order)
        got = u_rows[:, lane, :, :P.order]
        assert np.array_equal(got, ref), np.argwhere(got != ref)[:5]
