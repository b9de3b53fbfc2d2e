"""Kernel selection (hy_batch::decide() and commit(), batch.cu): set_launch_config() keeps the selected tape, a refused
request leaves the batch exactly as it was, and batches that run the same kernel with different shared-memory sizes do
not limit one another (the dynamic shared-memory limit is an attribute of the kernel, shared by the whole process)."""
import functools

import numpy as np
import pytest

import heyoka_b200 as hb
from common import (FFNN_TOL, ffnn_batch_state, nbody32_batch_state, outer_ss_batch_state, sys_ffnn, sys_nbody32,
                    sys_outer_ss, sys_pendulum, sys_two_body, two_body_batch_state)
from test_gpu_coop_shapes import coop_expected
from test_nb_plan import nb_lane_states, nb_order_program, nb_order_tol

BATCH = 64

SYSTEMS = {
    "outer_ss": (sys_outer_ss, 0., outer_ss_batch_state),
    "pendulum": (sys_pendulum, 0., lambda n: np.random.default_rng(3).uniform(-1., 1., (2, n))),
    "two_body": (sys_two_body, 0., two_body_batch_state),
    "ffnn": (sys_ffnn, FFNN_TOL, ffnn_batch_state),
    "nbody32": (sys_nbody32, 0., nbody32_batch_state),
}


@functools.cache
def program(name):
    sys_, tol, _ = SYSTEMS[name]
    return hb.Program(sys_(), tol=tol) if tol else hb.Program(sys_())


def make(P, request=None, batch=BATCH):
    b = hb.Batch(P, batch)
    if request is not None:
        b.set_kernel(**request)
    return b


def run_step(b, st):
    """One step with write_tc from state st at t = 0: state, times, step size and Taylor coefficients."""
    n = st.shape[1]
    b.upload(st, None, np.zeros(n), np.zeros(n))
    b.step(write_tc=True)
    return b.download() + (b.tc(),)


def assert_same_bits(a, b, what):
    for k, (x, y) in enumerate(zip(a, b)):
        assert np.array_equal(x, y), (what, k)


# ---- set_launch_config() -------------------------------------------------------------------------------------------

# (system, set_kernel() request, block_threads given to set_launch_config()). nbody-cta runs CTAs of exactly 512
# threads; the network kernel has a fixed shape and ignores the CTA size.
LAUNCH_CASES = [("outer_ss", "hbm", 128), ("outer_ss", "smem", 64), ("outer_ss", "global", 256),
                ("outer_ss", "global-cta", 256), ("outer_ss", "nbody", 64), ("outer_ss", "nbody-cta", 512),
                ("two_body", "nbody-lane", 64), ("ffnn", "nn", 64)]


@pytest.mark.gpu
@pytest.mark.parametrize("name,tape,threads", LAUNCH_CASES, ids=["%s-%s" % (n, t) for n, t, _ in LAUNCH_CASES])
def test_set_launch_config_keeps_the_tape(name, tape, threads):
    """set_launch_config() re-runs the selected tape mode with its lanes and the new CTA size: the tape is unchanged,
    every kernel_info() field is that of a batch given the same request through set_kernel(), and a step gives that
    batch's bits."""
    P = program(name)
    st = SYSTEMS[name][2](BATCH)
    b = make(P, dict(tape=tape))
    assert b.kernel_info()["tape"] == tape
    b.set_launch_config(block_threads=threads)
    ki = b.kernel_info()
    assert ki["tape"] == tape
    if tape != "nn":
        assert ki["block_threads"] == threads
    twin = make(P, dict(tape=tape, lanes_per_warp=ki["lanes_per_warp"],
                        lanes_per_thread=0 if tape.startswith("nbody") else ki["lanes_per_thread"],
                        block_threads=threads))
    assert ki == twin.kernel_info()
    assert_same_bits(run_step(b, st), run_step(twin, st), tape)


# ---- refusals ------------------------------------------------------------------------------------------------------

# (system, request that selects the starting kernel (None: the automatic choice), its tape).
START_CASES = [("nbody32", None, "nbody-cta"), ("pendulum", dict(tape="global-cta"), "global-cta"),
               ("outer_ss", None, "nbody"), ("ffnn", None, "nn"), ("pendulum", dict(tape="smem"), "smem")]
N_BODY = {"outer_ss", "nbody32"}


def refused_requests(name, tape, batch):
    """(call, arguments, message) of requests the batch must refuse."""
    out = [("set_kernel", dict(tape="hbm", block_threads=48), "multiple of 32"),
           ("set_kernel", dict(tape="global", lanes_per_warp=16), r"\(global tape\)")]
    for kw in (dict(tape="smem"), dict(tape="smem", lanes_per_warp=32, lanes_per_thread=1, block_threads=512)):
        if coop_expected(program(name), batch, **kw) == ("refused", "does not fit in shared memory"):
            out.append(("set_kernel", kw, "does not fit in shared memory"))
            break
    if tape != "nn":
        out.append(("set_launch_config", dict(block_threads=48), "Invalid number of threads"))
    if name not in N_BODY:
        out.append(("set_kernel", dict(tape="nbody"), "The N-body kernel cannot run this program"))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name,request_,tape", START_CASES, ids=["%s-%s" % (n, t) for n, _, t in START_CASES])
def test_refusal_changes_nothing(name, request_, tape):
    """After each refused request, kernel_info() is what it was and a step gives the bits of an untouched twin."""
    P = program(name)
    batch = 32
    st = SYSTEMS[name][2](batch)
    b, twin = make(P, request_, batch), make(P, request_, batch)
    ki = b.kernel_info()
    assert ki["tape"] == tape and twin.kernel_info() == ki
    ref = run_step(twin, st)
    for call, kw, msg in refused_requests(name, tape, batch):
        with pytest.raises(ValueError, match=msg):
            getattr(b, call)(**kw)
        assert b.kernel_info() == ki, (call, kw)
        assert_same_bits(run_step(b, st), ref, (call, kw))


# ---- the shared-memory limit ---------------------------------------------------------------------------------------

def _pendulum(order):
    return hb.Program(sys_pendulum(), tol=nb_order_tol(order))


def _ffnn(order):
    return hb.Program(sys_ffnn(), tol=nb_order_tol(order))


# (kernel, (program, initial states) at the larger and at the smaller order, the request that forces one shape).
SMEM_CASES = [
    ("k_coop", lambda: (_pendulum(30), _pendulum(10)), SYSTEMS["pendulum"][2],
     dict(tape="smem", lanes_per_warp=4, lanes_per_thread=2, block_threads=128)),
    ("k_nb", lambda: (nb_order_program("nbody3", 25), nb_order_program("nbody3", 10)),
     lambda n: nb_lane_states("nbody3", n), dict(tape="nbody", lanes_per_warp=8, block_threads=128)),
    ("k_nn", lambda: (_ffnn(15), _ffnn(8)), ffnn_batch_state, dict(tape="nn")),
]


@pytest.mark.gpu
@pytest.mark.parametrize("kernel,programs,states,request_", SMEM_CASES, ids=[c[0] for c in SMEM_CASES])
def test_batches_do_not_share_a_shared_memory_limit(kernel, programs, states, request_):
    """The same compiled shape at two orders needs two shared-memory sizes: configuring the smaller batch after the
    larger one does not change what the larger one's launches may use."""
    P_big, P_small = programs()
    st = states(BATCH)
    big = make(P_big, request_)
    ref = run_step(big, st)
    small = make(P_small, request_)
    kb, ks = big.kernel_info(), small.kernel_info()
    shape = ("tape", "lanes_per_warp", "lanes_per_thread", "block_threads")
    assert {k: kb[k] for k in shape} == {k: ks[k] for k in shape}, (kb, ks)
    assert kb["smem_bytes"] > ks["smem_bytes"] > 0
    assert_same_bits(run_step(big, st), ref, kernel)
    run_step(small, st)
