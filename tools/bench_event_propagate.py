"""Lane-steps/s of propagate_until() on an integrator with events: the device loop (hy_batch_propagate_until_ev(), taken
when there is no step callback) against the front end's host lock-step loop (forced by a step callback that returns
True), for a pendulum with
  - "nt":  a non-terminal event at every zero of x: nearly every iteration calls back to the host;
  - "te":  a terminal event (with a callback that continues) at x = 1.2, which a few lanes reach once.
Prints one JSON line per (workload, lanes, path) with the iterations, the iterations that called back and the bytes
moved between host and device per iteration (counted from shapes, for both paths). The host loop at 2^20 lanes gets a shorter t_final
(--host-tf-big): its two Python loops over the lanes take seconds per iteration."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import heyoka_b200 as hb  # noqa: E402


def make(kind, n, calls):
    x, v = hb.make_vars("x", "v")
    sys = [(x, v), (v, -9.8 * hb.sin(x))]
    rng = np.random.default_rng(0)
    amp = 0.05 + 0.5 * rng.random(n)
    if kind == "te":
        amp[::4096] = 1.25  # a few lanes reach x = 1.2

    def ntcb(ta, t, d_sgn, i):
        calls[0] += 1

    def tcb(ta, d_sgn, i):
        calls[0] += 1
        return True
    ev = dict(nt_events=[hb.nt_event_batch(x, ntcb)]) if kind == "nt" else \
        dict(t_events=[hb.t_event_batch(x - 1.2, callback=tcb)])
    return hb.taylor_adaptive_batch(sys, np.vstack([amp, np.zeros(n)]), n, **ev)


def run(kind, n, host, tf):
    calls = [0]
    ta = make(kind, n, calls)
    cb_iters, n_recs = [0], [0]
    orig = ta._device_event_callbacks

    def counted(*a):
        cb_iters[0] += 1
        n_recs[0] += len(a[0])
        return orig(*a)
    ta._device_event_callbacks = counted
    iters = [0]

    def step_cb(ta):
        iters[0] += 1
        return True
    ta.propagate_until(0.01, **({"callback": step_cb} if host else {}))  # warm-up
    t0 = time.perf_counter()
    ta.propagate_until(tf, **({"callback": step_cb} if host else {}))
    dt = time.perf_counter() - t0
    steps = sum(r[3] for r in ta.propagate_res)
    P = ta._prog
    # Host loop, per iteration: state, pars, times up; state, times, last_h, tc, step results down.
    # Device loop: the detection counters (16 bytes) and the lock-step flags (16 bytes) of every iteration; per record,
    # the record read back (40 bytes), sent back for its absolute time (32) and the time read back (16); a terminal
    # record's lane whose callback continues (4, counted for every record: an upper bound). Iterations: the largest
    # step count of a lane (the loop ends with its last step).
    if host:
        per_iter = n * 8 * (2 * P.n_eq + P.n_pars + 2 + 3 + P.n_eq * (P.order + 1) + 2)
    else:
        dev_iters = max(1, max(r[3] for r in ta.propagate_res))
        per_iter = 32 + n_recs[0] * (40 + 32 + 16 + 4) / dev_iters
    return dict(workload=kind, lanes=n, path="host" if host else "device", t_final=tf, seconds=dt,
                lane_steps_per_s=steps / dt, lane_steps=int(steps), callback_calls=calls[0],
                host_loop_iterations=iters[0] if host else None,
                iterations_called_back=None if host else cb_iters[0], records=None if host else n_recs[0],
                bytes_per_iteration=per_iter)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lanes", default="4096,65536,1048576")
    ap.add_argument("--tf", type=float, default=2.0)
    ap.add_argument("--host-tf-big", type=float, default=0.3, help="t_final of the host loop at 2^20 lanes")
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    for kind in ("nt", "te"):
        for n in (int(s) for s in a.lanes.split(",")):
            for host in (False, True):
                tf = a.host_tf_big if host and n >= (1 << 20) else a.tf
                r = run(kind, n, host, tf)
                r["gpu"] = gpu
                print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
