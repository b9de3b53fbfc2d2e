#!/usr/bin/env python3
"""Informational timings of the other BASELINE.json configurations (they are parity-test cases, not bench lines):
lane-steps/s of one GPU, device-timed around the C-ABI calls with host buffers already uploaded.

    python tools/bench_configs.py [tb] [n32] [nn] [s6step]
"""
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import heyoka_b200 as hb  # noqa: E402
from common import (FFNN_TOL, ffnn_batch_state, nbody32_batch_state, outer_ss_batch_state, sys_ffnn, sys_nbody32,  # noqa: E402
                    sys_outer_ss, sys_two_body, two_body_batch_state)


def timed(fn, reps=3):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return min(ts)


def run(name, P, st, t_final=None, **kernel):
    batch = st.shape[1]
    b = hb.Batch(P, batch)
    if kernel:
        b.set_kernel(**kernel)
    z = np.zeros(batch)
    res = {"config": name, "lanes": batch, "kernel": b.kernel_info()["tape"], "costs": P.costs()}

    def step():
        b.upload(st, None, z, z)
        b.sync()
        t0 = time.perf_counter()
        if t_final is None:
            b.step()
        else:
            b.propagate_until(np.full(batch, t_final))
        b.sync()
        step.dt = time.perf_counter() - t0

    timed(step, reps=2)
    if t_final is None:
        n_steps = batch
    else:
        n_steps = int(b.prop_res()[3].sum())
    res.update(seconds=step.dt, lane_steps=n_steps, lane_steps_per_s=n_steps / step.dt,
               b_tape_gbs=n_steps * P.costs()["b_tape"] / step.dt / 1e9)
    print(json.dumps(res), flush=True)


def grid_sharded():
    """The "grid" workload (6-body, 16384 lanes x 1000 grid points over 20 yr, pinned output) on one device and on
    sharded batches (two shards on device 0, and one shard per GPU when the box has several), through the C ABI. Then
    the front end's host loop over the shards (forced by a step callback that returns True), on 2 yr and 100 grid points
    because it runs per-lane Python loops at every iteration. Each line carries the card it ran on."""
    import ctypes as C
    import subprocess
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip().splitlines()
    batch, n_pts = 16384, 1000
    P = hb.Program(sys_outer_ss(), high_accuracy=True)
    st = outer_ss_batch_state(batch)
    z = np.zeros(batch)
    grid = np.ascontiguousarray(np.linspace(0., 20., n_pts)[:, None] * np.ones(batch)[None, :])
    out = np.empty((n_pts, 36, batch))
    dp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))  # noqa: E731
    hb.check(hb.lib.hy_host_pin(C.c_void_p(out.ctypes.data), C.c_size_t(out.nbytes)))
    n_dev = hb.lib.hy_device_count()
    ref = None
    for device in [-1, [0, 0]] + ([list(range(n_dev))] if n_dev > 1 else []):
        b = hb.Batch(P, batch, device=device)
        times = []
        for _ in range(3):
            b.upload(st, None, z, z)
            b.sync()
            l0 = b.launch_count()
            t0 = time.perf_counter()
            hb.check(hb.lib.hy_batch_propagate_grid(b._h, dp(grid), n_pts, None, 0, dp(out)))
            times.append(time.perf_counter() - t0)
            launches = b.launch_count() - l0
        if ref is None:
            ref = out.copy()
        print(json.dumps({"config": "outer_ss 6-body propagate_grid, %d lanes x %d grid points over 20 yr" % (batch, n_pts),
                          "device": device, "shards": max(b.n_shards, 1), "kernel": b.kernel_info()["tape"],
                          "seconds": min(times), "seconds_all": times, "launches": int(launches),
                          "readbacks_per_iteration": 1 if b.n_shards <= 1 else 2,
                          "lane_steps": int(b.prop_res()[3].sum()),
                          "same_bits_as_one_device": bool(np.array_equal(out.view(np.uint64), ref.view(np.uint64))),
                          "card": card}), flush=True)
        del b
    hb.lib.hy_host_unpin(C.c_void_p(out.ctypes.data))
    del out, ref
    # The front end's host loop over the shards, as every sharded grid ran before it ran on the device.
    span, pts = 2.0, 100
    g = np.linspace(0., span, pts)[:, None] * np.ones(batch)[None, :]
    for device, cb in (([0, 0], None), ([0, 0], lambda ta: True)):
        ta = hb.taylor_adaptive_batch(sys_outer_ss(), st, batch, high_accuracy=True, device=device)
        t0 = time.perf_counter()
        ta.propagate_grid(g, callback=cb)
        dt = time.perf_counter() - t0
        print(json.dumps({"config": "outer_ss 6-body propagate_grid, %d lanes x %d grid points over %g yr, front end"
                                    % (batch, pts, span), "device": device,
                          "path": "device loop" if cb is None else "host loop (step callback)", "seconds": dt,
                          "card": card}), flush=True)


def main():
    which = sys.argv[1:] or ["tb", "n32", "nn", "s6step"]
    if "tbsmall" in which:
        run("two_body_step_batch 2^22 lanes, one step", hb.Program(sys_two_body()), two_body_batch_state(1 << 22))
    if "tb" in which:
        run("two_body_step_batch 2^24 lanes, one step", hb.Program(sys_two_body()), two_body_batch_state(1 << 24))
    if "tbteam" in which:
        run("two_body_step_batch 2^24 lanes, one step, k_nb with 32 lanes per warp", hb.Program(sys_two_body()),
            two_body_batch_state(1 << 24), tape="nbody")
    if "tbsweep" in which:
        for kw in (dict(block_threads=256), dict(block_threads=384), dict(block_threads=512),
                   dict(block_threads=256, lanes_per_thread=2), dict(block_threads=512, lanes_per_thread=2)):
            run("two_body_step_batch 2^22 lanes, one step, k_nb1 %r" % (kw,), hb.Program(sys_two_body()),
                two_body_batch_state(1 << 22), tape="nbody-lane", **kw)
    if "s6long" in which:
        # Long horizon (SURVEY 8(d)): 1000 yr, ~1370 steps per lane (the bench step propagates 20 yr, ~27 steps).
        run("outer_ss 6-body 262144 lanes, propagate_until(1000 yr)", hb.Program(sys_outer_ss(), high_accuracy=True),
            outer_ss_batch_state(1 << 18, perturb=1e-3), 1000.0)
    if "s6step" in which:
        run("outer_ss 6-body 2^20 lanes, one step", hb.Program(sys_outer_ss(), high_accuracy=True),
            outer_ss_batch_state(1 << 20))
    if "grid" in which:
        # propagate_grid(): the 6-body system sampled on 1000 grid points per lane over 20 yr (the dense output of
        # every step goes to a [n_pts][n_eq][batch] array: this one is bandwidth work).
        batch, n_pts = 16384, 1000
        st = outer_ss_batch_state(batch)
        b = hb.Batch(hb.Program(sys_outer_ss(), high_accuracy=True), batch)
        z = np.zeros(batch)
        grid = np.ascontiguousarray(np.linspace(0., 20., n_pts)[:, None] * np.ones(batch)[None, :])
        import ctypes as C
        out = np.empty((n_pts, 36, batch))
        dp = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))  # noqa: E731
        res = {}
        for pinned in (False, True):
            if pinned:
                hb.check(hb.lib.hy_host_pin(C.c_void_p(out.ctypes.data), C.c_size_t(out.nbytes)))
            best = None
            for _ in range(2):
                b.upload(st, None, z, z)
                b.sync()
                l0 = b.launch_count()
                t0 = time.perf_counter()
                hb.check(hb.lib.hy_batch_propagate_grid(b._h, dp(grid), n_pts, None, 0, dp(out)))
                dt = time.perf_counter() - t0
                best = dt if best is None else min(best, dt)
            res["pinned" if pinned else "pageable"] = best
            launches = b.launch_count() - l0
        hb.lib.hy_host_unpin(C.c_void_p(out.ctypes.data))
        assert np.all(np.isfinite(out)) and np.array_equal(out[0], st)
        print(json.dumps({"config": "outer_ss 6-body propagate_grid, %d lanes x %d grid points over 20 yr" % (batch, n_pts),
                          "lanes": batch, "kernel": b.kernel_info()["tape"], "seconds": res["pinned"],
                          "seconds_pageable_output": res["pageable"], "launches": int(launches),
                          "lane_steps": int(b.prop_res()[3].sum()), "output_bytes": int(out.nbytes),
                          "output_gbs_incl_d2h": out.nbytes / res["pinned"] / 1e9}), flush=True)
    if "gridshard" in which:
        grid_sharded()
    if "n32" in which:
        st = nbody32_batch_state(8192)
        run("nbody N=32, 8192 lanes, propagate_until(1)", hb.Program(sys_nbody32()), st, 1.0)
        run("nbody N=32, 8192 lanes, propagate_until(1), generic cooperative kernel (CTA teams, global tape)",
            hb.Program(sys_nbody32()), st, 1.0, tape="global-cta")
        if "n32all" in which:
            run("nbody N=32, 8192 lanes, propagate_until(1), warp teams", hb.Program(sys_nbody32()), st, 1.0, tape="global")
            run("nbody N=32, 8192 lanes, propagate_until(1), thread-per-lane HBM kernel", hb.Program(sys_nbody32()), st,
                1.0, tape="hbm")
    if "nnsmall" in which:
        run("ffnn 3x64 tanh order 15, 16384 lanes, propagate_until(0.5)", hb.Program(sys_ffnn(), tol=FFNN_TOL),
            ffnn_batch_state(1 << 14), 0.5)
    if "nn" in which:
        run("ffnn 3x64 tanh order 15, 262144 lanes, propagate_until(0.5)", hb.Program(sys_ffnn(), tol=FFNN_TOL),
            ffnn_batch_state(1 << 18), 0.5)
        run("ffnn 3x64 tanh order 15, 262144 lanes, propagate_until(0.5), CTA teams", hb.Program(sys_ffnn(), tol=FFNN_TOL),
            ffnn_batch_state(1 << 18), 0.5, tape="global-cta")


if __name__ == "__main__":
    main()
