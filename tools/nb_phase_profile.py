#!/usr/bin/env python3
"""Where the cycles of a k_nb warp-step go: per-phase clock64() attribution of the N-body kernel on the bench workload.

    python tools/nb_phase_profile.py [--batch N] [--tfinal YEARS] [--json FILE]

Builds a copy of the library with -DHY_NB_PHASE_CLOCK in a temporary directory (the source tree is not touched), runs
bench.py's workload (the 6-body outer Solar System, 2^20 lanes, propagate_until(20 yr)) once to warm up and once
measured, and prints the cycles per warp-step (one Taylor step of a warp team's lanes) of each phase of the kernel
(see the phase list in csrc/nb_kernel.cuh), their sum, and the team's whole lifetime per warp-step. The clock reads
and the fire-and-forget atomics add a little to every phase: compare the instrumented kernel time printed here with
an uninstrumented bench.py run to see how much.
"""
import argparse
import ctypes as C
import importlib.util
import json
import os
import shutil
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PHASES = ["pair", "sum", "init", "step_size", "update", "prop"]  # order of nb_kernel.cuh's nb_phase
# Sub-phases of "pair" and "sum" (slots 8 on; see nb_kernel.cuh): each ends where its instructions have been issued,
# the latency of a load is charged to the sub-phase that first uses the value, and the rest of the phase ("sync") is
# the wait at the synchronisation that ends it.
SUB_PHASES = {"pair": ["sum_sq", "main_loop", "pow_quotients", "outputs"],
              "sum": ["role_load", "term_loads", "sum_quotients", "stores_sync"]}
N_SLOTS = 16  # per team: the phases, the warp-steps, the lifetime, then the sub-phases


def build_instrumented(tmp, force=True):
    """Copies the package sources and headers to tmp and builds the library there with the phase clock on (without
    force, only the objects older than their sources are rebuilt)."""
    shutil.copytree(os.path.join(ROOT, "heyoka_b200"), os.path.join(tmp, "heyoka_b200"),
                    ignore=shutil.ignore_patterns("lib", "__pycache__"), dirs_exist_ok=True)
    shutil.copytree(os.path.join(ROOT, "include"), os.path.join(tmp, "include"), dirs_exist_ok=True)
    spec = importlib.util.spec_from_file_location("hb_build_clock", os.path.join(tmp, "heyoka_b200", "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.CUDA_FLAGS = mod.CUDA_FLAGS + ["-DHY_NB_PHASE_CLOCK=1"]
    mod.build(force=force, verbose=False)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=1 << 20)
    ap.add_argument("--tfinal", type=float, default=20.0)
    ap.add_argument("--json", default=None, help="also write the table as JSON")
    ap.add_argument("--build-dir", default=None, help="build the instrumented copy in this directory and keep it "
                    "(a build already there is brought up to date), instead of a temporary directory")
    ap.add_argument("--build-only", action="store_true", help="build the instrumented copy, do not run it")
    args = ap.parse_args()

    with tempfile.TemporaryDirectory(prefix="heyoka_nb_clock_") as tmp:
        t0 = time.perf_counter()
        if args.build_dir:
            tmp = os.path.abspath(args.build_dir)
            os.makedirs(tmp, exist_ok=True)
        build_instrumented(tmp, force=not args.build_dir)
        if args.build_only:
            return
        print("instrumented build: %.0f s" % (time.perf_counter() - t0), flush=True)
        sys.path.insert(0, tmp)
        sys.path.insert(1, os.path.join(ROOT, "tests"))
        import heyoka_b200 as hb
        assert os.path.dirname(os.path.abspath(hb.__file__)).startswith(tmp), hb.__file__
        from common import outer_ss_batch_state, sys_outer_ss

        P = hb.Program(sys_outer_ss(), high_accuracy=True)
        st = outer_ss_batch_state(args.batch, perturb=1e-3, seed=42)
        b = hb.Batch(P, args.batch)
        ki = b.kernel_info()
        if ki["tape"] != "nbody":
            raise SystemExit("the workload does not run on k_nb with warp teams: %r" % (ki,))
        read = getattr(hb.lib, "hy_nb_phase_clock_lt%d_cta0" % ki["lanes_per_warp"])
        read.restype = C.c_int
        read.argtypes = [C.POINTER(C.c_ulonglong), C.c_size_t]
        cap = read(None, 0)
        z = np.zeros(args.batch)
        tf = np.full(args.batch, args.tfinal)

        def run():
            b.upload(st, None, z, z)
            b.sync()
            t = time.perf_counter()
            b.propagate_until(tf)
            b.sync()
            return time.perf_counter() - t

        run()  # warm-up
        buf = (C.c_ulonglong * (cap * N_SLOTS))()
        read(buf, 0)  # reset
        secs = run()
        if read(buf, cap * N_SLOTS) < 0:
            raise SystemExit("hy_nb_phase_clock failed")
        a = np.frombuffer(buf, dtype=np.uint64).reshape(cap, N_SLOTS).astype(np.float64)
        teams = int(np.count_nonzero(a[:, 7]))
        steps = a[:, 6].sum()
        per = {ph: a[:, i].sum() / steps for i, ph in enumerate(PHASES)}
        sub = {}
        slot = 8
        for ph, names in SUB_PHASES.items():
            sub[ph] = {nm: a[:, slot + i].sum() / steps for i, nm in enumerate(names)}
            sub[ph]["sync"] = per[ph] - sum(sub[ph].values())
            slot += len(names)
        life = a[:, 7].sum() / steps
        lane_steps = int(b.prop_res()[3].sum())
        res = {"kernel_info": {k: ki[k] for k in ("tape", "lanes_per_warp", "block_threads", "smem_bytes")},
               "lanes": args.batch, "lane_steps": lane_steps, "teams": teams, "warp_steps": int(steps),
               "seconds_instrumented": secs, "cycles_per_warp_step": per, "sub_phases": sub,
               "sum": sum(per.values()),
               "lifetime_per_warp_step": life,
               # The SM clock the cycles ran at: the longest team lifetime over the propagate call's wall time.
               "sm_ghz_effective": a[:, 7].max() / secs / 1e9}
        print("%-10s %10s %7s" % ("phase", "cycles", "share"))
        for ph in PHASES:
            print("%-10s %10.0f %6.1f%%" % (ph, per[ph], 100. * per[ph] / life))
            for nm, v in sub.get(ph, {}).items():
                print("  %-14s %8.0f %6.1f%%" % (nm, v, 100. * v / life))
        print("%-10s %10.0f %6.1f%%" % ("sum", res["sum"], 100. * res["sum"] / life))
        print("%-10s %10.0f   (team lifetime / warp-steps: %d teams, %d warp-steps, %d lane-steps, %.3f s, "
              "%.2f GHz effective)" % ("lifetime", life, teams, steps, lane_steps, secs, res["sm_ghz_effective"]))
        print(json.dumps(res))
        if args.json:
            with open(args.json, "w") as f:
                json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
