"""Variational integrators: lane-steps/s of propagate_until() for the variational pendulum, two-body (156 equations)
and 6-body (1332 equations) systems next to the same systems without variational equations, the kernel that automatic
selection picked, and the device Taylor map (k_taylor_map) timed with CUDA events over many launches on inputs
resident in HBM. One JSON line per measurement, plus one with the card's name and power limit.

    python tools/bench_variational.py [--out FILE]
"""
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import heyoka_b200 as hb  # noqa: E402
from common import outer_ss_batch_state, sys_outer_ss, sys_two_body, two_body_batch_state  # noqa: E402

HBM_PEAK = 3.35e12  # H100 SXM HBM3, bytes/s


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
        name, plim = [s.strip() for s in q.split(",")]
    except Exception as e:  # noqa: BLE001
        name, plim = "unknown (%s)" % e, "unknown"
    return {"card": name, "power_limit": plim}


def propagate(label, sys_, x0, t_final, variational, reps=3):
    batch = x0.shape[1]
    vs = hb.var_ode_sys(sys_, hb.var_args.vars) if variational else None
    P = hb.Program(vs if variational else sys_)
    st = hb._var_initial_state(vs, x0, batch) if variational else x0
    b = hb.Batch(P, batch)
    z = np.zeros(batch)
    tf = np.full(batch, t_final)
    best = None
    for _ in range(reps):
        b.upload(st, None, z, z)
        b.sync()
        t0 = time.perf_counter()
        b.propagate_until(tf)
        b.sync()
        dt = time.perf_counter() - t0
        best = dt if best is None else min(best, dt)
    ns = int(b.prop_res()[3].sum())
    ki = b.kernel_info()
    return {"system": label, "variational": variational, "n_eq": P.n_eq, "lanes": batch, "t_final": t_final,
            "lane_steps": ns, "seconds": best, "lane_steps_per_s": ns / best,
            "kernel": {k: ki[k] for k in ("tape", "lanes_per_warp", "lanes_per_thread", "block_threads", "smem_bytes")}}


def taylor_map(label, sys_, batch, launches=20):
    import torch
    vs = hb.var_ode_sys(sys_, hb.var_args.vars)
    n, m = vs.n_orig_sv, len(vs.vargs)
    P = hb.Program(vs)
    # The state stays device-resident as the batch allocated it: its values do not change the traffic of the map.
    b = hb.Batch(P, batch)
    dx = torch.empty((m, batch), dtype=torch.float64, device="cuda").uniform_(-1e-3, 1e-3)
    out = torch.empty((n, batch), dtype=torch.float64, device="cuda")
    b.eval_taylor_map_dev(n, m, dx.data_ptr(), out.data_ptr())  # warm-up
    b.sync()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(launches):
        b.eval_taylor_map_dev(n, m, dx.data_ptr(), out.data_ptr())
    e1.record()
    e1.synchronize()
    sec = e0.elapsed_time(e1) / 1e3 / launches
    nbytes = 8.0 * batch * (n * m + n + m + n)  # Phi and x read, dx read, out written
    return {"taylor_map": label, "n_orig_sv": n, "n_args": m, "lanes": batch, "seconds_per_launch": sec,
            "bytes": nbytes, "GB_per_s": nbytes / sec / 1e9, "share_of_3.35TB_per_s": nbytes / sec / HBM_PEAK}


def main():
    out = sys.argv[sys.argv.index("--out") + 1] if "--out" in sys.argv else None
    lines = [card()]
    pend = hb.model.pendulum()
    rng = np.random.default_rng(3)
    for label, sys_, x0, tf in (("pendulum", pend, np.stack([rng.uniform(-1, 1, 1 << 20), rng.uniform(-1, 1, 1 << 20)]),
                                 10.0),
                                ("two-body", sys_two_body(), two_body_batch_state(1 << 16), 10.0),
                                ("6-body", sys_outer_ss(), outer_ss_batch_state(4096), 100.0)):
        for variational in (False, True):
            lines.append(propagate(label, sys_, x0, tf, variational))
            print(json.dumps(lines[-1]), flush=True)
    lines.append(taylor_map("6-body", sys_outer_ss(), 1 << 20))
    print(json.dumps(lines[-1]), flush=True)
    lines.append(taylor_map("two-body", sys_two_body(), 1 << 20))
    print(json.dumps(lines[-1]), flush=True)
    print(json.dumps(lines[0]))
    if out:
        with open(out, "w") as f:
            f.write("\n".join(json.dumps(ln) for ln in lines) + "\n")


if __name__ == "__main__":
    main()
