"""What the angle reducer costs: a rotating pendulum (above the separatrix, the angle grows without bound) over 2^20 lanes,
propagate_until() three ways, in lane-steps per second:

  none    no callback: the whole loop in one device launch;
  device  callback.angle_reducer: the reduction inside the same device loop (hy_batch_set_angles());
  host    the reducer wrapped in a function: the front end's lock-step loop on the host, one device step and one state
          download / upload per iteration.

The host loop is timed over a shorter interval (--host-tf): its rate does not depend on the length of the run, and at
2^20 lanes each of its iterations takes a large fraction of a second. Prints one JSON line, with the card's name and
power limit read in the same process.

    python tools/bench_angle_reducer.py [--lanes 1048576] [--tf 10] [--host-tf 0.2] [--repeat 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import heyoka_b200 as hb  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def make(lanes):
    x, v = hb.make_vars("x", "v")
    sys_ = [(x, v), (v, -9.8 * hb.sin(x))]
    rng = np.random.default_rng(1)
    st = np.concatenate([rng.uniform(-np.pi, np.pi, lanes), (6.5 + 2 * rng.random(lanes)) * rng.choice([-1, 1], lanes)])
    return hb.taylor_adaptive_batch(sys_, st, lanes), x


def rate(lanes, tf, mode, repeat):
    best = None
    for _ in range(repeat):
        ta, x = make(lanes)
        ar = hb.callback.angle_reducer([x])
        cb = {"none": None, "device": ar, "host": lambda t: ar(t)}[mode]
        t0 = time.perf_counter()
        ta.propagate_until(tf, callback=cb)
        dt = time.perf_counter() - t0
        steps = sum(r[3] for r in ta.propagate_res)
        if mode != "none":
            assert np.all((ta.state[0] >= 0) & (ta.state[0] < 2 * np.pi))
        r = steps / dt
        best = r if best is None else max(best, r)
    return best, steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lanes", type=int, default=1 << 20)
    ap.add_argument("--tf", type=float, default=10.0)
    ap.add_argument("--host-tf", type=float, default=0.2)
    ap.add_argument("--repeat", type=int, default=3)
    a = ap.parse_args()
    rate(1024, 0.5, "device", 1)  # warm-up: module load, kernel selection
    res = {"card": card(), "lanes": a.lanes}
    for mode, tf, rep in (("none", a.tf, a.repeat), ("device", a.tf, a.repeat), ("host", a.host_tf, 1)):
        r, steps = rate(a.lanes, tf, mode, rep)
        res[mode] = {"tf": tf, "lane_steps": steps, "lane_steps_per_s": r}
    res["device_over_none"] = res["device"]["lane_steps_per_s"] / res["none"]["lane_steps_per_s"]
    res["device_over_host"] = res["device"]["lane_steps_per_s"] / res["host"]["lane_steps_per_s"]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
