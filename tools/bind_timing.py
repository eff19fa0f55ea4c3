#!/usr/bin/env python
"""Wall time of hb200_bind after a full set of factor lists, on the cfg1 and cfg2 windows of bench.py.

Each repetition sets the four factor lists again (not timed) and then times one hb200_bind on the host clock; the call
ends in a stream synchronise, so the time covers its kernels, copies and host work.  Prints one JSON line with the
median and minimum per config and the card's name and power limit read in the same run.  Needs an H100.

  python tools/bind_timing.py [--reps 20] [--configs 1,2]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from hyperslam_b200 import runtime, synthetic  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown (nvidia-smi unavailable)"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--configs", default="1,2")
    args = ap.parse_args()
    out = dict(card=card())
    for config in (int(c) for c in args.configs.split(",")):
        win = synthetic.make_window(seed=synthetic.SEED_BASE + config + 1, constant_knots=2, **synthetic.CONFIGS[config])   # as bench.py
        ctx = runtime.Context(0)
        ctx.load_window(win)
        times = []
        for _ in range(args.reps + 2):   # the first two: warm-up
            ctx.set_pixel_factors(win.v_stamp, win.v_cam, win.v_lm, win.v_pixel)
            ctx.set_inertial_factors(win.i_stamp, win.i_meas)
            ctx.set_bearing_factors(win.b_stamp, win.b_cam, win.b_lm, win.b_bearing)
            ctx.set_manifold_factors(win.m_stamp, win.m_sensor, win.m_pose)
            ctx.synchronize()
            t0 = time.perf_counter()
            ctx.bind()
            times.append(1e3 * (time.perf_counter() - t0))
        ctx.close()
        times = sorted(times[2:])
        out[f"cfg{config}"] = dict(factors=win.num_factors, bind_ms_median=round(times[len(times) // 2], 3), bind_ms_min=round(times[0], 3))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
