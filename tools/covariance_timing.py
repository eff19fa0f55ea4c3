"""Time the marginal covariances on the device: hb200_build_covariance, hb200_compute_covariance (selected inverse +
landmark marginals) and hb200_interpolate_covariance at 1000 stamps, with CUDA events around each call, on cfg1, cfg2
and a K = 500 window.  Prints the card and its power limit first; one JSON line per window.

    python tools/covariance_timing.py [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        return q.stdout.strip().splitlines()[0]
    except Exception as e:   # no nvidia-smi: the device name from torch
        import torch
        return f"{torch.cuda.get_device_name(0)}, power limit unknown ({e})"


def window(name):
    import covref as cr
    from hyperslam_b200 import synthetic
    if name == "cfg1":
        win = synthetic.make_config(1)
    elif name == "cfg2":
        win = synthetic.make_config(2)
    else:
        win = synthetic.make_window(order=4, num_knots=500, num_landmarks=8192, frames_per_landmark=3, num_imu=4000, seed=synthetic.SEED_BASE + 2021)
    win = synthetic.add_bearing_and_pose_factors(win, num_pose=20)
    win.knot_const[:win.order] = 1
    win.knot_const[cr.untouched_knots(win)] = 1
    return win


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch
    from hyperslam_b200 import runtime
    print(f"# {card()}")
    for name in ("cfg1", "cfg2", "K500"):
        win = window(name)
        ctx = runtime.Context(0)
        ctx.load_window(win)
        stream = torch.cuda.ExternalStream(ctx.stream)
        kt = win.knots[:, 7]
        stamps = np.linspace(kt[win.order], kt[-win.order], 1000)
        t = dict(build=[], compute=[], interpolate=[])
        info = None
        for r in range(args.reps + 1):
            for key, fn in (("build", ctx.build_covariance), ("compute", ctx.compute_covariance), ("interpolate", lambda: ctx.interpolate_covariance(stamps))):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                out = fn()
                e1.record(stream)
                e1.synchronize()
                if key == "compute":
                    info = out
                if r:   # first round: warm-up
                    t[key].append(e0.elapsed_time(e1))
        K, beta, m, L = info["K"], info["beta"], info["m"], info["L"]
        print(json.dumps(dict(window=name, K=K, beta=beta, m=m, L=L, status=info["status"], min_pivot_ratio=info["min_pivot_ratio"],
                              **{f"{k}_ms": float(np.median(v)) for k, v in t.items()}, reps=args.reps)))
        ctx.close()


if __name__ == "__main__":
    main()
