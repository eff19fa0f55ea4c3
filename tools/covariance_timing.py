"""Time the marginal covariances on the device: hb200_build_covariance, hb200_compute_covariance (selected inverse +
landmark marginals), hb200_interpolate_covariance and hb200_interpolate_state_covariance at 1000 stamps, with CUDA
events around each call (host copies included), on cfg1, cfg2 and a K = 500 window.  Prints the card and its power
limit first; one JSON line per window.  --baseline-lib PATH alternates, round by round, with contexts of another build
of libhyperb200.so (the calls it lacks are skipped) and prints its line (lib = "baseline") after each window's.
--blocks times the compute alone with requested blocks outside the pattern (see blocks()), after the card, its power
limit and SM clocks.  --stamp-pairs N times the compute alone without and with N registered stamp pairs (see
stamp_pairs()); with --baseline-lib the compute without pairs alternates with the other build's.

    python tools/covariance_timing.py [--reps 5] [--baseline-lib PATH] [--blocks | --stamp-pairs N]
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


def blocks(reps):
    """--blocks: hb200_compute_covariance with no requested blocks, with every far knot pair of cfg1 (all knot pairs more
    than beta apart), and with 1000 landmark x knot plus 1000 landmark x landmark pairs on the K = 500 window."""
    import torch
    from hyperslam_b200 import runtime
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                       timeout=30)
    print(f"# {q.stdout.strip().splitlines()[0]}")
    rng = np.random.default_rng(7)
    for name in ("cfg1", "K500"):
        win = window(name)
        ctx = runtime.Context(0)
        ctx.load_window(win)
        K, L, beta = win.knots.shape[0], win.landmarks.shape[0], ctx.bandwidth()
        cases = {"none": np.zeros((0, 4), np.int32)}
        if name == "cfg1":
            cases["far_knot_pairs"] = np.array([(0, i, 0, j) for j in range(K) for i in range(j - beta)], np.int32)
        else:
            lk = np.stack([np.full(1000, 4), rng.integers(0, L, 1000), np.zeros(1000, int), rng.integers(0, K, 1000)], 1)
            ll = np.stack([np.full(1000, 4), rng.integers(0, L, 1000), np.full(1000, 4), rng.integers(0, L, 1000)], 1)
            cases["landmark_pairs"] = np.concatenate([lk, ll]).astype(np.int32)
        stream = torch.cuda.ExternalStream(ctx.stream)
        for case, req in cases.items():
            ctx.set_covariance_blocks(req)
            times, launches = [], 0
            for r in range(reps + 1):
                ctx.build_covariance()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                l0 = ctx.launch_count
                e0.record(stream)
                info = ctx.compute_covariance()
                e1.record(stream)
                e1.synchronize()
                launches = ctx.launch_count - l0
                if r:   # first round: warm-up
                    times.append(e0.elapsed_time(e1))
            _, st = ctx.covariance_blocks()
            print(json.dumps(dict(window=name, case=case, K=K, beta=beta, L=L, pairs=len(req), status=info["status"], launches=launches,
                                  computed=int((st == 0).sum()), compute_ms=float(np.median(times)), reps=reps)))
        ctx.close()


def load_baseline(path):
    import ctypes
    base = ctypes.CDLL(os.path.abspath(path))   # RTLD_LOCAL: both builds' symbols stay apart
    for fn, res in (("hb200_last_error_string", ctypes.c_char_p), ("hb200_stream", ctypes.c_void_p), ("hb200_launch_count", ctypes.c_longlong)):
        getattr(base, fn).restype = res
    base.hb200_launch_count.argtypes = [ctypes.c_void_p]
    base.hb200_destroy.argtypes, base.hb200_destroy.restype = [ctypes.c_void_p], None
    return base


def stamp_pairs(reps, npairs, baseline_lib):
    """--stamp-pairs N: hb200_compute_covariance on cfg1 and the K = 500 window without stamp pairs and with N pairs drawn
    uniformly over the valid span (most of them more than beta knots apart, so the far-column march runs); with a
    baseline build, its compute without pairs alternates round by round with this build's."""
    import torch
    from hyperslam_b200 import runtime
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                       timeout=30)
    print(f"# {q.stdout.strip().splitlines()[0]}")
    libs = dict(current=runtime.load_library())
    if baseline_lib:
        libs["baseline"] = load_baseline(baseline_lib)
    for name in ("cfg1", "K500"):
        win = window(name)
        kt, k = win.knots[:, 7], win.order
        left = (k - 1) // 2
        pairs = np.random.default_rng(11).uniform(kt[left], kt[len(kt) - k + left + 1], (npairs, 2))
        runs = []   # (lib, case, context)
        for lib_name, lib in libs.items():
            runtime._lib = lib          # a Context keeps the library it was created with
            for case in (("none", "pairs") if lib_name == "current" else ("none",)):
                ctx = runtime.Context(0)
                ctx.load_window(win)
                if case == "pairs":
                    ctx.set_covariance_stamp_pairs(pairs)
                runs.append((lib_name, case, ctx))
        runtime._lib = libs["current"]
        times = {(l, c): [] for l, c, _ in runs}
        launches, info = {}, {}
        for r in range(reps + 1):
            for lib_name, case, ctx in runs:
                stream = torch.cuda.ExternalStream(ctx.stream)
                ctx.build_covariance()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                l0 = ctx.launch_count
                e0.record(stream)
                info[lib_name, case] = ctx.compute_covariance()
                e1.record(stream)
                e1.synchronize()
                launches[lib_name, case] = ctx.launch_count - l0
                if r:   # first round: warm-up
                    times[lib_name, case].append(e0.elapsed_time(e1))
        for lib_name, case, ctx in runs:
            computed = int((ctx.pose_pair_covariance()[2] == 0).sum()) if case == "pairs" else 0
            print(json.dumps(dict(window=name, lib=lib_name, case=case, K=win.knots.shape[0], beta=info[lib_name, case]["beta"],
                                  pairs=npairs if case == "pairs" else 0, computed=computed, status=info[lib_name, case]["status"],
                                  launches=launches[lib_name, case], compute_ms=float(np.median(times[lib_name, case])),
                                  spread_ms=float(np.ptp(times[lib_name, case])), reps=reps)))
            ctx.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--baseline-lib", default=None)
    ap.add_argument("--blocks", action="store_true", help="time the compute with requested blocks outside the pattern")
    ap.add_argument("--stamp-pairs", type=int, default=0, help="time the compute with this many registered stamp pairs")
    args = ap.parse_args()
    if args.blocks:
        return blocks(args.reps)
    if args.stamp_pairs:
        return stamp_pairs(args.reps, args.stamp_pairs, args.baseline_lib)
    import torch
    from hyperslam_b200 import runtime
    libs = dict(current=runtime.load_library())
    if args.baseline_lib:
        libs["baseline"] = load_baseline(args.baseline_lib)
    print(f"# {card()}")
    for name in ("cfg1", "cfg2", "K500"):
        win = window(name)
        ctxs = {}
        for lib_name, lib in libs.items():
            runtime._lib = lib          # a Context keeps the library it was created with
            ctxs[lib_name] = runtime.Context(0)
            ctxs[lib_name].load_window(win)
        runtime._lib = libs["current"]
        kt = win.knots[:, 7]
        stamps = np.linspace(kt[win.order], kt[-win.order], 1000)
        t = {n: dict(build=[], compute=[], interpolate=[], interpolate_state=[]) for n in ctxs}
        info = {}
        for r in range(args.reps + 1):
            for lib_name, ctx in ctxs.items():
                stream = torch.cuda.ExternalStream(ctx.stream)
                calls = [("build", ctx.build_covariance), ("compute", ctx.compute_covariance),
                         ("interpolate", lambda: ctx.interpolate_covariance(stamps))]
                if hasattr(ctx.lib, "hb200_interpolate_state_covariance"):
                    calls.append(("interpolate_state", lambda: ctx.interpolate_state_covariance(stamps)))
                for key, fn in calls:
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(stream)
                    out = fn()
                    e1.record(stream)
                    e1.synchronize()
                    if key == "compute":
                        info[lib_name] = out
                    if r:   # first round: warm-up
                        t[lib_name][key].append(e0.elapsed_time(e1))
        for lib_name, ctx in ctxs.items():
            inf = info[lib_name]
            K, beta, m, L = inf["K"], inf["beta"], inf["m"], inf["L"]
            print(json.dumps(dict(window=name, lib=lib_name, K=K, beta=beta, m=m, L=L, status=inf["status"], min_pivot_ratio=inf["min_pivot_ratio"],
                                  **{f"{k}_ms": float(np.median(v)) for k, v in t[lib_name].items() if v}, reps=args.reps)))
            ctx.close()


if __name__ == "__main__":
    main()
