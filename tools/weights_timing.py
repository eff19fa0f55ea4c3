#!/usr/bin/env python
"""LM step time without family weight matrices and with one set for every family (hb200_set_weights).

For cfg1, cfg2 (the order-6 200-knot window) and the 1M-factor window (cfg4): one context per mode on the same window,
the two modes timed alternately in rounds, each step as bench.py times it (device snapshot restored before every step,
256 MiB L2 flush, CUDA events around one graph-launched iteration).  Also prints the per-kernel split of one iteration in
each mode (hb200_profile_iteration) -- on cfg1 a set inertial matrix moves the inertial J^T J from the scalar kernel to
the tensor-core one -- and the card's name and power limit read in the same run.  Needs an H100.

  python tools/weights_timing.py [--steps 50] [--rounds 4] [--configs 1,2,4]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from hyperslam_b200 import runtime, synthetic  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown (nvidia-smi unavailable)"


def weights():
    """A dense, non-symmetric matrix per family, close to a whitening matrix (diagonal dominant)."""
    rng = np.random.default_rng(7)
    out = {}
    for kind, d in runtime.Context.WEIGHT_SIDES.items():
        out[kind] = np.eye(d) * 2.0 + rng.uniform(-0.25, 0.25, size=(d, d))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--configs", default="1,2,4")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device")
    flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device="cuda")
    out = dict(card=card())
    print(json.dumps(out), flush=True)
    for cfg in (int(c) for c in args.configs.split(",")):
        win = synthetic.make_config(cfg, constant_knots=2)
        ctxs = {}
        for mode in ("off", "weighted"):
            ctx = runtime.Context(0, use_graph=True)
            ctx.load_window(win)
            if mode == "weighted":
                for kind, W in weights().items():
                    ctx.set_weights(kind, W)
            ctx.snapshot()
            ctx.iterate(1, records=False)
            ctx.restore()
            ctx.synchronize()
            ctxs[mode] = ctx
        ext = {m: torch.cuda.ExternalStream(c.stream) for m, c in ctxs.items()}
        ms = {m: [] for m in ctxs}
        for _ in range(args.rounds):
            for mode, ctx in ctxs.items():
                for _ in range(3):   # warm-up
                    ctx.restore(); ctx.iterate(1, records=False)
                ctx.synchronize()
                ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
                for a, b in ev:
                    ctx.restore()
                    with torch.cuda.stream(ext[mode]):
                        flush.fill_(1.0)
                    a.record(ext[mode])
                    ctx.iterate(1, records=False)
                    b.record(ext[mode])
                ctx.synchronize(); torch.cuda.synchronize()
                ms[mode].append(sum(a.elapsed_time(b) for a, b in ev) / args.steps)
        prof = {}
        for mode, ctx in ctxs.items():
            ctx.restore()
            agg = {}
            for name, t in ctx.profile_iteration(reps=3):
                agg[name] = round(agg.get(name, 0.0) + t, 4)
            prof[mode] = agg
        entry = dict(workload=synthetic.CONFIG_NAMES[cfg], factors=win.num_factors,
                     ms_per_step={m: dict(per_round=[round(x, 4) for x in v], median=round(sorted(v)[len(v) // 2], 4)) for m, v in ms.items()},
                     iteration_kernel_ms=prof)
        print(json.dumps(entry), flush=True)
        for ctx in ctxs.values():
            ctx.close()
    print(json.dumps(dict(card=out["card"])))


if __name__ == "__main__":
    main()
