"""A long stereo-inertial frame loop on the device-side window whose bias splines start with kb knots and grow with the
sequence (hb200_append_bias_knots before each frame's IMU samples), with and without HB200_SLIDE_DROP_BIAS.

Per frame, on each of two contexts (frame by frame alternately, same data): one state element, the frame's stereo
tracks, updateSensor for the newest IMU sample + the IMU factors, one pose factor every 3rd frame, hb200_slide
(DROP_INERTIAL | DROP_MANIFOLD, and DROP_BIAS on the "drop_bias" context), 5 LM iterations, state read-back.
Prints one JSON line: per variant the median wall clock per frame at the start and at the end of the run, Kbg, Kba and
m = 3 (Kbg + Kba) + 2 at the end, the solver kernel of the last iteration, and the card's name and power limit read in
the same run.  A variant whose window stops fitting a solver reports the frame and the error instead."""
import argparse
import dataclasses
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hyperslam_b200 import runtime, synthetic  # noqa: E402

SOLVER_KERNELS = {"band_solve_kernel", "band_solve_kernel<false>", "bcr_solve_kernel", "cholesky_kernel"}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "unknown"


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--frames", type=int, default=400, help="frames in the run (one state element each, 0.1 s)")
    p.add_argument("--warm", type=int, default=50, help="frames before the first timed block (the window fills up)")
    p.add_argument("--block", type=int, default=30, help="frames per median (start and end)")
    p.add_argument("--bias-dt", type=float, default=1.0, help="bias knot separation, seconds")
    p.add_argument("--K0", type=int, default=50, help="state elements in the window")
    a = p.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bias_frame_loop needs a CUDA device")
    K0, k, kb, frame_dt = a.K0, 4, 4, 0.05
    total = a.frames
    full = synthetic.make_window(order=k, num_knots=K0 + total + 4, num_landmarks=0, num_imu=int(425 * (K0 + total) * 0.1), seed=synthetic.SEED_BASE + 4700)
    full = synthetic.add_bearing_and_pose_factors(full, num_pose=(K0 + total) // 3, seed=synthetic.SEED_BASE + 4701)
    st = full.knots[:, 7]
    lo0, hi0 = st[1], st[K0 - 2]
    tracks = synthetic.make_stereo_tracks(full, hi0, hi0 + 0.1 * total, frame_dt=frame_dt, new_per_frame=13, frames_per_landmark=4, seed=synthetic.SEED_BASE + 4702)
    bias = []
    for src in (full.gyro_bias, full.accel_bias):   # kb knots whose valid span starts with the window
        b = np.zeros((kb, 4))
        b[:, :3] = src[0, :3]
        b[:, 3] = lo0 + (np.arange(kb) - (kb - 1) // 2) * a.bias_dt
        bias.append(b)
    kc = np.zeros(K0, np.uint8); kc[:2] = 1
    win = dataclasses.replace(full, knots=full.knots[:K0].copy(), gyro_bias=bias[0], accel_bias=bias[1], landmarks=np.zeros((0, 3)), v_stamp=np.zeros(0),
                              v_cam=np.zeros(0, np.int32), v_lm=np.zeros(0, np.int32), v_pixel=np.zeros((0, 2)), i_stamp=np.zeros(0), i_meas=np.zeros((0, 6)),
                              m_stamp=np.zeros(0), m_sensor=np.zeros(0, np.int32), m_pose=np.zeros((0, 7)), knot_const=kc, truth=None)
    im0 = (full.i_stamp >= lo0) & (full.i_stamp < hi0)
    ctxs = dict(drop_bias=runtime.Context(0), keep_bias=runtime.Context(0))
    slots = {name: {} for name in ctxs}
    times = {name: [] for name in ctxs}
    failed = {}
    for ctx in ctxs.values():
        ctx.load_window(win)
        ctx.append_bias_knots(full.i_stamp[im0].max())
        ctx.append_inertial_factors(full.i_stamp[im0], full.i_meas[im0])

    # the window's own stamps: hb200_append_knots continues them at the last separation (one rounding per element),
    # so the frame boundaries follow them rather than the template's, and every sample of a frame binds
    wst = list(st[:K0])
    prev_hi = hi0
    for f in range(total):
        wst.append(wst[-1] + (wst[-1] - wst[-2]))
        hi = wst[K0 + f - 1]
        cam_frames = np.unique(tracks["stamp"][(tracks["stamp"] >= prev_hi) & (tracks["stamp"] < hi)])
        ii = (full.i_stamp >= prev_hi) & (full.i_stamp < hi)
        mi = np.flatnonzero((full.m_stamp >= prev_hi) & (full.m_stamp < hi))[:1] if f % 3 == 0 else np.zeros(0, np.int64)
        prev_hi = hi
        lower = st[f + 1] + 1e-9
        for name, ctx in (ctxs.items() if f % 2 == 0 else reversed(list(ctxs.items()))):
            if name in failed:
                continue
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            try:
                ctx.append_knots(1)
                for s in cam_frames:
                    t = tracks["stamp"] == s
                    gids = tracks["gid"][t]
                    n = gids.size
                    given = np.array([slots[name].get(g, -1) for g in gids.tolist()], dtype=np.int32)
                    out, _ = ctx.append_stereo_tracks(np.full(n, s), np.zeros(n, np.int32), np.ones(n, np.int32), tracks["px0"][t], tracks["px1"][t], given)
                    for g, l in zip(gids.tolist(), out.tolist()):
                        slots[name][g] = l
                if ii.any():
                    ctx.append_bias_knots(full.i_stamp[ii].max())
                    ctx.append_inertial_factors(full.i_stamp[ii], full.i_meas[ii])
                ctx.append_manifold_factors(full.m_stamp[mi], full.m_sensor[mi], full.m_pose[mi])
                ctx.slide(lower, drop_inertial=True, drop_manifold=True, drop_bias=(name == "drop_bias"))
                ctx.iterate(5, records=False)
                ctx.state()
            except runtime.HB200Error as e:
                failed[name] = dict(frame=f, Kbg=ctx.Kbg, Kba=ctx.Kba, m=3 * (ctx.Kbg + ctx.Kba) + 2, error=str(e))
                continue
            times[name].append(time.perf_counter() - t0)
            lmap = ctx.landmark_map()
            slots[name] = {g: int(lmap[l]) for g, l in slots[name].items() if lmap[l] >= 0}
    out = dict(tool="bias_frame_loop", card=card(), order=k, K0=K0, frames=total, bias_dt=a.bias_dt,
               per_frame="append 1 state element + the frame's stereo tracks + bias knots for the newest IMU sample + IMU factors "
               "(+ 1 pose factor every 3rd frame), hb200_slide, 5 LM iterations, state read-back; wall clock")
    for name, ctx in ctxs.items():
        tt = times[name]
        r = dict(ms_per_frame_median_start=statistics.median(tt[a.warm:a.warm + a.block]) * 1e3 if len(tt) >= a.warm + a.block else None,
                 ms_per_frame_median_end=statistics.median(tt[-a.block:]) * 1e3 if len(tt) >= a.warm + 2 * a.block else None,
                 frames_run=len(tt))
        if name in failed:
            r["failed"] = failed[name]
        else:
            solver = sorted({n for n, _ in ctx.profile_iteration(reps=1)} & SOLVER_KERNELS)
            r.update(Kbg=ctx.Kbg, Kba=ctx.Kba, m=3 * (ctx.Kbg + ctx.Kba) + 2, K=ctx.K, solver=solver)
        out[name] = r
    print(json.dumps(out))
    for ctx in ctxs.values():
        ctx.close()


if __name__ == "__main__":
    main()
