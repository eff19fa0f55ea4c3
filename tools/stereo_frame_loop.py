"""The reference's live frame loop on the device-side window (the twin of bench.py's sliding_section in the reference's
own configuration): per frame one state element, the frame's stereo tracks -> bearing factors + new landmarks, the IMU
factors, one pose factor every few frames, hb200_slide with both drop flags, 5 LM iterations and a state read-back.

Two variants of the stereo-track step run on two contexts, frame by frame alternately, over the same data:
  composed: hb200_ingest_stereo (bearings + landmarks to the host), hb200_append_landmarks, hb200_append_bearing_factors
  device:   hb200_append_stereo_tracks
Prints one JSON line: median / minimum wall clock per frame of each (host bookkeeping and every copy included), the
window sizes, and the card's name and power limit read in the same run.  --deterministic: both contexts assemble
deterministically, so every frame also pays the slot layout and the entry index of its new window (DESIGN.md §5.4)."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hyperslam_b200 import runtime, synthetic  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "unknown"


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--warm", type=int, default=50, help="frames before timing (the window starts without landmarks and fills up)")
    p.add_argument("--frames", type=int, default=30, help="timed frames per variant")
    p.add_argument("--deterministic", action="store_true", help="both contexts with the deterministic assembly (hb200_set_deterministic)")
    a = p.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("stereo_frame_loop needs a CUDA device")
    K0, k, frame_dt = 50, 4, 0.05
    total = a.warm + a.frames
    # about cfg1's rates: ~2100 visual factors and ~425 IMU samples per second of window
    full = synthetic.make_window(order=k, num_knots=K0 + total + 4, num_landmarks=0, num_imu=int(425 * (K0 + total) * 0.1), seed=synthetic.SEED_BASE + 4600)
    full = synthetic.add_bearing_and_pose_factors(full, num_pose=(K0 + total) // 3, seed=synthetic.SEED_BASE + 4601)
    st = full.knots[:, 7]
    hi0 = st[K0 - 2]
    tracks = synthetic.make_stereo_tracks(full, hi0, hi0 + 0.1 * total, frame_dt=frame_dt, new_per_frame=13, frames_per_landmark=4, seed=synthetic.SEED_BASE + 4602)
    import dataclasses
    kc = np.zeros(K0, np.uint8); kc[:2] = 1
    im0 = full.i_stamp < hi0
    win = dataclasses.replace(full, knots=full.knots[:K0].copy(), landmarks=np.zeros((0, 3)), v_stamp=np.zeros(0), v_cam=np.zeros(0, np.int32), v_lm=np.zeros(0, np.int32),
                              v_pixel=np.zeros((0, 2)), i_stamp=full.i_stamp[im0], i_meas=full.i_meas[im0], m_stamp=np.zeros(0), m_sensor=np.zeros(0, np.int32),
                              m_pose=np.zeros((0, 7)), knot_const=kc, truth=None)
    ctxs = dict(composed=runtime.Context(0), device=runtime.Context(0))
    slots = {name: {} for name in ctxs}   # caller's landmark id -> window slot, per context
    for ctx in ctxs.values():
        ctx.set_deterministic(a.deterministic)
        ctx.load_window(win)
    times = {name: [] for name in ctxs}
    sizes = {}

    def stereo_step(name, ctx, s, gids, px0, px1):
        n = gids.size
        slot = slots[name]
        given = np.array([slot.get(g, -1) for g in gids.tolist()], dtype=np.int32)
        stamp, c0, c1 = np.full(n, s), np.zeros(n, np.int32), np.ones(n, np.int32)
        if name == "device":
            out, _ = ctx.append_stereo_tracks(stamp, c0, c1, px0, px1, given)
        else:
            b0, b1, lm_w, _ = ctx.ingest_stereo(stamp, c0, c1, px0, px1)
            new = given < 0
            out = given.copy()
            out[new] = ctx.L + np.arange(int(new.sum()))
            ctx.append_landmarks(lm_w[new])
            ctx.append_bearing_factors(np.repeat(stamp, 2), np.stack([c0, c1], 1).ravel(), np.repeat(out, 2), np.stack([b0, b1], 1).reshape(-1, 3))
        for g, l in zip(gids.tolist(), out.tolist()):
            slot[g] = l

    prev_hi = hi0
    for f in range(total):
        hi = st[K0 + f - 1]
        cam_frames = np.unique(tracks["stamp"][(tracks["stamp"] >= prev_hi) & (tracks["stamp"] < hi)])
        ii = (full.i_stamp >= prev_hi) & (full.i_stamp < hi)
        mi = np.flatnonzero((full.m_stamp >= prev_hi) & (full.m_stamp < hi))[:1] if f % 3 == 0 else np.zeros(0, np.int64)
        prev_hi = hi
        lower = st[f + 1] + 1e-9   # the window keeps its length: one element in, one out
        for name, ctx in (ctxs.items() if f % 2 == 0 else reversed(list(ctxs.items()))):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ctx.append_knots(1)
            for s in cam_frames:
                t = tracks["stamp"] == s
                stereo_step(name, ctx, s, tracks["gid"][t], tracks["px0"][t], tracks["px1"][t])
            ctx.append_inertial_factors(full.i_stamp[ii], full.i_meas[ii])
            ctx.append_manifold_factors(full.m_stamp[mi], full.m_sensor[mi], full.m_pose[mi])
            stats = ctx.slide(lower, drop_inertial=True, drop_manifold=True)
            ctx.iterate(5, records=False)
            ctx.state()
            dt = time.perf_counter() - t0
            # the caller's id -> slot map follows the slide (outside the timed region: it is the caller's bookkeeping)
            lmap = ctx.landmark_map()
            slots[name] = {g: int(lmap[l]) for g, l in slots[name].items() if lmap[l] >= 0}
            if f >= a.warm:
                times[name].append(dt)
            counts = ctx.factor_counts()
            sizes[name] = dict(knots=stats["knots"], landmarks=stats["landmarks"], bearing_factors=int(counts[runtime.BEARING]),
                               inertial_factors=int(counts[runtime.INERTIAL]), manifold_factors=int(counts[runtime.MANIFOLD]))
    assert sizes["device"] == sizes["composed"], sizes
    out = dict(tool="stereo_frame_loop", card=card(), deterministic=a.deterministic, order=k, K0=K0, warm_frames=a.warm, timed_frames=a.frames,
               window=sizes["device"], per_frame="append 1 state element + the frame's stereo tracks (2 camera frames) + IMU factors (+ 1 pose factor "
               "every 3rd frame), hb200_slide (both drop flags), 5 LM iterations, state read-back; wall clock")
    for name in ctxs:
        out[name] = dict(ms_per_frame_median=statistics.median(times[name]) * 1e3, ms_per_frame_min=min(times[name]) * 1e3)
    print(json.dumps(out))
    for ctx in ctxs.values():
        ctx.close()


if __name__ == "__main__":
    main()
