"""The reference's live frame loop (tools/stereo_frame_loop.py's sequence) on a sharded window: N contexts on device 0
reduce through the all-reduce hook (tests/test_gpu_sharded.py's HostReducer, one thread per rank), alternating frame by
frame with one context on the whole window.  Per frame: one state element on every rank, the frame's stereo tracks to
their landmark's owner (gid mod N; every rank makes every append_stereo_tracks call, n = 0 included), IMU and pose
factors to one rank in turn, hb200_slide (both drop flags) on every rank, 5 LM iterations, state read-back.

Prints one JSON line: median / minimum wall clock per frame of both, the agreement rounds per frame (hook calls outside
the LM iterations), window sizes, and the card's name and power limit read in the same run.  On one GPU the N ranks share
the device and the hook is a host-side barrier plus a sum on the device: the numbers show what the agreement and the
hook cost per frame, not multi-GPU scaling.  The NCCL and peer-memory reductions are not measured by this tool."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from hyperslam_b200 import runtime, synthetic  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "unknown"


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--world", type=int, default=2, help="ranks (contexts on device 0)")
    p.add_argument("--warm", type=int, default=50, help="frames before timing (the window starts without landmarks and fills up)")
    p.add_argument("--frames", type=int, default=30, help="timed frames")
    a = p.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("sharded_frame_loop needs a CUDA device")
    from test_gpu_sharded import HostReducer, on_ranks
    import dataclasses
    N, K0, k, frame_dt = a.world, 50, 4, 0.05
    total = a.warm + a.frames
    full = synthetic.make_window(order=k, num_knots=K0 + total + 4, num_landmarks=0, num_imu=int(425 * (K0 + total) * 0.1), seed=synthetic.SEED_BASE + 4600)
    full = synthetic.add_bearing_and_pose_factors(full, num_pose=(K0 + total) // 3, seed=synthetic.SEED_BASE + 4601)
    st = full.knots[:, 7]
    hi0 = st[K0 - 2]
    tracks = synthetic.make_stereo_tracks(full, hi0, hi0 + 0.1 * total, frame_dt=frame_dt, new_per_frame=13, frames_per_landmark=4, seed=synthetic.SEED_BASE + 4602)
    kc = np.zeros(K0, np.uint8); kc[:2] = 1
    im0 = full.i_stamp < hi0
    win = dataclasses.replace(full, knots=full.knots[:K0].copy(), landmarks=np.zeros((0, 3)), v_stamp=np.zeros(0), v_cam=np.zeros(0, np.int32), v_lm=np.zeros(0, np.int32),
                              v_pixel=np.zeros((0, 2)), i_stamp=full.i_stamp[im0], i_meas=full.i_meas[im0], m_stamp=np.zeros(0), m_sensor=np.zeros(0, np.int32),
                              m_pose=np.zeros((0, 7)), knot_const=kc, truth=None)
    single = runtime.Context(0)
    single.load_window(win)
    ranks = [runtime.Context(0, use_graph=False) for _ in range(N)]
    for r, c in enumerate(ranks):
        c.load_window(win if r == 0 else dataclasses.replace(win, i_stamp=win.i_stamp[:0], i_meas=win.i_meas[:0]))
    red = HostReducer(N)
    calls = [0]
    hook0 = red.hook(0, ranks[0].stream)

    def counted(ptr, count, stream):
        calls[0] += 1
        return hook0(ptr, count, stream)
    ranks[0].set_allreduce(counted)
    for r in range(1, N):
        ranks[r].set_allreduce(red.hook(r, ranks[r].stream))
    slots = [dict() for _ in range(N + 1)]   # caller's landmark id -> slot: ranks, then the single context
    times = dict(sharded=[], single=[])
    rounds, sizes = [], {}

    def stereo(ctx, slot, s, gids, px0, px1):
        n = gids.size
        given = np.array([slot.get(g, -1) for g in gids.tolist()], dtype=np.int32)
        out, _ = ctx.append_stereo_tracks(np.full(n, s), np.zeros(n, np.int32), np.ones(n, np.int32), px0, px1, given)
        for g, l in zip(gids.tolist(), out.tolist()):
            slot[g] = l

    def follow(ctx, slot):
        lmap = ctx.landmark_map()
        return {g: int(lmap[l]) for g, l in slot.items() if lmap[l] >= 0}

    prev_hi = hi0
    for f in range(total):
        hi = st[K0 + f - 1]
        cam_frames = np.unique(tracks["stamp"][(tracks["stamp"] >= prev_hi) & (tracks["stamp"] < hi)])
        ii = (full.i_stamp >= prev_hi) & (full.i_stamp < hi)
        mi = np.flatnonzero((full.m_stamp >= prev_hi) & (full.m_stamp < hi))[:1] if f % 3 == 0 else np.zeros(0, np.int64)
        prev_hi = hi
        lower = st[f + 1] + 1e-9
        imu_rank = f % N

        def rank_frame(r, c):
            c.append_knots(1)
            for s in cam_frames:
                t = tracks["stamp"] == s
                own = (tracks["gid"][t] % N) == r
                stereo(c, slots[r], s, tracks["gid"][t][own], tracks["px0"][t][own], tracks["px1"][t][own])
            if r == imu_rank:
                c.append_inertial_factors(full.i_stamp[ii], full.i_meas[ii])
                c.append_manifold_factors(full.m_stamp[mi], full.m_sensor[mi], full.m_pose[mi])
            stats = c.slide(lower, drop_inertial=True, drop_manifold=True)
            if r == 0:
                rounds.append(calls[0] - before)
            c.iterate(5, records=False)
            c.state()
            return stats

        def single_frame():
            single.append_knots(1)
            for s in cam_frames:
                t = tracks["stamp"] == s
                stereo(single, slots[N], s, tracks["gid"][t], tracks["px0"][t], tracks["px1"][t])
            single.append_inertial_factors(full.i_stamp[ii], full.i_meas[ii])
            single.append_manifold_factors(full.m_stamp[mi], full.m_sensor[mi], full.m_pose[mi])
            stats = single.slide(lower, drop_inertial=True, drop_manifold=True)
            single.iterate(5, records=False)
            single.state()
            return stats

        for name in (("sharded", "single") if f % 2 == 0 else ("single", "sharded")):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            if name == "sharded":
                before = calls[0]
                stats = on_ranks(red, ranks, rank_frame)[0]
            else:
                sstats = single_frame()
            torch.cuda.synchronize()
            if f >= a.warm:
                times[name].append(time.perf_counter() - t0)
        for r in range(N):
            slots[r] = follow(ranks[r], slots[r])
        slots[N] = follow(single, slots[N])
        assert stats["knots"] == sstats["knots"] and sum(c.L for c in ranks) == single.L, (f, stats, sstats)
        sizes = dict(knots=sstats["knots"], landmarks=sstats["landmarks"], bandwidth=single.bandwidth(),
                     bearing_factors_per_rank=[int(c.factor_counts()[runtime.BEARING]) for c in ranks])
    out = dict(tool="sharded_frame_loop", card=card(), world=N, order=k, K0=K0, warm_frames=a.warm, timed_frames=a.frames, window=sizes,
               agreement_rounds_per_frame=statistics.median(rounds[a.warm:]),
               per_frame="append 1 state element + the frame's stereo tracks (2 camera frames) + IMU factors (+ 1 pose factor every 3rd frame), "
               "hb200_slide (both drop flags), 5 LM iterations, state read-back; wall clock",
               note="one GPU: the ranks share device 0 and reduce through the hook; agreement and hook overhead, not scaling",
               nccl="not measured", peer="not measured")
    for name in times:
        out[name] = dict(ms_per_frame_median=statistics.median(times[name]) * 1e3, ms_per_frame_min=min(times[name]) * 1e3)
    print(json.dumps(out))
    for c in ranks + [single]:
        c.close()


if __name__ == "__main__":
    main()
