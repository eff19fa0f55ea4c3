"""Worker for tests/test_gpu_multi_window.py: the live frame loop on a window sharded over the ranks of torch.distributed
(one GPU each) in one reduction mode.  Stereo tracks go to their landmark's owner (gid mod world; every rank makes every
append_stereo_tracks call, n = 0 included), IMU and pose factors to one rank per frame, every rank slides and iterates.
Rank 0 runs one context on the whole window alongside.  After every slide: K, knots_dropped and beta equal on every rank
and equal to the single context's, landmark and bearing counts summing to its own; then two LM iterations, records
identical across ranks and within tests/multi_gpu_worker.py's tolerances of the single context's; the single context's
state is then carried to every rank.  One JSON line."""
import dataclasses
import json
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
from hyperslam_b200 import runtime, synthetic  # noqa: E402
from multi_gpu_covariance_worker import connect  # noqa: E402
from test_gpu_stereo_window import frame_loop_setup  # noqa: E402

COST_TOL, COST_NEW_TOL = 1e-7, 1e-6
K0, WIDTH, FRAMES = 14, 9, 16


def valid_hi(knots, k):
    left = (k - 1) // 2
    return knots[len(knots) - (k - 1 - left) - 1, 7]


def gather(obj, world):
    out = [None] * world
    dist.all_gather_object(out, obj)
    return out


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    mode = sys.argv[1]
    if mode != "peer":
        os.environ["HB200_PEER_REDUCE"] = "0"
    order = 4
    full, hw, prev_hi, tracks = frame_loop_setup(order, K0, FRAMES, synthetic.SEED_BASE + 6900)
    win = hw.window()
    ctx = runtime.Context(local, use_graph=(mode != "callback"))
    ctx.load_window(win if rank == 0 else dataclasses.replace(win, i_stamp=win.i_stamp[:0], i_meas=win.i_meas[:0]))
    comm = connect(ctx, mode, local)
    if mode == "callback":
        ctx.set_min_bandwidth(0)   # no iteration before the first collective call: let the band follow the agreement
    single = runtime.Context(local) if rank == 0 else None
    if single:
        single.load_window(win)
    ids, sids, msg = [], [], []
    for frame in range(FRAMES):
        ctx.append_knots(1)
        if single:
            single.append_knots(1)
        hi = valid_hi(ctx.state()["knots"], order)
        for s in np.unique(tracks["stamp"][(tracks["stamp"] >= prev_hi) & (tracks["stamp"] < hi)]):
            t = tracks["stamp"] == s
            gids, px0, px1 = tracks["gid"][t], tracks["px0"][t], tracks["px1"][t]
            for c, lst, m in ((ctx, ids, gids % world == rank), (single, sids, np.ones(gids.size, bool))):
                if c is None:
                    continue
                pos = {g: p for p, g in enumerate(lst)}
                given = np.array([pos.get(g, -1) for g in gids[m].tolist()], dtype=np.int32)
                n = int(m.sum())
                c.append_stereo_tracks(np.full(n, s), np.zeros(n, np.int32), np.ones(n, np.int32), px0[m], px1[m], given)
                lst += [g for g, v in zip(gids[m].tolist(), given.tolist()) if v < 0]
        ii = (full.i_stamp >= prev_hi) & (full.i_stamp < hi)
        mi = np.flatnonzero((full.m_stamp >= prev_hi) & (full.m_stamp < hi))[:1] if frame % 3 == 0 else np.zeros(0, np.int64)
        prev_hi = hi
        for c in ([ctx] if frame % world == rank else []) + ([single] if single else []):
            c.append_inertial_factors(full.i_stamp[ii], full.i_meas[ii])
            c.append_manifold_factors(full.m_stamp[mi], full.m_sensor[mi], full.m_pose[mi])
        knots = ctx.state()["knots"]
        lower = knots[len(knots) - 1 - WIDTH, 7] + 1e-9
        stats = ctx.slide(lower, drop_inertial=True, drop_manifold=True)
        lmap = ctx.landmark_map()
        ids = [g for g, p in zip(ids, lmap.tolist()) if p >= 0]
        mine = (ctx.K, stats["knots_dropped"], stats["knots_constant"], ctx.bandwidth(), ctx.L, int(ctx.factor_counts()[runtime.BEARING]))
        allr = gather(mine, world)
        if single:
            sst = single.slide(lower, drop_inertial=True, drop_manifold=True)
            smap = single.landmark_map()
            sids = [g for g, p in zip(sids, smap.tolist()) if p >= 0]
            want = (single.K, sst["knots_dropped"], sst["knots_constant"], single.bandwidth())
            if any(a[:4] != want for a in allr):
                msg.append(f"frame {frame}: ranks {allr} vs single {want}")
            if (sum(a[4] for a in allr), sum(a[5] for a in allr)) != (single.L, int(single.factor_counts()[runtime.BEARING])):
                msg.append(f"frame {frame}: counts {allr} vs single L {single.L}")
        recs = ctx.iterate(2)
        allrec = gather([(x["cost"], x["cost_new"], x["accepted"]) for x in recs], world)
        if any(a != allrec[0] for a in allrec):
            msg.append(f"frame {frame}: records differ between ranks")
        if single:
            for a, b in zip(recs, single.iterate(2)):
                if not (abs(a["cost"] - b["cost"]) <= COST_TOL * b["cost"] and abs(a["cost_new"] - b["cost_new"]) <= COST_NEW_TOL * abs(b["cost_new"])
                        and a["accepted"] == b["accepted"] and a["spd"] == 1):
                    msg.append(f"frame {frame}: {a} vs single {b}")
        # the single context's state to every rank, each rank's own landmarks picked by id
        box = [None]
        if single:
            s = single.state()
            box = [dict(s, ids=list(sids))]
        dist.broadcast_object_list(box, src=0)
        s = box[0]
        spos = {g: p for p, g in enumerate(s["ids"])}
        if single:
            single.optimize(0, s["knots"].copy(), s["gyro_bias"].copy(), s["accel_bias"].copy(), s["gravity"].copy(), s["landmarks"].copy(), records=False)
        lm = np.ascontiguousarray(s["landmarks"][[spos[g] for g in ids]].reshape(-1, 3))
        ctx.optimize(0, s["knots"].copy(), s["gyro_bias"].copy(), s["accel_bias"].copy(), s["gravity"].copy(), lm, records=False)
    flag = torch.tensor([0.0 if msg else 1.0], device="cuda")
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    if rank == 0:
        print(json.dumps(dict(ok=bool(flag.item() == 1.0), msg="; ".join(msg)[:2000], world=world, mode=mode,
                              comm=ctx.comm_info() if mode != "callback" else comm, frames=FRAMES)))
    ctx.close()
    if single:
        single.close()
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
