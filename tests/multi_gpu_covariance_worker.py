"""Worker for tests/test_gpu_multi_covariance.py: every rank holds a landmark-block shard of one window, computes the
marginal covariances collectively (one system reduction in the given mode), then runs iterate(2) -> covariance ->
iterate(2) and, after a restore, iterate(4).  Rank 0 compares with one context on the whole window; one JSON line."""
import json
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import covref as cr  # noqa: E402
import sysref as sr  # noqa: E402
from hyperslam_b200 import runtime  # noqa: E402
from test_gpu_covariance import e2e_window, read_system  # noqa: E402

COST_TOL, COST_NEW_TOL, STATE_TOL = 1e-7, 1e-6, 1e-6   # the tolerances of tests/multi_gpu_worker.py


def connect(ctx, mode, local):
    if mode != "callback":
        return ctx.connect_torch_distributed(dist, peer_mailbox=(mode in ("peer", "nccl+mailbox")))
    ext = torch.cuda.ExternalStream(ctx.stream, device=torch.device("cuda", local))
    cache = {}

    def allreduce(ptr, count, stream):
        if (ptr, count) not in cache:
            class _Arr:
                __cuda_array_interface__ = dict(shape=(count,), typestr="<f8", data=(ptr, False), version=2)
            cache[(ptr, count)] = torch.as_tensor(_Arr(), device=torch.device("cuda", local))
        with torch.cuda.stream(ext):
            dist.all_reduce(cache[(ptr, count)])
        return 0

    ctx.set_allreduce(allreduce)
    beta = torch.tensor([ctx.bandwidth()], device="cuda")
    dist.all_reduce(beta, op=dist.ReduceOp.MAX)
    ctx.set_min_bandwidth(int(beta.item()))
    return {}


def covariance(ctx):
    ctx.build_covariance()
    sysbuf = read_system(ctx)
    info = ctx.compute_covariance()
    packed, lm, _ = ctx.covariance_packed() if info["status"] == 0 else (None, None, None)
    return info, sysbuf, packed, lm


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    mode = sys.argv[1]
    if mode != "peer":
        os.environ["HB200_PEER_REDUCE"] = "0"
    win = e2e_window(4, num_knots=30, num_landmarks=300, num_imu=800, bearing=150, pose=10, seed=81)
    L = win.landmarks.shape[0]
    owner = np.searchsorted([(L * r) // world for r in range(world + 1)], np.arange(L), side="right") - 1
    ctx = runtime.Context(local, use_graph=(mode != "callback"))
    ctx.load_window(win.shard(rank, world))
    comm = connect(ctx, mode, local)
    msg = []

    # 1. covariance at the initial state
    info, sysbuf, packed, lm = covariance(ctx)
    if info["status"] != 0:
        msg.append(f"rank {rank}: status {info}")
    else:
        gathered = [torch.zeros(packed.size, dtype=torch.float64, device="cuda") for _ in range(world)]
        dist.all_gather(gathered, torch.from_numpy(packed).cuda())
        identical = all(torch.equal(g, gathered[0]) for g in gathered)
        if not identical:
            msg.append("Sigma differs between ranks")
        lm[owner != rank] = np.where(lm[owner != rank] == 0, 0.0, np.nan)   # non-owned blocks must be exactly 0
        lm_sum = torch.from_numpy(lm).cuda()
        dist.all_reduce(lm_sum)
        lm_owned = lm_sum.cpu().numpy()
    res = dict(identical=info["status"] == 0 and identical)
    if rank == 0 and info["status"] == 0:
        single = runtime.Context(local)
        single.load_window(win)
        beta = ctx.bandwidth()
        single.set_min_bandwidth(beta)
        s_info, s_sys, s_packed, s_lm = covariance(single)
        single.close()
        K, Kbg, Kba = win.knots.shape[0], win.gyro_bias.shape[0], win.accel_bias.shape[0]
        m = 3 * (Kbg + Kba) + 2
        n = 6 * K + m
        fixed = sr.fixed_mask(K, Kbg, Kba, win.knot_const, win.bias_const, win.gravity_const)
        S_dev, *_ = sr.unpack_system(sysbuf, K, beta, m)
        S_one, *_ = sr.unpack_system(s_sys, K, beta, m)
        ref, P, _, _ = cr.selected_inverse(S_dev, K, beta, m, fixed)
        kap = cr.kappa(S_dev, fixed)
        got = cr.packed_to_dense(packed, K, beta, m)
        one = cr.packed_to_dense(s_packed, K, beta, m)
        keep = ~fixed
        eS = sr.entry_error(S_dev[np.ix_(keep, keep)], S_one[np.ix_(keep, keep)])
        bound, bound_one = sr.forward_bound(n, kap), kap * (n * eS + 8 * n * sr.EPS)
        seen = np.abs(s_lm).reshape(L, -1).max(1) > 0
        err_lm = max(cr.cov_error(lm_owned[l], s_lm[l]) for l in np.nonzero(seen)[0])
        res.update(err_own=cr.cov_error(got, ref, P), bound_own=bound, err_single=cr.cov_error(got, one, P), bound_single=bound_one,
                   err_landmarks=err_lm, landmarks_finite=bool(np.isfinite(lm_owned).all()), single_status=s_info["status"])

    # 2. iterate(2) -> covariance -> iterate(2) against iterate(4) from the same snapshot
    ctx.snapshot()
    recs = ctx.iterate(2)
    info2, *_ = covariance(ctx)
    recs += ctx.iterate(2)
    graph_after = ctx.comm_info()["graph"] if mode != "callback" else False
    state_a = ctx.state()
    ctx.restore()
    plain = ctx.iterate(4)
    state_b = ctx.state()
    for it, (a, b) in enumerate(zip(recs, plain)):
        if not (abs(a["cost"] - b["cost"]) <= COST_TOL * b["cost"] and abs(a["cost_new"] - b["cost_new"]) <= COST_NEW_TOL * abs(b["cost_new"])
                and a["accepted"] == b["accepted"] and a["spd"] == b["spd"] == 1):
            msg.append(f"rank {rank} iteration {it}: {a} vs {b}")
    for key in ("knots", "gyro_bias", "accel_bias", "gravity"):
        if np.abs(state_a[key] - state_b[key]).max() > STATE_TOL:
            msg.append(f"rank {rank}: {key} differs after the covariance")
    res.update(status_between=info2["status"], graph_after=graph_after)
    flag = torch.tensor([0.0 if msg else 1.0], device="cuda")
    dist.all_reduce(flag, op=dist.ReduceOp.MIN)
    if rank == 0:
        print(json.dumps(dict(ok=bool(flag.item() == 1.0), msg="; ".join(msg), world=world, mode=mode,
                              comm=ctx.comm_info() if mode != "callback" else comm, **res)))
    ctx.close()
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
