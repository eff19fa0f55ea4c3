"""Worker for tests/test_gpu_deterministic.py's two-GPU case: every rank runs LM iterations on its factor shard with the
deterministic assembly, the partial systems reduced through peer memory (peer_reduce_kernel, rank order) inside the
iteration's CUDA graph.  Rank 0 prints one JSON line: the records and the raw bytes of every rank's state (hex), so that
two runs can be compared bit for bit."""
import json
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from hyperslam_b200 import runtime, synthetic  # noqa: E402


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    win = synthetic.make_window(order=4, num_knots=20, num_landmarks=160, num_imu=400, seed=synthetic.SEED_BASE + 700, constant_knots=2)
    ctx = runtime.Context(local, use_graph=True)
    ctx.set_deterministic(True)
    ctx.load_window(win.shard(rank, world))
    ctx.connect_torch_distributed(dist, peer_mailbox=True)
    recs = ctx.iterate(4)
    state = ctx.state()
    blob = "".join(state[k].tobytes().hex() for k in sorted(state))
    states = [None] * world
    dist.all_gather_object(states, blob)
    info = ctx.comm_info()
    if rank == 0:
        print(json.dumps(dict(records=recs, states=states, comm=info, deterministic=ctx.deterministic())))
    ctx.close()
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
