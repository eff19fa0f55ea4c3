"""The sharded frame loop on two GPUs in every reduction mode (peer memory, NCCL with and without the peer mailbox, the
callback hook over torch.distributed): the agreement rounds of the collective sliding-window calls run through
ncclAllReduce (or the hook), and K, knots_dropped, beta and the counts follow one context on the whole window
(tests/multi_gpu_window_worker.py).  Needs >= 2 GPUs, skipped otherwise."""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("mode", ["peer", "nccl+mailbox", "nccl", "callback"])
def test_two_rank_frame_loop(built, mode):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29561", os.path.join(ROOT, "tests", "multi_gpu_window_worker.py"), mode]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]
    out = json.loads([l for l in res.stdout.splitlines() if l.startswith("{")][-1])
    assert out["ok"], out
    if mode != "callback":
        assert out["comm"]["nccl"] and out["comm"]["peer_reduce"] == (mode == "peer"), out
