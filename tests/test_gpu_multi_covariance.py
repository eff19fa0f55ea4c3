"""Marginal covariances on two GPUs in every reduction mode (peer memory, NCCL with and without the peer mailbox, the
callback hook over torch.distributed); needs >= 2 GPUs, skipped otherwise.  Sigma is identical on both ranks, matches
covref's selected inverse of the reduced system and one context on the whole window, the owners' landmark blocks match
that context's, non-owned blocks are 0, and iterate(2) -> covariance -> iterate(2) matches iterate(4) (in the graph modes
still as a CUDA graph)."""
import json
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("mode", ["peer", "nccl+mailbox", "nccl", "callback"])
def test_two_rank_covariance(built, record_property, mode):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29541", os.path.join(ROOT, "tests", "multi_gpu_covariance_worker.py"), mode]
    res = subprocess.run(cmd, capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]
    out = json.loads([l for l in res.stdout.splitlines() if l.startswith("{")][-1])
    for k in ("err_own", "bound_own", "err_single", "bound_single", "err_landmarks"):
        record_property(k, out.get(k))
    assert out["ok"] and out["identical"], out
    assert out["single_status"] == 0 and out["status_between"] == 0, out
    assert out["err_own"] < out["bound_own"] and out["err_single"] < out["bound_single"], out
    assert out["landmarks_finite"] and out["err_landmarks"] < 10 * out["bound_single"], out
    if mode != "callback":
        assert out["comm"]["nccl"] and out["graph_after"], out
        assert out["comm"]["peer_reduce"] == (mode == "peer"), out
