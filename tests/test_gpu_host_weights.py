"""GPU test of Optimizer::setWeights (hyperslam_b200/host), driven by the C++ binary hyperslam_b200/lib/weights_test: with a
matrix set for every family, ExteroceptiveCost::Evaluate returns W r and W J (calibration blocks included, the inertial
bias blocks dense), the reference's Probe protocol passes on the weighted costs, and clearing the matrices restores the
unweighted outputs bit for bit."""
import os
import subprocess

import numpy as np
import pytest

import weightref as wr
from hyperslam_b200 import synthetic
from test_gpu_host import dump_window

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("order", [4, 6])
def test_cpp_set_weights(built, tmp_path, order):
    exe = os.path.join(ROOT, "hyperslam_b200", "lib", "weights_test")
    assert os.path.exists(exe), "weights_test not built (python -c 'import __graft_entry__ as g; g.build()')"
    win = synthetic.make_window(order=order, num_knots=14, num_landmarks=30, num_imu=40, seed=synthetic.SEED_BASE + 540 + order, constant_knots=2)
    win = synthetic.add_bearing_and_pose_factors(win, num_bearing=40, num_pose=12, seed=synthetic.SEED_BASE + 560 + order)
    src, wts = tmp_path / "window.txt", tmp_path / "weights.txt"
    dump_window(win, src, 2)
    W = wr.all_weights(seed=order)
    with open(wts, "w") as f:
        for kind in range(4):   # ExteroceptiveCost::Kind order == runtime.PIXEL, INERTIAL, BEARING, MANIFOLD
            f.write(" ".join(repr(float(x)) for x in np.asarray(W[kind]).ravel()) + "\n")
    res = subprocess.run([exe, str(src), str(wts)], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stdout + res.stderr
    assert "failures 0" in res.stdout and "cleared mismatches 0" in res.stdout, res.stdout
