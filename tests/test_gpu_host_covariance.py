"""GPU test of hyper::Covariance (hyperslam_b200/host), driven by the C++ binary hyperslam_b200/lib/covariance_test.

The binary builds the hyper:: object graph of a window, checks that Compute refuses pairs outside the computed pattern
(state elements beta + 1 apart, a landmark with a state element, two landmarks, an unknown block) and that a pair not
computed is not served, then writes the ambient and Ceres-tangent blocks of a set of pairs.  Here they are compared with
the device covariance of the same window through the C-ABI, converted with tests/covref.py and the oracle's
manifold_plus_jacobian:
* tangent blocks: T S T^T, T = diag(1/2 I3, I3) on state elements (Ceres' quaternion tangent), identity elsewhere;
* ambient blocks: P_a (T S T^T) P_b^T with the oracle's PlusJacobian of each block, and exactly the host's own tangent
  block mapped through it.
"""
import os
import subprocess

import numpy as np
import pytest

import covref as cr
import oracle_lib as ol
from hyperslam_b200 import runtime, synthetic

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def dump_window(win, path):
    """The window format of host_test, followed by one constancy flag per state element."""
    with open(path, "w") as f:
        w = lambda a: f.write(" ".join(repr(float(x)) for x in np.asarray(a).ravel()) + "\n")
        f.write(f"{win.order} {win.knots.shape[0]} {win.gyro_bias.shape[0]} {win.cameras.shape[0]} {win.landmarks.shape[0]} "
                f"{win.v_stamp.size} {win.i_stamp.size} 0 {win.b_stamp.size} {win.m_stamp.size} {win.pose_sensors.shape[0]}\n")
        w(win.knots); w(win.gyro_bias); w(win.accel_bias); w(win.gravity); w(win.cameras); w(win.imu); w(win.landmarks)
        for i in range(win.v_stamp.size):
            f.write(f"{float(win.v_stamp[i])!r} {int(win.v_cam[i])} {int(win.v_lm[i])} {float(win.v_pixel[i, 0])!r} {float(win.v_pixel[i, 1])!r}\n")
        for i in range(win.i_stamp.size):
            f.write(f"{float(win.i_stamp[i])!r} " + " ".join(repr(float(x)) for x in win.i_meas[i]) + "\n")
        for i in range(win.b_stamp.size):
            f.write(f"{float(win.b_stamp[i])!r} {int(win.b_cam[i])} {int(win.b_lm[i])} " + " ".join(repr(float(x)) for x in win.b_bearing[i]) + "\n")
        w(win.pose_sensors) if win.pose_sensors.size else None
        for i in range(win.m_stamp.size):
            f.write(f"{float(win.m_stamp[i])!r} {int(win.m_sensor[i])} " + " ".join(repr(float(x)) for x in win.m_pose[i]) + "\n")
        f.write(" ".join(str(int(c)) for c in win.knot_const) + "\n")


@pytest.mark.parametrize("order", [4, 6])
def test_host_covariance(built, tmp_path, record_property, order):
    exe = os.path.join(ROOT, "hyperslam_b200", "lib", "covariance_test")
    assert os.path.exists(exe), "covariance_test not built (python -c 'import __graft_entry__ as g; g.build()')"
    base = synthetic.make_window(order=order, num_knots=20, num_landmarks=60, num_imu=400, seed=synthetic.SEED_BASE + 2400 + order)
    win = synthetic.add_bearing_and_pose_factors(base, num_bearing=20, num_pose=8, seed=synthetic.SEED_BASE + 2450 + order)
    win.knot_const = np.zeros(20, np.uint8)
    win.knot_const[:order] = 1
    win.knot_const[cr.untouched_knots(win)] = 1
    win.bias_const, win.gravity_const = 0, 0
    src, dst = tmp_path / "window.txt", tmp_path / "out.txt"
    dump_window(win, src)
    res = subprocess.run([exe, str(src), str(dst)], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stdout + res.stderr
    it = iter(open(dst).read().split("\n"))
    head = next(it).split()
    assert head[0] == "refused" and head[1] == head[2]
    beta = int(head[4])
    comp = next(it).split()
    assert comp[:3] == ["compute", "1", "0"]

    # the same window through the C-ABI
    ctx = runtime.Context(0)
    try:
        ctx.load_window(win)
        assert ctx.bandwidth() == beta
        ctx.build_covariance()
        assert ctx.compute_covariance()["status"] == 0
        packed, lm, (K, b, m, L) = ctx.covariance_packed()
    finally:
        ctx.close()
    Sig = cr.packed_to_dense(packed, K, b, m)
    Kbg, Kba = win.gyro_bias.shape[0], win.accel_bias.shape[0]

    def block(kind, j):
        if kind == "state":
            return np.arange(6 * j, 6 * j + 6), np.diag([0.5, 0.5, 0.5, 1, 1, 1]), ol.manifold_plus_jacobian(ol.M_STATE, win.knots[j])
        if kind == "gyro":
            return 6 * K + 3 * j + np.arange(3), np.eye(3), ol.manifold_plus_jacobian(ol.M_BIAS, win.gyro_bias[j])
        if kind == "accel":
            return 6 * K + 3 * Kbg + 3 * j + np.arange(3), np.eye(3), ol.manifold_plus_jacobian(ol.M_BIAS, win.accel_bias[j])
        if kind == "gravity":
            return 6 * K + 3 * (Kbg + Kba) + np.arange(2), np.eye(2), ol.manifold_plus_jacobian(ol.M_SPHERE, win.gravity)
        return None, np.eye(3), ol.manifold_plus_jacobian(ol.M_EUCLIDEAN, win.landmarks[j])

    npairs, worst_t, worst_a, worst_map = 0, 0.0, 0.0, 0.0
    line = next(it)
    while line.startswith("pair"):
        _, ka, ja, kb, jb = line.split()
        ja, jb = int(ja), int(jb)
        tan = np.array(next(it).split(), dtype=float)
        amb = np.array(next(it).split(), dtype=float)
        ra, Ta, Pa = block(ka, ja)
        rb, Tb, Pb = block(kb, jb)
        if ka == "landmark":
            D, da, db = lm[ja], np.abs(np.diag(lm[ja])), np.abs(np.diag(lm[jb]))
        else:
            D, da, db = Sig[np.ix_(ra, rb)], np.abs(np.diag(Sig)[ra]), np.abs(np.diag(Sig)[rb])
        want_t = Ta @ D @ Tb.T
        tan = tan.reshape(want_t.shape)
        amb = amb.reshape(Pa.shape[0], Pb.shape[0])
        scale_t = np.sqrt(np.outer(np.diag(Ta) ** 2 * da, np.diag(Tb) ** 2 * db))
        worst_t = max(worst_t, float((np.abs(tan - want_t) / np.where(scale_t > 0, scale_t, 1)).max()))
        want_a = Pa @ want_t @ Pb.T
        worst_a = max(worst_a, float(np.abs(amb - want_a).max() / max(np.abs(want_a).max(), 1e-300)))
        own = Pa @ tan @ Pb.T   # the host's ambient block is its own tangent block through the PlusJacobians
        worst_map = max(worst_map, float(np.abs(amb - own).max() / max(np.abs(own).max(), 1e-300)))
        npairs += 1
        line = next(it)
    assert npairs == 9
    assert line.split() == ["failures", "0"]
    record_property("beta", beta)
    record_property("tangent_err", worst_t)
    record_property("ambient_err", worst_a)
    record_property("ambient_map_err", worst_map)
    # two computes of the same window differ only by the assembly's floating-point atomics
    assert worst_t < 1e-8 and worst_a < 1e-8, (worst_t, worst_a)
    assert worst_map < 1e-12, worst_map
