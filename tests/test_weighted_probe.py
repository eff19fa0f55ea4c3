"""The reference's gradient-probe protocol on weighted costs (CPU).

ExteroceptiveCost::Evaluate with CostConfiguration::weights returns W r and W J (reference exteroceptive.cpp:110-111,
130-133,140-142).  Restated here on the oracle's per-factor Evaluate (cost_evaluate) with W applied in numpy -- what the
device returns with hb200_set_weights, and what weightref assembles -- and probed as the reference's evaluator tests do
(reference tests/include/tests/optimizers/evaluators/evaluator.hpp:26-65): every block non-constant, the analytic
tangent Jacobian W J_b PlusJacobian_b against central differences of W r(x_b (+) delta) through Manifold::Plus, with a
non-symmetric, non-triangular W per family.  The inertial bias blocks of W J are the dense wg[m] W[:, 0:3] /
wa[m] W[:, 3:6] the device's copy-out serves.
"""
import numpy as np
import pytest

import oracle_lib as ol
import weightref as wr
from hyperslam_b200 import runtime
from test_oracle import random_state, sphere_point, unit_quat

H = 1e-6
SAMPLES = 40


def weighted_probe(kind, stamp, meas, params, ids, W, k=4):
    """Worst (relative, normalised absolute) error per block of W J P against central differences of W r."""
    L = ol.layout(kind, k)
    r, J = ol.cost_evaluate(kind, stamp, meas, params, k=k)
    worst = []
    for b, mid in enumerate(ids):
        o, s = int(L["offsets"][b]), int(L["sizes"][b])
        x = params[o:o + s].copy()
        P = ol.manifold_plus_jacobian(mid, x)
        Ja = W @ J[b] @ P
        Jn = np.zeros_like(Ja)
        for c in range(P.shape[1]):
            rs = []
            for sgn in (1.0, -1.0):
                d = np.zeros(P.shape[1])
                d[c] = sgn * H
                q = params.copy()
                q[o:o + s] = ol.manifold_plus(mid, x, d)
                rs.append(W @ ol.cost_evaluate(kind, stamp, meas, q, k=k, jac=False)[0])
            Jn[:, c] = (rs[0] - rs[1]) / (2 * H)
        ae = np.abs(Ja - Jn)
        den = np.maximum(np.abs(Ja), np.abs(Jn))
        rel = np.where((Ja == 0) | (Jn == 0), ae, ae / np.where(den > 0, den, 1.0))
        na, nn = np.linalg.norm(Ja), np.linalg.norm(Jn)
        nabs = np.abs(Ja / na - Jn / nn) if na > 0 and nn > 0 else ae
        worst.append((float(rel.max()), float(nabs.max())))
    return r, J, worst


def failed(worst, tol=1e-5):
    return any(rel > tol and nabs > tol for rel, nabs in worst)


def test_weighted_pixel_and_bearing_probe():
    rng = np.random.default_rng(7100)
    W = wr.all_weights(seed=71)
    ids = [ol.M_STATE] * 4 + [ol.M_SE3, ol.M_EUCLIDEAN, ol.M_EUCLIDEAN, ol.M_EUCLIDEAN]
    fails = {ol.PIXEL: 0, ol.BEARING: 0}
    for _ in range(SAMPLES):
        cps, stamp = random_state(rng, 4)
        T_bs = np.concatenate([unit_quat(rng), rng.uniform(-1, 1, 3)])
        intr = np.array([367.215, 248.375, 458.654, 457.296])
        dist = np.array([-0.28340811, 0.07395907, 1.76187114e-05, 0.00019359])
        params = np.concatenate([cps.ravel(), T_bs, intr, dist, sphere_point(rng, 10.0)])
        _, _, w = weighted_probe(ol.PIXEL, stamp, rng.uniform(-1, 1, 2), params, ids, W[runtime.PIXEL])
        fails[ol.PIXEL] += failed(w)
        _, _, w = weighted_probe(ol.BEARING, stamp, sphere_point(rng, 1.0), params, ids, W[runtime.BEARING])
        fails[ol.BEARING] += failed(w)
    # as in the unweighted protocol: a landmark near the camera plane occasionally defeats h = 1e-6 differences
    assert fails[ol.PIXEL] <= 1 and fails[ol.BEARING] == 0, fails


def test_weighted_inertial_probe_and_dense_bias_blocks():
    rng = np.random.default_rng(7200)
    W = wr.all_weights(seed=72)[runtime.INERTIAL]
    k, kb = 4, 4
    ids = [ol.M_STATE] * k + [ol.M_SE3] + [ol.M_EUCLIDEAN] * 4 + [ol.M_BIAS] * (2 * kb) + [ol.M_SPHERE]
    n_fail = 0
    for _ in range(SAMPLES):
        cps, stamp = random_state(rng, k)
        T_bs = np.concatenate([unit_quat(rng), rng.uniform(-1, 1, 3)])
        ig = np.array([1, 1, 1, 0, 0, 0.0]) + rng.uniform(-0.1, 0.1, 6)
        ia = np.array([1, 1, 1, 0, 0, 0.0]) + rng.uniform(-0.1, 0.1, 6)

        def bias():
            b = np.zeros((kb, 4))
            b[:, :3] = rng.uniform(-1, 1, (kb, 3))
            b[:, 3] = stamp - 0.4 * 10.0 + (np.arange(kb) - 1) * 10.0
            return b
        params = np.concatenate([cps.ravel(), T_bs, ig, ia, rng.uniform(-0.01, 0.01, 9), rng.uniform(-0.05, 0.05, 9),
                                 bias().ravel(), bias().ravel(), sphere_point(rng, 9.81)])
        _, J, w = weighted_probe(ol.INERTIAL, stamp, rng.uniform(-1, 1, 6), params, ids, W)
        n_fail += failed(w)
        for m in range(kb):
            g, a = J[k + 5 + m], J[k + 5 + kb + m]
            wg, wa = g[0, 0], a[3, 0]
            want_g, want_a = np.zeros((6, 4)), np.zeros((6, 4))
            want_g[:, :3], want_a[:, :3] = wg * W[:, 0:3], wa * W[:, 3:6]
            assert np.array_equal(W @ g, want_g) and np.array_equal(W @ a, want_a)
    assert n_fail == 0, n_fail


def test_weighted_manifold_probe():
    rng = np.random.default_rng(7300)
    W = wr.all_weights(seed=73)[runtime.MANIFOLD]
    ids = [ol.M_STATE] * 4 + [ol.M_SE3]
    n_fail = 0
    for _ in range(SAMPLES):
        cps, stamp = random_state(rng, 4)
        T_bs = np.concatenate([unit_quat(rng), rng.uniform(-1, 1, 3)])
        element = np.concatenate([unit_quat(rng), rng.uniform(-1, 1, 3)])
        _, _, w = weighted_probe(ol.MANIFOLD, stamp, element, np.concatenate([cps.ravel(), T_bs]), ids, W)
        n_fail += failed(w)
    # rotation differences near pi put Log at its branch cut (as in the unweighted protocol)
    assert n_fail <= 1, n_fail
