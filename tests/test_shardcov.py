"""Marginal covariances of a landmark-owner partition on the long-double references (CPU only).

A sharded hb200_build_covariance sums the ranks' undamped partial systems (mu = 0) and every rank inverts the sum; the
landmark marginals come from each landmark's owner, from its own factors and the summed Sigma.  Here the oracle evaluates
each shard, tests/asmref.py assembles it at mu = 0, the shards are summed in long double, and tests/covref.py checks:
* the selected inverse of the sum equals that of the whole-window assembly within sysref.forward_bound(n, kappa);
* the landmark marginals from each owner's own problem and the summed Sigma equal the whole window's, and a rank's
  non-owned landmarks (held but not observed) get zero blocks;
* a partition that moves one observation to a rank that does not own the landmark is rejected: the receiving rank's V_l
  is rank-deficient (a degenerate landmark there, so status 2 on every rank), and with that term left out the summed
  Sigma leaves the bound.
"""
import numpy as np
import pytest

import asmref as ar
import covref as cr
import oracle_lib as ol
import sysref as sr
from hyperslam_b200 import synthetic
from test_gpu_sharded import shard_by_owner


def window(order, seed):
    """Pixel, bearing, inertial and pose factors; the first `order` knots and the untouched ones constant (gauge)."""
    base = synthetic.make_window(order=order, num_knots=14, num_landmarks=36, num_imu=160, seed=synthetic.SEED_BASE + 3100 + seed)
    win = synthetic.add_bearing_and_pose_factors(base, num_bearing=30, num_pose=8, seed=synthetic.SEED_BASE + 3150 + seed)
    win.knot_const = np.zeros(win.knots.shape[0], np.uint8)
    win.knot_const[:order] = 1
    win.knot_const[cr.untouched_knots(win)] = 1
    return win


def problem(win):
    ow = ol.OracleWindow(win)
    assert ow.bad == 0
    return ar.problem(ow.evaluate(), win, ow.index_maps())


def shape(win):
    K, Kbg, Kba = win.knots.shape[0], win.gyro_bias.shape[0], win.accel_bias.shape[0]
    m = 3 * (Kbg + Kba) + 2
    return K, m, 6 * K + m, sr.fixed_mask(K, Kbg, Kba, win.knot_const, win.bias_const, win.gravity_const)


def whole(win):
    """(problem, Sigma, pattern, beta, bound) of the whole window at mu = 0."""
    K, m, n, fixed = shape(win)
    p = problem(win)
    S = ar.assemble(p, np.inf)["S"]
    beta = sr.block_bandwidth(S.astype(np.float64), K)
    Sig, P, _, bad = cr.selected_inverse(S, K, beta, m, fixed)
    assert bad == -1
    return p, Sig, P, beta, sr.forward_bound(n, cr.kappa(S, fixed))


def summed_sigma(win, shards, beta, skip=None):
    """Problems of the shards and the selected inverse of the long-double sum of their mu = 0 assemblies.
    skip: {rank: local landmarks whose Schur term that rank leaves out}."""
    K, m, _, fixed = shape(win)
    probs = [problem(s) for s in shards]
    S = sum(ar.assemble(p, np.inf, skip_landmarks=(skip or {}).get(r, ()))["S"] for r, p in enumerate(probs))
    Sig, _, _, bad = cr.selected_inverse(S, K, beta, m, fixed)
    assert bad == -1
    return probs, Sig


CASES = [(4, 2, "scattered", False), (4, 3, "scattered", True), (6, 2, "blocks", True), (6, 3, "scattered", False)]


@pytest.mark.parametrize("order,world,owners,compact", CASES, ids=[f"k{o}-n{w}-{s}{'-compact' if c else ''}" for o, w, s, c in CASES])
def test_owner_partition_gives_the_window_covariance(order, world, owners, compact):
    win = window(order, order + world)
    L = win.landmarks.shape[0]
    owner = (np.random.default_rng(3100 + world).integers(0, world, L) if owners == "scattered"
             else np.searchsorted([(L * r) // world for r in range(world + 1)], np.arange(L), side="right") - 1)
    p_full, ref, P, beta, bound = whole(win)
    shards, index = shard_by_owner(win, owner, world, compact=compact)
    probs, got = summed_sigma(win, shards, beta)
    err = cr.cov_error(got, ref, P)
    print(f"order {order}, {world} ranks ({owners}, compact {compact}): Sigma err {err:.3e} / bound {bound:.3e}")
    assert err < bound, (err, bound)
    # landmark blocks from their owners: each rank's own problem with the summed Sigma
    lm_ref = cr.landmark_marginals(p_full, ref)
    lm = np.full((L, 3, 3), np.nan, np.longdouble)
    for r, p in enumerate(probs):
        mine = owner[index[r]] == r
        blocks = cr.landmark_marginals(p, got)
        assert np.all(blocks[~mine] == 0), r          # held, not observed: zero block
        lm[index[r][mine]] = blocks[mine]
    assert not np.isnan(lm.astype(np.float64)).any()
    seen = np.abs(lm_ref).reshape(L, -1).max(1) > 0
    errs = [cr.cov_error(lm[l], lm_ref[l]) for l in np.nonzero(seen)[0]]
    assert max(errs) < 10 * bound, (max(errs), bound)
    assert np.all(lm[~seen] == 0)


def test_one_observation_on_the_wrong_rank_is_rejected():
    """One pixel observation of a landmark seen at least three times moves to the other rank.  That rank's V_l comes from
    one pixel factor (rank 2): a degenerate landmark there.  Leaving its Schur term out, the summed Sigma is far off."""
    win = window(4, 40)
    world = 2
    L = win.landmarks.shape[0]
    owner = np.searchsorted([0, L // 2, L], np.arange(L), side="right") - 1
    _, ref, P, beta, bound = whole(win)
    counts = np.bincount(win.v_lm, minlength=L) + np.bincount(win.b_lm, minlength=L)
    f = next(i for i, l in enumerate(win.v_lm) if counts[l] >= 3)
    lm = int(win.v_lm[f])
    ranks = dict(pixel=owner[win.v_lm].copy(), bearing=owner[win.b_lm], inertial=np.zeros(win.i_stamp.size, int),
                 pose=np.zeros(win.m_stamp.size, int))
    ranks["pixel"][f] = 1 - owner[lm]
    shards = ar.partition(win, ranks, world)
    recv = 1 - owner[lm]
    p = problem(shards[recv])
    V = cr._landmark_terms(p)[lm][1].astype(np.float64)
    ev = np.linalg.eigvalsh(V)
    assert ev[0] <= 1e-10 * ev[-1], ev                 # rank-deficient: cov_landmark_flags_kernel counts it
    _, got = summed_sigma(win, shards, beta, skip={recv: [lm]})
    err = cr.cov_error(got, ref, P)
    print(f"moved observation: Sigma err {err:.3e} / bound {bound:.3e}")
    assert err > 100 * bound, (err, bound)
