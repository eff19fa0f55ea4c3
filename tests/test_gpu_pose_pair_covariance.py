"""Joint and relative covariance of the poses at two stamps on the device (need an H100):
hb200_set_covariance_stamp_pairs / hb200_get_pose_pair_covariance against tests/posepairref.py.

* joint and relative equal posepairref on covref.dense_inverse_ld of the device's own undamped system within
  sysref.forward_bound(n, kappa) (the joint in covref's correlation metric, the relative normalised by |A| sqrt(diag joint)
  since it is a difference of the joint's blocks); the largest normalised reference entry among the pairs more than
  beta apart is >= 1e3 x the bound, so a march that returned zeros fails;
* the diagonal blocks are bit-identical to hb200_interpolate_covariance (the same Jacobian builder and the same sums,
  term for term; their correlation-metric distance is recorded); (t_b, t_a) is exactly
  the permutation of (t_a, t_b); both blocks are exactly symmetric; constant knots give zero rows; an out-of-span stamp
  gives status 1 and zero blocks; a non-finite stamp is refused at registration;
* launches: stamp pairs alone add the span kernel, one far-column launch and the pair kernel; block requests registered
  beside pairs are bit-identical to the same requests alone, as are Sigma and the landmark marginals (deterministic mode);
* snapshot: iterations, a slide, a failed compute and a registration without a compute leave the results bit for bit;
* deterministic mode: two computes are bit-identical; sharded on one GPU (2 contexts, the all-reduce callback): the
  results are bit-identical across ranks and match the dense inverse of the rank-order sum.
"""
import numpy as np
import pytest

import covref as cr
import posepairref as pp
import sysref as sr
from hyperslam_b200 import runtime
from test_gpu_covariance import e2e_window, failure_window, gauge_free_window, read_system
from test_gpu_cross_covariance import requests
from test_gpu_sharded import HostReducer, on_ranks, open_ranks, shard_by_owner

pytestmark = pytest.mark.gpu


def same_bits(a, b):
    return np.array_equal(np.asarray(a, np.float64).view(np.int64), np.asarray(b, np.float64).view(np.int64))


def valid_span(knots, order):
    kt, left = knots[:, 7], (order - 1) // 2
    return kt[left], kt[len(kt) - order + left + 1]


def stamp_pairs(knots, order, n, seed):
    """n pairs spread over the valid span (many far apart), the same pairs swapped, a same-stamp pair, one pair with a
    stamp in the first segment (constant knots), and one pair with an out-of-span stamp (last)."""
    lo, hi = valid_span(knots, order)
    rng = np.random.default_rng(seed)
    ab = rng.uniform(lo, hi, (n, 2))
    ab[: n // 4, 1] = np.clip(ab[: n // 4, 0] + rng.uniform(-0.05, 0.05, n // 4), lo, np.nextafter(hi, -np.inf))   # close pairs
    kt = knots[:, 7]
    first = kt[(order - 1) // 2] + 0.3 * (kt[(order - 1) // 2 + 1] - kt[(order - 1) // 2])
    extra = [(ab[0, 0], ab[0, 0]), (first, 0.5 * (lo + hi)), (np.nextafter(hi, -np.inf), lo), (0.5 * (lo + hi), hi)]
    return np.concatenate([ab, ab[:, ::-1], np.array(extra)])


def run(ctx, pairs, blocks=None):
    """register, build, read the system, compute; (system, launches, joint, relative, status)."""
    ctx.set_covariance_stamp_pairs(pairs)
    if blocks is not None:
        ctx.set_covariance_blocks(blocks)
    ctx.build_covariance()
    buf = read_system(ctx)
    l0 = ctx.launch_count
    info = ctx.compute_covariance()
    launches = ctx.launch_count - l0
    assert info["status"] == 0, info
    joint, rel, st = ctx.pose_pair_covariance()
    return buf, launches, joint, rel, st


CASES = {"k4-cfg1": (4, 50), "k6-cfg1": (6, 50)}


@pytest.mark.parametrize("case", list(CASES))
def test_against_reference(built, record_property, case):
    order, K = CASES[case]
    win = e2e_window(order, num_knots=K, seed=80 + order + K)
    Kbg, Kba = win.gyro_bias.shape[0], win.accel_bias.shape[0]
    m = 3 * (Kbg + Kba) + 2
    n = 6 * K + m
    npair = 60
    pairs = stamp_pairs(win.knots, order, npair, seed=order)
    ctx = runtime.Context(0)
    try:
        ctx.load_window(win)
        beta = ctx.bandwidth()
        buf, launches, joint, rel, st = run(ctx, pairs)
        knots = ctx.state()["knots"]
        pose, bad = ctx.interpolate_covariance(pairs.ravel())
        with pytest.raises(runtime.HB200Error, match="hb200 error -1"):
            ctx.set_covariance_stamp_pairs([(0.5, np.nan)])
        with pytest.raises(runtime.HB200Error, match="hb200 error -1"):
            ctx.set_covariance_stamp_pairs([(np.inf, 0.5)])
    finally:
        ctx.close()
    # selected inverse, landmark marginals, stamp spans, far columns, pairs
    assert launches == 5, launches
    fixed = sr.fixed_mask(K, Kbg, Kba, win.knot_const, win.bias_const, win.gravity_const)
    S_dev, *_ = sr.unpack_system(buf, K, beta, m)
    Sig = cr.dense_inverse_ld(S_dev, fixed)
    bound = sr.forward_bound(n, cr.kappa(S_dev, fixed))
    pose = pose.reshape(-1, 2, 6, 6)
    assert list(st[:-1]) == [0] * (len(pairs) - 1) and st[-1] == 1
    assert np.all(joint[-1] == 0) and np.all(rel[-1] == 0)
    err_joint = err_rel = err_diag = biggest = 0.0
    for q in range(len(pairs) - 1):
        ta, tb = pairs[q]
        assert np.array_equal(joint[q], joint[q].T) and np.array_equal(rel[q], rel[q].T), q
        want, want_rel = pp.pose_pair(knots, order, ta, tb, Sig)
        err_joint = max(err_joint, cr.cov_error(joint[q], want))
        _, Ra, pa = pp.pose_value(knots, order, ta)
        _, _, pb = pp.pose_value(knots, order, tb)
        s = np.abs(np.asarray(pp.relative_jacobian(Ra, pa, pb), np.float64)) @ np.sqrt(np.abs(np.diagonal(want)).astype(np.float64))
        ok = np.outer(s, s) > 0
        if ok.any():
            err_rel = max(err_rel, float((np.abs(np.asarray(rel[q] - want_rel, np.float64))[ok] / np.outer(s, s)[ok]).max()))
        err_diag = max(err_diag, cr.cov_error(joint[q][:6, :6], pose[q, 0]), cr.cov_error(joint[q][6:, 6:], pose[q, 1]))
        assert same_bits(joint[q][:6, :6], pose[q, 0]) and same_bits(joint[q][6:, 6:], pose[q, 1]), q
        ba, bb = pp.pose_value(knots, order, ta)[0], pp.pose_value(knots, order, tb)[0]
        if abs(ba - bb) + order - 1 > beta:   # the off-diagonal block reads far columns
            dg = np.sqrt(np.abs(np.diagonal(want)).astype(np.float64))
            nz = np.outer(dg[:6], dg[6:]) > 0
            if nz.any():
                biggest = max(biggest, float((np.abs(np.asarray(want[:6, 6:], np.float64))[nz] / np.outer(dg[:6], dg[6:])[nz]).max()))
    # swapped pairs: exact permutations
    perm = np.r_[6:12, 0:6]
    for q in range(npair):
        assert same_bits(joint[npair + q], joint[q][np.ix_(perm, perm)]), q
    # a same-stamp pair: off-diagonal blocks equal the diagonal ones, relative zero to rounding
    same = 2 * npair
    assert same_bits(joint[same][:6, 6:], joint[same][:6, :6]) and same_bits(joint[same][6:, 6:], joint[same][:6, :6])
    assert np.abs(rel[same]).max() <= 1e-14 * np.abs(joint[same]).max()
    # a stamp in the first segment: every control point constant, zero rows and columns where Sigma is zero
    assert np.all(joint[same + 1][:6] == 0) and np.all(joint[same + 1][:, :6] == 0) and np.abs(joint[same + 1][6:, 6:]).max() > 0
    for k, v in dict(n=n, beta=beta, bound=bound, err_joint=err_joint, err_relative=err_rel, err_diag=err_diag, largest_reference=biggest).items():
        record_property(k, v)
    print(f"{case}: beta {beta}, joint err {err_joint:.3e}, relative err {err_rel:.3e}, diag err {err_diag:.3e}, bound {bound:.3e}, largest {biggest:.3e}")
    assert err_joint < bound, (err_joint, bound)
    assert err_rel < bound, (err_rel, bound)
    assert biggest >= 1e3 * bound, (biggest, bound)


def test_blocks_beside_pairs_unchanged(built):
    """Deterministic mode: block requests, Sigma and the landmark marginals are bit-identical with and without stamp
    pairs registered beside them; launch counts without a list, with pairs alone, with both."""
    win = e2e_window(4, num_knots=30, num_landmarks=300, num_imu=800, bearing=100, pose=10, seed=91)
    K, L = 30, win.landmarks.shape[0]
    pairs = stamp_pairs(win.knots, 4, 20, seed=91)

    def once(with_pairs, with_blocks):
        ctx = runtime.Context(0)
        try:
            ctx.set_deterministic(True)
            ctx.load_window(win)
            req = requests(K, win.gyro_bias.shape[0], win.accel_bias.shape[0], L, ctx.bandwidth(), np.random.default_rng(91), n_lm=20)
            _, launches, joint, rel, st = run(ctx, pairs if with_pairs else np.zeros((0, 2)), req if with_blocks else np.zeros((0, 4)))
            packed, lm, _ = ctx.covariance_packed()
            blocks, bst = ctx.covariance_blocks()
        finally:
            ctx.close()
        return launches, packed, lm, blocks, bst, joint, rel, st

    none, pairs_only, blocks_only, both = once(False, False), once(True, False), once(False, True), once(True, True)
    assert none[0] == 2 and pairs_only[0] == 5 and blocks_only[0] == 5 and both[0] == 7, (none[0], pairs_only[0], blocks_only[0], both[0])
    for a, b in ((none, pairs_only), (blocks_only, both), (none, blocks_only)):
        assert same_bits(a[1], b[1]) and same_bits(a[2], b[2])
    assert same_bits(blocks_only[3], both[3]) and np.array_equal(blocks_only[4], both[4])
    assert same_bits(pairs_only[5], both[5]) and same_bits(pairs_only[6], both[6]) and np.array_equal(pairs_only[7], both[7])


def test_snapshot_and_refusals(built):
    win = failure_window()
    kt = win.knots[:, 7]
    pairs = stamp_pairs(win.knots, 4, 10, seed=5)
    ctx = runtime.Context(0)
    try:
        ctx.set_deterministic(True)
        with pytest.raises(runtime.HB200Error, match="hb200 error -2"):
            ctx.pose_pair_covariance()                       # before any compute
        ctx.load_window(win)
        lib, h = ctx.lib, ctx.h
        t = runtime._d(np.array([0.5, 0.6]))
        assert lib.hb200_set_covariance_stamp_pairs(h, -1, t) == -1
        assert lib.hb200_set_covariance_stamp_pairs(h, 1, None) == -1
        assert lib.hb200_set_covariance_stamp_pairs(h, 0, None) == 0
        _, _, joint, rel, st = run(ctx, pairs)

        def same(what):
            j, r, s = ctx.pose_pair_covariance()
            assert same_bits(j, joint) and same_bits(r, rel) and np.array_equal(s, st), what
        ctx.iterate(2)
        same("iterate")
        ctx.set_covariance_stamp_pairs(pairs[:3])         # registered, not computed
        same("registration")
        with pytest.raises(runtime.HB200Error, match="hb200 error -1"):
            ctx.set_covariance_stamp_pairs([(0.5, np.nan)])
        assert lib.hb200_get_pose_pair_covariance(h, 3, None, None, None) == -2
        assert lib.hb200_get_pose_pair_covariance(h, len(pairs), None, None, None) == 0
        ctx.slide(kt[8], drop_inertial=True)
        same("slide")
        ctx.load_window(gauge_free_window())
        ctx.set_covariance_stamp_pairs(pairs[:4])
        ctx.build_covariance()
        assert ctx.compute_covariance()["status"] == 1
        same("failed compute")
    finally:
        ctx.close()


def test_deterministic_repeat(built):
    win = e2e_window(6, num_knots=30, num_landmarks=300, num_imu=800, bearing=100, pose=10, seed=92)
    pairs = stamp_pairs(win.knots, 6, 30, seed=92)
    ctx = runtime.Context(0)
    try:
        ctx.set_deterministic(True)
        ctx.load_window(win)
        first = run(ctx, pairs)
        second = run(ctx, pairs)
    finally:
        ctx.close()
    assert same_bits(first[0], second[0])
    assert same_bits(first[2], second[2]) and same_bits(first[3], second[3]) and np.array_equal(first[4], second[4])


def test_sharded(built, record_property):
    world = 2
    win = e2e_window(4, num_knots=30, num_landmarks=300, num_imu=800, bearing=150, pose=10, seed=93)
    K, Kbg, Kba, L = 30, win.gyro_bias.shape[0], win.accel_bias.shape[0], win.landmarks.shape[0]
    m = 3 * (Kbg + Kba) + 2
    n = 6 * K + m
    owner = np.random.default_rng(93).integers(0, world, L)
    shards, _ = shard_by_owner(win, owner, world)
    pairs = stamp_pairs(win.knots, 4, 20, seed=93)
    ctxs, _, beta = open_ranks(shards)
    try:
        red = HostReducer(world)
        red.attach(ctxs)
        res = on_ranks(red, ctxs, lambda r, c: (c.set_covariance_stamp_pairs(pairs), c.build_covariance(), c.compute_covariance())[2])
        assert all(i["status"] == 0 for i in res), res
        got = [c.pose_pair_covariance() for c in ctxs]
        bufs = [read_system(c) for c in ctxs]
        knots = ctxs[0].state()["knots"]
    finally:
        for c in ctxs:
            c.close()
    for r in range(1, world):
        assert all(same_bits(a, b) for a, b in zip(got[r][:2], got[0][:2])) and np.array_equal(got[r][2], got[0][2])
    assert same_bits(bufs[0], bufs[1])
    S_dev, *_ = sr.unpack_system(bufs[0], K, beta, m)
    fixed = sr.fixed_mask(K, Kbg, Kba, win.knot_const, win.bias_const, win.gravity_const)
    Sig = cr.dense_inverse_ld(S_dev, fixed)
    bound = sr.forward_bound(n, cr.kappa(S_dev, fixed))
    joint, _, st = got[0]
    err = 0.0
    for q, (ta, tb) in enumerate(pairs):
        want, _ = pp.pose_pair(knots, 4, ta, tb, Sig)
        if want is None:
            assert st[q] == 1
            continue
        err = max(err, cr.cov_error(joint[q], want))
    record_property("err_joint", err)
    assert err < bound, (err, bound)
