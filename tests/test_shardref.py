"""Additivity of the normal equations over a landmark-owner partition, on the long-double assembly reference (CPU only).

A sharded iteration sums per-rank partial systems; that sum is the system of the whole window only when every landmark's
observations live on one rank (the Schur complement of a sum is not the sum of the Schur complements).  Here the oracle
evaluates each shard, tests/asmref.py assembles it, and the long-double sum over the shards is compared with the assembly
of the whole window within the sum of their bounds (asmref.compare_shard_sum).  The same comparison rejects a partition
that moves a single observation of one landmark to another rank, so the metric the GPU tests use sees a broken contract.
"""
import numpy as np
import pytest

import asmref as ar
import oracle_lib as ol
from hyperslam_b200 import synthetic

RADIUS = 1e4


def window(order, seed):
    """Pixel, bearing, inertial and pose factors; one constant knot."""
    base = synthetic.make_window(order=order, num_knots=16, num_landmarks=40, num_imu=200, seed=synthetic.SEED_BASE + 800 + seed, constant_knots=1)
    return synthetic.add_bearing_and_pose_factors(base, num_bearing=40, num_pose=10, seed=synthetic.SEED_BASE + 850 + seed)


def reference(win):
    ow = ol.OracleWindow(win, radius=RADIUS)
    assert ow.bad == 0
    return ar.assemble(ar.problem(ow.evaluate(), win, ow.index_maps()), RADIUS)


def by_index(n, world):
    """Rank of each of n factors split into contiguous index ranges, as Window.shard splits them."""
    cuts = [(n * r) // world for r in range(world + 1)]
    return np.searchsorted(cuts, np.arange(n), side="right") - 1


def owner_ranks(win, owner, world):
    """Visual factors follow their landmark's owner; inertial and pose factors are split by index."""
    owner = np.asarray(owner)
    return dict(pixel=owner[win.v_lm], bearing=owner[win.b_lm], inertial=by_index(win.i_stamp.size, world),
                pose=by_index(win.m_stamp.size, world))


@pytest.mark.parametrize("order,world", [(4, 2), (4, 3), (6, 3), (4, 8)])
def test_default_partition_sums_to_the_window(order, world):
    """Window.shard (landmark blocks to ranks) is the owner partition with block owners, and its shard systems add up."""
    win = window(order, order)
    L = win.landmarks.shape[0]
    owner = by_index(L, world)
    shards = [win.shard(r, world) for r in range(world)]
    for a, b in zip(shards, ar.partition(win, owner_ranks(win, owner, world), world)):
        for keys in ar.SHARD_FIELDS.values():
            for key in keys:
                assert np.array_equal(getattr(a, key), getattr(b, key)), key
    res = ar.compare_shard_sum([reference(s) for s in shards], reference(win))
    assert res["nonzero_outside"] == 0 and all(v <= 1.0 for k, v in res.items() if k != "nonzero_outside"), res


def test_scattered_owners_sum_to_the_window():
    """Owners drawn at random over three ranks: every rank's landmarks are scattered over the whole window."""
    win = window(4, 11)
    owner = np.random.default_rng(5).integers(0, 3, win.landmarks.shape[0])
    shards = ar.partition(win, owner_ranks(win, owner, 3), 3)
    res = ar.compare_shard_sum([reference(s) for s in shards], reference(win))
    assert res["nonzero_outside"] == 0 and all(v <= 1.0 for k, v in res.items() if k != "nonzero_outside"), res


@pytest.mark.parametrize("family", ["pixel", "bearing"])
def test_one_observation_on_the_wrong_rank_is_rejected(family):
    """Two ranks; one observation of one landmark is moved to the rank that does not own it.  Its V_l is then split over
    two Schur complements and the summed S and b leave the bound."""
    win = window(4, 12)
    world = 2
    owner = by_index(win.landmarks.shape[0], world)
    ranks = owner_ranks(win, owner, world)
    lm = win.v_lm if family == "pixel" else win.b_lm
    both = win.v_lm.tolist() + win.b_lm.tolist()
    f = next(i for i, l in enumerate(lm) if both.count(l) >= 3)
    ranks[family] = ranks[family].copy()
    ranks[family][f] = 1 - ranks[family][f]
    res = ar.compare_shard_sum([reference(s) for s in ar.partition(win, ranks, world)], reference(win))
    assert res["S"] > 1.0 and res["b"] > 1.0, res
    # what a moved observation does not change: J^T W J's diagonal, g and the cost are sums over factors
    assert res["diagH"] <= 1.0 and res["g"] <= 1.0 and res["cost"] <= 1.0, res
