"""The agreement of a sharded window's sliding calls (tests/shardwindow.py) against the whole-window rule, on the CPU.

Host windows of the live frame loop (StereoHostWindow of test_gpu_stereo_window.py, BiasHostWindow of
test_gpu_bias_window.py) are split over ranks at random every frame -- landmarks by owner, inertial and pose factors
anywhere -- and each rank votes with what it alone keeps.  The summed votes must give the knot shift, the bias shifts
and the band half-width the whole window's rule gives, with empty ranks, ranks holding a single family, and ranks whose
own smallest base would drop more knots than the window may."""
import copy

import numpy as np
import pytest

import shardwindow as sw
from hyperslam_b200 import synthetic
from test_bias_extension import bias_base
from test_gpu_bias_window import KB, BiasHostWindow, start_splines
from test_gpu_stereo_window import StereoHostWindow, frame_loop_setup

K0, WIDTH = 14, 9
SLIDE = 4   # call kind of hb200_slide in the header


def rank_lists(hw, part, r):
    """Rank r's share of the window: its visual factors (bases, gids, stamps), inertial stamps and bases, pose bases."""
    vis = part["owner"][hw.b["gid"]] == r
    return dict(v_base=hw.base_of(hw.b["stamp"][vis]), v_gid=hw.b["gid"][vis], v_stamp=hw.b["stamp"][vis],
                i_stamp=hw.i["stamp"][part["imu"] == r], m_base=hw.base_of(hw.m["stamp"][part["pose"] == r]))


def rank_votes(hw, part, r, lower, drop_manifold, drop_bias):
    """What rank r keeps of its own share under the slide rules and the minima it votes with."""
    own = rank_lists(hw, part, r)
    k = hw.k
    ub = int(np.searchsorted(hw.knots[:, 7], lower, side="right"))
    last = {}
    for g, t in zip(own["v_gid"].tolist(), own["v_stamp"].tolist()):
        last[g] = max(last.get(g, -np.inf), t)
    v_keep = np.array([last[g] >= lower for g in own["v_gid"].tolist()], dtype=bool)
    i_base = hw.base_of(own["i_stamp"])
    i_keep = ~(i_base + k - 1 <= ub - 1)
    m_keep = ~(own["m_base"] + k - 1 <= ub - 1) if drop_manifold else np.ones(own["m_base"].size, dtype=bool)
    mins = [int(b[m].min()) for b, m in ((own["v_base"], v_keep), (i_base, i_keep), (own["m_base"], m_keep)) if m.any()]
    bias = (None, None)
    if drop_bias and i_keep.any():
        kept = own["i_stamp"][i_keep]
        bias = (int(bias_base(hw.bg[:, 3], kept).min()), int(bias_base(hw.ba[:, 3], kept).min()))
    return (min(mins) if mins else None), bias


def header(hw, lower, flags):
    ub = [int(np.searchsorted(s, lower, side="right")) for s in (hw.knots[:, 7], hw.bg[:, 3], hw.ba[:, 3])]
    return [1, len(hw.knots), len(hw.bg), len(hw.ba), SLIDE, flags] + ub


def agreed_slide(hw, part, world, lower, drop_manifold, drop_bias):
    K, Kbg, Kba, k = len(hw.knots), len(hw.bg), len(hw.ba), hw.k
    flags = 1 | (2 if drop_manifold else 0) | (4 if drop_bias else 0)
    h = header(hw, lower, flags)
    votes = [rank_votes(hw, part, r, lower, drop_manifold, drop_bias) for r in range(world)]
    a = sw.agree(sw.summed([sw.payload(K, Kbg, Kba, h, knot_min=m, bias_min=b) for m, b in votes]), K, Kbg, Kba, h)
    assert not a["mismatch"] and a["status"] == 0
    ub = h[6]
    begin = max(0, ub - 1 - (k - 1) // 2)
    shift = sw.knot_shift(begin, a["knot_min"], K, k)
    bias = (sw.bias_shift(hw.bg[:, 3], lower, a["gyro_min"], KB), sw.bias_shift(hw.ba[:, 3], lower, a["accel_min"], KB)) if drop_bias else (0, 0)
    greedy = [sw.knot_shift(begin, sw.NO_VOTE if m is None else m, K, k) for m, _ in votes]   # each rank's own rule
    return shift, bias, greedy


def agreed_beta(hw, part, world):
    K, Kbg, Kba, k = len(hw.knots), len(hw.bg), len(hw.ba), hw.k
    h = [1, K, Kbg, Kba, SLIDE, 0, 0, 0, 0]
    pays = []
    for r in range(world):
        own = rank_lists(hw, part, r)
        lm = {}
        for g, b in zip(own["v_gid"].tolist(), own["v_base"].tolist()):
            lm.setdefault(g, []).append(b)
        pays.append(sw.payload(K, Kbg, Kba, h, beta=sw.own_beta(k, lm)))
    return max(k - 1, sw.agree(sw.summed(pays), K, Kbg, Kba, h)["beta"])


def whole_beta(hw):
    lm = {}
    for g, b in zip(hw.b["gid"].tolist(), hw.base_of(hw.b["stamp"]).tolist()):
        lm.setdefault(g, []).append(b)
    return max(hw.k - 1, sw.own_beta(hw.k, lm) or 0)


def partitions(rng, hw, world, G):
    """A random owner partition, one with an empty last rank, one whose last rank holds only pose factors."""
    Ni, Nm = hw.i["stamp"].size, hw.m["stamp"].size
    out = [dict(owner=rng.integers(0, world, G), imu=rng.integers(0, world, Ni), pose=rng.integers(0, world, Nm))]
    out.append(dict(owner=rng.integers(0, world - 1, G), imu=rng.integers(0, world - 1, Ni), pose=rng.integers(0, world - 1, Nm)))
    out.append(dict(owner=rng.integers(0, world - 1, G), imu=rng.integers(0, world - 1, Ni), pose=np.full(Nm, world - 1)))
    return out


def frame_loop(order, frames, seed, bias):
    """The host window of the live frame loop, frame by frame, just before each slide (bearings are not needed here)."""
    full, _, _, tracks = frame_loop_setup(order, K0, frames, seed)
    lo, hi = StereoHostWindow(full, K0).valid_range()
    # bias: splines that start short, grow with the IMU samples and slide; else the template's, which never move
    hw = BiasHostWindow(full, K0, *(start_splines(lo, 0.5, 0.6, full) if bias else (full.gyro_bias, full.accel_bias)))
    im = (full.i_stamp >= lo) & (full.i_stamp < hi)
    if bias:
        hw.append_bias(full.i_stamp[im].max())
    hw.add_lists(i=dict(stamp=full.i_stamp[im], meas=full.i_meas[im]))
    prev = hi
    for frame in range(frames):
        hw.append_knot()
        _, hi = hw.valid_range()
        ii = (full.i_stamp >= prev) & (full.i_stamp < hi)
        if bias and ii.any():
            hw.append_bias(full.i_stamp[ii].max())
        for s in np.unique(tracks["stamp"][(tracks["stamp"] >= prev) & (tracks["stamp"] < hi)]):
            gids = tracks["gid"][tracks["stamp"] == s]
            new = [g for g in gids.tolist() if g not in set(hw.lm_ids)]
            hw.add_landmarks(new, np.zeros((len(new), 3)))
            n = gids.size
            hw.add_lists(b=dict(stamp=np.full(2 * n, s), cam=np.tile([0, 1], n), gid=np.repeat(gids, 2), bearing=np.zeros((2 * n, 3))))
        mi = np.flatnonzero((full.m_stamp >= prev) & (full.m_stamp < hi))[:1] if frame % 3 == 0 else np.zeros(0, np.int64)
        hw.add_lists(i=dict(stamp=full.i_stamp[ii], meas=full.i_meas[ii]), m=dict(stamp=full.m_stamp[mi], sensor=full.m_sensor[mi], pose=full.m_pose[mi]))
        prev = hi
        yield hw, hw.knots[len(hw.knots) - 1 - WIDTH, 7] + 1e-9, int(tracks["gid"].max()) + 1


@pytest.mark.parametrize("order,frames,bias,world", [(4, 20, False, 2), (4, 20, False, 3), (6, 8, True, 2), (4, 12, True, 3)])
def test_agreed_shifts_and_band_are_the_whole_window_rule(order, frames, bias, world):
    rng = np.random.default_rng(7000 + 10 * order + world)
    drop_manifold = True
    greedy_seen = False
    for hw, lower, G in frame_loop(order, frames, synthetic.SEED_BASE + 7000 + order, bias):
        parts = partitions(rng, hw, world, G)
        results = [agreed_slide(hw, p, world, lower, drop_manifold, bias) for p in parts]
        ref = copy.deepcopy(hw)
        dropped, _ = ref.slide(lower, drop_inertial=True, drop_manifold=drop_manifold, drop_bias=bias)
        for shift, bshift, greedy in results:
            assert shift == dropped["knots"] and bshift == ref.bias_dropped, (shift, bshift, dropped, ref.bias_dropped)
            greedy_seen |= max(greedy) > shift
        hw.slide(lower, drop_inertial=True, drop_manifold=drop_manifold, drop_bias=bias)
        for p in partitions(rng, hw, world, G):
            assert agreed_beta(hw, p, world) == whole_beta(hw)
    assert greedy_seen   # some rank's own smallest base alone would have dropped more knots


def test_header_and_status():
    K, Kbg, Kba = 6, 4, 5
    h = [1, K, Kbg, Kba, SLIDE, 1, 3, 1, 1]
    ok = [sw.payload(K, Kbg, Kba, h, knot_min=m) for m in (2, None, 4)]
    a = sw.agree(sw.summed(ok), K, Kbg, Kba, h)
    assert (a["mismatch"], a["status"], a["knot_min"], a["gyro_min"], a["beta"]) == (False, 0, 2, sw.NO_VOTE, 0)
    other = list(h)
    other[5] = 3   # different slide flags on one rank
    a = sw.agree(sw.summed(ok[:2] + [sw.payload(K, Kbg, Kba, other)]), K, Kbg, Kba, h)
    assert a["mismatch"]
    # symmetric differences on three ranks: flags 1, 3, 5 sum to 3 x 3, yet the rank holding 3 must see them too
    for field, values in ((5, (1, 3, 5)), (6, (2, 3, 4)), (1, (5, 6, 7)), (4, (3, 4, 5))):
        heads = []
        for v in values:
            x = list(h)
            x[field] = v
            heads.append(x)
        total = sw.summed([sw.payload(K, Kbg, Kba, x) for x in heads])
        assert all(sw.agree(total, K, Kbg, Kba, x)["mismatch"] for x in heads), (field, values)
    total = sw.summed([sw.payload(K, Kbg, Kba, h) for _ in range(3)])
    assert not sw.agree(total, K, Kbg, Kba, h)["mismatch"]
    statuses = [(0, 0), (0, 2), (1, 1)]   # passed, arrival order, bad index and order
    a = sw.agree(sw.summed([sw.payload(K, Kbg, Kba, h, status=s) for s in statuses]), K, Kbg, Kba, h)
    assert a["status"] == 2
    a = sw.agree(sw.summed([sw.payload(K, Kbg, Kba, h, status=s) for s in statuses[:2]]), K, Kbg, Kba, h)
    assert a["status"] == 3
    a = sw.agree(sw.summed([sw.payload(K, Kbg, Kba, h, beta=b) for b in (3, 5, None)]), K, Kbg, Kba, h)
    assert a["beta"] == 5
