"""The live frame loop on a sharded window (need an H100): N contexts on device 0, each holding one shard, reduce through
the all-reduce hook (test_gpu_sharded.py's HostReducer) while one context runs the whole sequence alongside.

Routing: stereo tracks go to their landmark's owner (gid mod N unless a case says otherwise) and every rank makes every
collective call -- append_stereo_tracks per camera frame, with n = 0 when it owns none of the frame's tracks, and slide;
append_knots / append_bias_knots are replicated; inertial and pose factors go to one rank per frame (rank-local calls:
a stray collective there would leave the others waiting in the reducer).  After every slide each rank must have the
single context's knots, stamps, constancy, knots_dropped and band half-width; factor counts summed over the ranks and
each owner's landmarks must be the single context's; then two LM iterations on both sides.  The state is carried over
from the single context every frame (sync_state), so the bookkeeping compares bit for bit.
"""
import dataclasses

import numpy as np
import pytest

import asmref as ar
import covref as cr
import sysref as sr
from hyperslam_b200 import runtime, synthetic
from test_gpu_bias_window import BiasHostWindow, start_splines
from test_gpu_covariance import read_system
from test_gpu_sharded import STATE_TOL, check_record, on_ranks, worst
from test_gpu_sharded_covariance import KeepingReducer, same_bits
from test_gpu_stereo_window import StereoHostWindow, error_code, frame_loop_setup

pytestmark = pytest.mark.gpu

K0, WIDTH, ITERS, RADIUS = 14, 9, 2, 1e4
REPLICATED = ("knots", "gyro_bias", "accel_bias", "gravity")


def by_gid(world):
    return lambda gids: np.asarray(gids) % world


def valid_hi(knots, k):
    left = (k - 1) // 2
    return knots[len(knots) - (k - 1 - left) - 1, 7]


def extend_track(full, tracks, extra):
    """The first landmark born stays in view of both cameras for `extra` more camera frames: the window's longest track,
    which later leaves it."""
    g = int(tracks["gid"][0])
    last = tracks["stamp"][tracks["gid"] == g].max()
    t = np.unique(tracks["stamp"])
    t = t[t > last][:extra]
    lm, idx = tracks["landmarks"], np.full(t.size, g)
    px0, p0 = synthetic.pixel_model(full.truth["knots"], full.order, full.cameras, lm, t, np.zeros(t.size, np.int32), idx)
    px1, p1 = synthetic.pixel_model(full.truth["knots"], full.order, full.cameras, lm, t, np.ones(t.size, np.int32), idx)
    assert (p0[:, 2] > 0.5).all() and (p1[:, 2] > 0.5).all()
    out = dict(tracks)
    for key, add in (("stamp", t), ("cam0", np.zeros(t.size, tracks["cam0"].dtype)), ("cam1", np.ones(t.size, tracks["cam1"].dtype)),
                     ("px0", px0), ("px1", px1), ("gid", idx.astype(tracks["gid"].dtype))):
        out[key] = np.concatenate([tracks[key], add])
    o = np.argsort(out["stamp"], kind="stable")
    for key in ("stamp", "cam0", "cam1", "px0", "px1", "gid"):
        out[key] = np.ascontiguousarray(out[key][o])
    return out


class Loop:
    """One sharded frame loop and its single-context twin.  owner(gids) -> rank; imu_rank(frame), pose_rank(frame): the
    rank that receives the frame's inertial / pose factors."""

    def __init__(self, world, order, frames, seed, owner=None, imu_rank=None, pose_rank=None, bias=False, long_track=0, floor=0,
                 deterministic=False):
        self.world, self.order, self.frames, self.bias = world, order, frames, bias
        self.owner = owner or by_gid(world)
        self.imu_rank = imu_rank or (lambda f: f % world)
        self.pose_rank = pose_rank or (lambda f: (f + 1) % world)
        full, hw, hi, tracks = frame_loop_setup(order, K0, frames, seed)
        if bias:   # bias splines that start short and grow with the IMU samples (test_gpu_bias_window.py's loop)
            lo, hi = StereoHostWindow(full, K0).valid_range()
            hw = BiasHostWindow(full, K0, *start_splines(lo, 0.5, 0.6, full))
            hw.knot_const[:2] = 1
        if long_track:
            tracks = extend_track(full, tracks, long_track)
        self.full, self.tracks, self.prev_hi = full, tracks, hi
        win = hw.window()
        self.S = runtime.Context(0)
        self.ctxs = [runtime.Context(0, use_graph=False) for _ in range(world)]
        self.S.load_window(win)
        first = self.imu_rank(-1)
        for r, c in enumerate(self.ctxs):   # the initial inertial factors live on one rank
            c.load_window(win if r == first else dataclasses.replace(win, i_stamp=win.i_stamp[:0], i_meas=win.i_meas[:0]))
        for c in self.all():
            c.set_deterministic(deterministic)
            if floor:
                c.set_min_bandwidth(floor)
        self.red = KeepingReducer(world)
        self.red.attach(self.ctxs)
        self.sids, self.ids = [], [[] for _ in range(world)]   # global landmark id of every slot
        # bearing stamps / landmark ids and pose stamps of every rank's lists (then the single context's), in list order:
        # what asmref needs besides the device's own outputs
        self.lists = [dict(b_stamp=[], b_gid=[], m_stamp=[]) for _ in range(world + 1)]
        if bias:
            im = (full.i_stamp >= lo) & (full.i_stamp < hi)
            self.append_bias(full.i_stamp[im].max())
            self.S.append_inertial_factors(full.i_stamp[im], full.i_meas[im])
            self.ctxs[first].append_inertial_factors(full.i_stamp[im], full.i_meas[im])
        self.betas, self.summed_frames = [], []

    def all(self):
        return [self.S] + self.ctxs

    def close(self):
        for c in self.all():
            c.close()

    def on_ranks(self, fn):
        return on_ranks(self.red, self.ctxs, fn)

    def append_bias(self, t):
        want = self.S.append_bias_knots(t)
        for c in self.ctxs:
            assert c.append_bias_knots(t) == want

    def frame_tracks(self, s):
        t = self.tracks["stamp"] == s
        return [self.tracks[key][t] for key in ("stamp", "cam0", "cam1", "px0", "px1", "gid")]

    def append_frame(self, s, mangle=None, known_only=False):
        """One camera frame: the whole frame on the single context, each owner's tracks on its rank.  mangle(r, args)
        may corrupt a rank's arguments; known_only: only tracks of landmarks already in the window.  Returns each rank's
        error code (0: appended)."""
        stamp, c0, c1, px0, px1, gids = self.frame_tracks(s)
        if known_only:
            t = np.isin(gids, self.sids)
            stamp, c0, c1, px0, px1, gids = (a[t] for a in (stamp, c0, c1, px0, px1, gids))
        own = self.owner(gids)

        def call(r, c):
            m = own == r
            pos = {g: p for p, g in enumerate(self.ids[r])}
            given = np.array([pos.get(g, -1) for g in gids[m].tolist()], dtype=np.int32)
            args = [stamp[m], c0[m].astype(np.int32), c1[m].astype(np.int32), px0[m], px1[m], given]
            if mangle:
                args = mangle(r, args)
            code = error_code(c.append_stereo_tracks, *args)
            if code == 0:
                self.ids[r] += [g for g, v in zip(gids[m].tolist(), given.tolist()) if v < 0]
                self.add_bearings(r, stamp[m], gids[m])
            return code
        codes = self.on_ranks(call)
        if all(code == 0 for code in codes):
            pos = {g: p for p, g in enumerate(self.sids)}
            given = np.array([pos.get(g, -1) for g in gids.tolist()], dtype=np.int32)
            self.S.append_stereo_tracks(stamp, c0.astype(np.int32), c1.astype(np.int32), px0, px1, given)
            self.sids += [g for g, v in zip(gids.tolist(), given.tolist()) if v < 0]
            self.add_bearings(self.world, stamp, gids)
        return codes

    def add_bearings(self, r, stamp, gids):
        self.lists[r]["b_stamp"] += np.repeat(stamp, 2).tolist()   # views 0 and 1 of every track, in track order
        self.lists[r]["b_gid"] += np.repeat(gids, 2).tolist()

    def begin_frame(self, frame):
        for c in self.all():
            c.append_knots(1)
        self.hi = valid_hi(self.S.state()["knots"], self.order)
        full = self.full
        self.ii = (full.i_stamp >= self.prev_hi) & (full.i_stamp < self.hi)
        if self.bias and self.ii.any():   # updateSensor on every rank with the frame's newest IMU stamp
            self.append_bias(full.i_stamp[self.ii].max())
        return np.unique(self.tracks["stamp"][(self.tracks["stamp"] >= self.prev_hi) & (self.tracks["stamp"] < self.hi)])

    def rank_local(self, frame, drop_manifold):
        full, ii = self.full, self.ii
        mi = np.flatnonzero((full.m_stamp >= self.prev_hi) & (full.m_stamp < self.hi))[:1] if frame % 3 == 0 else np.zeros(0, np.int64)
        self.prev_hi = self.hi
        for c in (self.S, self.ctxs[self.imu_rank(frame)]):
            c.append_inertial_factors(full.i_stamp[ii], full.i_meas[ii])
        for c in (self.S, self.ctxs[self.pose_rank(frame)]):
            c.append_manifold_factors(full.m_stamp[mi], full.m_sensor[mi], full.m_pose[mi])
        for r in (self.world, self.pose_rank(frame)):
            self.lists[r]["m_stamp"] += full.m_stamp[mi].tolist()

    def lower(self):
        knots = self.S.state()["knots"]
        return knots[len(knots) - 1 - WIDTH, 7] + 1e-9

    def slide(self, lower, drop_manifold, drop_bias):
        st = self.S.state()["knots"][:, 7]
        last_const = int(np.searchsorted(st, lower, side="right")) - 1
        single = self.S.slide(lower, drop_inertial=True, drop_manifold=drop_manifold, drop_bias=drop_bias)
        smap = self.S.landmark_map()
        self.sids = [g for g, p in zip(self.sids, smap.tolist()) if p >= 0]
        stats = self.on_ranks(lambda r, c: c.slide(lower, drop_inertial=True, drop_manifold=drop_manifold, drop_bias=drop_bias))
        for r, c in enumerate(self.ctxs):
            m = c.landmark_map()
            assert m.size == len(self.ids[r])
            self.ids[r] = [g for g, p in zip(self.ids[r], m.tolist()) if p >= 0]
        k = self.order
        for lists, kept in zip(self.lists, self.ids + [self.sids]):   # the slide rules on the host lists
            kept = set(kept)
            keep = [g in kept for g in lists["b_gid"]]
            lists["b_stamp"] = [t for t, f in zip(lists["b_stamp"], keep) if f]
            lists["b_gid"] = [g for g, f in zip(lists["b_gid"], keep) if f]
            if drop_manifold:
                base = np.searchsorted(st, lists["m_stamp"], side="right") - 1 - (k - 1) // 2
                lists["m_stamp"] = [t for t, b in zip(lists["m_stamp"], base.tolist()) if not b + k - 1 <= last_const]
        return single, stats

    def window_of(self, r, c):
        """The window rank r (self.world: the single context) holds, for asmref: its state and its list stamps."""
        lists, ids = self.lists[r], (self.ids + [self.sids])[r]
        st, pos = c.state(), {g: p for p, g in enumerate(ids)}
        return dataclasses.replace(self.full, knots=st["knots"], gyro_bias=st["gyro_bias"], accel_bias=st["accel_bias"], landmarks=st["landmarks"],
                                   v_stamp=np.zeros(0), v_lm=np.zeros(0, np.int32), b_stamp=np.array(lists["b_stamp"], dtype=np.float64),
                                   b_lm=np.array([pos[g] for g in lists["b_gid"]], dtype=np.int32), m_stamp=np.array(lists["m_stamp"], dtype=np.float64))

    def check_sums(self, frame):
        """The ranks' partial packed systems (captured at the one reduction of hb200_build_system), summed in rank order,
        against the long-double sum of asmref's systems of the ranks' windows -- the whole window's."""
        self.on_ranks(lambda r, c: (c.evaluate(), c.build_system()))
        parts = self.red.captured()
        beta = self.S.bandwidth()
        refs = [ar.assemble(ar.problem(c.outputs(), self.window_of(r, c), c.index_maps()), RADIUS) for r, c in enumerate(self.ctxs)]
        res = ar.compare_summed_buffers(parts, refs, beta)
        assert res["finite"] and res["nonzero_outside"] == 0 and worst(res) <= 1.0, (frame, res)
        tot = parts[0].copy()
        for p in parts[1:]:
            tot += p
        for c in self.ctxs:
            assert same_bits(read_system(c), tot), frame
        self.summed_frames.append(frame)

    def check_window(self, frame, single, stats):
        S = self.S
        beta = S.bandwidth()
        self.betas.append(beta)
        sst = S.state()
        for r, (c, st) in enumerate(zip(self.ctxs, stats)):
            for key in ("knots", "knots_dropped", "knots_constant"):
                assert st[key] == single[key], (frame, r, key, st, single)
            assert (c.K, c.Kbg, c.Kba) == (S.K, S.Kbg, S.Kba), (frame, r)
            assert c.bias_knots() == S.bias_knots(), (frame, r)
            assert c.bandwidth() == beta, (frame, r, c.bandwidth(), beta)
            cst = c.state()
            for key in REPLICATED:
                assert np.array_equal(cst[key], sst[key]), (frame, r, key)
            assert c.L == len(self.ids[r]) and set(self.owner(np.array(self.ids[r], dtype=np.int64))) <= {r}, (frame, r)
        counts = sum(c.factor_counts() for c in self.ctxs)
        assert counts.tolist() == S.factor_counts().tolist(), (frame, counts, S.factor_counts())
        assert sorted(g for ids in self.ids for g in ids) == sorted(self.sids), frame
        lms = self.owner_landmarks()
        assert np.array_equal(lms, sst["landmarks"]), frame

    def owner_landmarks(self):
        """The whole window's landmarks in the single context's slot order, each read from its owner."""
        out = np.full((len(self.sids), 3), np.nan)
        spos = {g: p for p, g in enumerate(self.sids)}
        for c, ids in zip(self.ctxs, self.ids):
            lm = c.state()["landmarks"]
            for p, g in enumerate(ids):
                out[spos[g]] = lm[p]
        return out

    def iterate(self, frame):
        recs = self.on_ranks(lambda r, c: c.iterate(ITERS))
        srecs = self.S.iterate(ITERS)
        states = [c.state() for c in self.ctxs]
        for r in range(1, self.world):
            assert recs[r] == recs[0], (frame, r)
            for key in REPLICATED:
                assert np.array_equal(states[r][key], states[0][key]), (frame, r, key)
        for a, b in zip(recs[0], srecs):
            check_record(a, b)
        sst = self.S.state()
        for key in REPLICATED:
            assert np.abs(states[0][key] - sst[key]).max() <= STATE_TOL, (frame, key)
        if self.sids:
            assert np.abs(self.owner_landmarks() - sst["landmarks"]).max() <= STATE_TOL, frame
        return recs[0]

    def sync_state(self):
        """The single context's state into every context (hb200_optimize with 0 iterations), each rank's own landmarks
        picked from it."""
        s = self.S.state()
        spos = {g: p for p, g in enumerate(self.sids)}
        self.S.optimize(0, s["knots"].copy(), s["gyro_bias"].copy(), s["accel_bias"].copy(), s["gravity"].copy(), s["landmarks"].copy(), records=False)

        def push(r, c):
            lm = np.ascontiguousarray(s["landmarks"][[spos[g] for g in self.ids[r]]].reshape(-1, 3))
            c.optimize(0, s["knots"].copy(), s["gyro_bias"].copy(), s["accel_bias"].copy(), s["gravity"].copy(), lm, records=False)
        self.on_ranks(push)

    def run(self, drop_manifold=True, drop_bias=False, frames=None, every_frame=None, last_known_only=False):
        records, n = [], self.frames if frames is None else frames
        for frame in range(n):
            for s in self.begin_frame(frame):
                assert self.append_frame(s, known_only=last_known_only and frame == n - 1) == [0] * self.world, frame
            self.rank_local(frame, drop_manifold)
            single, stats = self.slide(self.lower(), drop_manifold, drop_bias)
            self.check_window(frame, single, stats)
            if every_frame:
                every_frame(self, frame)
            if frame in (0, n - 1) or self.betas[-1] != self.betas[-2]:   # first, last, and where the band changes
                self.check_sums(frame)
            records.append(self.iterate(frame))
            self.sync_state()
        return records


@pytest.mark.parametrize("world", [2, 3])
def test_frame_loop(built, world):
    loop = Loop(world, 4, 20, synthetic.SEED_BASE + 6100)
    try:
        loop.run()
        counts = [c.factor_counts() for c in loop.ctxs]
        assert all(c[runtime.BEARING] > 0 and c[runtime.INERTIAL] > 0 for c in counts), counts
    finally:
        loop.close()


@pytest.mark.parametrize("owners", ["late", "gap"])
def test_rank_without_factors_of_its_own(built, owners):
    """Rank 1 holds no inertial or pose factor and owns only landmarks born late (the partition one context's slide rule
    drops more knots on: its own smallest base is the newest); "gap": rank 1 also owns early landmarks, so its visual list
    empties and refills, through n = 0 appends."""
    frames = 14
    births = {}

    def owner(gids):
        gids = np.asarray(gids)
        late = gids >= births["late"]
        return (late | (gids < births["early"])).astype(int) if owners == "gap" else late.astype(int)
    loop = Loop(2, 4, frames, synthetic.SEED_BASE + 6200, owner=owner, imu_rank=lambda f: 0, pose_rank=lambda f: 0)
    g = np.unique(loop.tracks["gid"])
    births["late"], births["early"] = int(np.quantile(g, 0.8)), int(np.quantile(g, 0.05))
    empty = []
    try:
        loop.run(every_frame=lambda lp, f: empty.append(lp.ctxs[1].factor_counts()[runtime.BEARING] == 0))
    finally:
        loop.close()
    assert empty[0] if owners == "late" else (not empty[0] and any(empty)), empty
    assert not empty[-1], empty


def test_band_shrinks_on_every_rank(built):
    """A long track on rank 0 widens the band of every rank; when it leaves the window, every rank's band narrows at the
    frame the single context's does.  With a floor, the band never goes below it."""
    loops = []
    try:
        for floor in (0, 6):
            loop = Loop(2, 4, 16, synthetic.SEED_BASE + 6300, long_track=14, floor=floor)
            loops.append(loop)
            loop.run()
        free, floored = loops[0].betas, loops[1].betas
        assert max(free) >= 7 and any(b < a for a, b in zip(free, free[1:])), free
        assert all(b >= 6 for b in floored) and floored == [max(b, 6) for b in free], (free, floored)
    finally:
        for loop in loops:
            loop.close()


def test_bias_drop(built):
    """Order 6, bias splines grown and slid with HB200_SLIDE_DROP_BIAS; rank 1 never holds an inertial factor."""
    loop = Loop(2, 6, 6, synthetic.SEED_BASE + 6400, bias=True, imu_rank=lambda f: 0)
    try:
        dropped = []
        loop.run(drop_bias=True, every_frame=lambda lp, f: dropped.append(lp.S.bias_knots()))
        assert sum(d["gyro_dropped"] + d["accel_dropped"] for d in dropped) > 0, dropped
        assert loop.ctxs[1].factor_counts()[runtime.INERTIAL] == 0
    finally:
        loop.close()


def snapshot(c):
    return c.factor_counts().tolist(), (c.K, c.L, c.Kbg, c.Kba, c.bandwidth()), c.state()


def assert_unchanged(c, before, what):
    counts, sizes, st = before
    assert c.factor_counts().tolist() == counts and (c.K, c.L, c.Kbg, c.Kba, c.bandwidth()) == sizes, what
    now = c.state()
    for key in st:
        assert np.array_equal(now[key], st[key]), (what, key)


@pytest.mark.parametrize("world", [2, 3])
def test_status_and_out_of_step_calls(built, world):
    """An invalid camera index on one rank's stereo append: every rank returns 2 and changes nothing, and the frame then
    goes on.  Different slide flags: -2 everywhere, nothing changed -- on three ranks flags 1, 3, 5, whose sum is three
    times the middle rank's own."""
    loop = Loop(world, 4, 8, synthetic.SEED_BASE + 6500)
    try:
        loop.run(frames=3)
        stamps = loop.begin_frame(3)
        before = [snapshot(c) for c in loop.ctxs]

        def bad_camera(r, args):
            if r == 1 and args[0].size:
                args[1] = args[1].copy()
                args[1][0] = 7
            return args
        s = next(s for s in stamps if (loop.owner(loop.frame_tracks(s)[5]) == 1).any())
        assert loop.append_frame(s, bad_camera) == [2] * world
        for c, b in zip(loop.ctxs, before):
            assert_unchanged(c, b, "status")
        for s in stamps:
            assert loop.append_frame(s) == [0] * world
        loop.rank_local(3, True)
        before = [snapshot(c) for c in loop.ctxs]
        lower = loop.lower()
        if world == 2:
            codes = loop.on_ranks(lambda r, c: error_code(c.slide, lower, True, r == 0, False))
        else:
            codes = loop.on_ranks(lambda r, c: error_code(c.slide, lower, True, r == 1, r == 2))
        assert codes == [-2] * world, codes
        for c, b in zip(loop.ctxs, before):
            assert_unchanged(c, b, "flags")
        single, stats = loop.slide(lower, True, False)
        loop.check_window(3, single, stats)
        loop.iterate(3)
    finally:
        loop.close()


def test_deterministic_reruns(built):
    """Deterministic assembly: two runs of the 2-rank sequence give bit-identical records, states and slot maps."""
    runs = []
    for _ in range(2):
        loop = Loop(2, 4, 8, synthetic.SEED_BASE + 6600, deterministic=True)
        try:
            recs = loop.run()
            runs.append((recs, [c.state() for c in loop.ctxs], [list(ids) for ids in loop.ids]))
        finally:
            loop.close()
    (ra, sa, ia), (rb, sb, ib) = runs
    assert ra == rb and ia == ib
    for a, b in zip(sa, sb):
        for key in a:
            assert np.array_equal(a[key], b[key]), key



def test_covariance_at_the_last_frame(built, record_property):
    """Marginal covariances after the sharded frame loop with growing and sliding bias splines (every bias knot keeps an
    inertial factor; the last frame only continues tracks, so that no landmark is seen by a single stereo pair), the
    state elements then held constant on every rank as in test_gpu_bias_window.py (the newest one, reached only by the
    newest segment's samples, would fail its pivot first): Sigma bit-identical across ranks, the reduced system every
    rank inverted is the rank-order sum of the captured partials, and Sigma is covref's selected inverse of that sum
    within its bound."""
    loop = Loop(2, 4, 10, synthetic.SEED_BASE + 6700, bias=True)
    try:
        loop.run(drop_bias=True, last_known_only=True)
        for c in loop.ctxs:   # replicated: the same constancy on every rank
            c.set_constant(np.ones(c.K, np.uint8), gravity_const=1, bias_const=0)
        infos = loop.on_ranks(lambda r, c: (c.build_covariance(), c.compute_covariance())[1])
        parts = loop.red.captured()
        reduced = [read_system(c) for c in loop.ctxs]
        packed = [c.covariance_packed()[0] if i["status"] == 0 else None for c, i in zip(loop.ctxs, infos)]
        c0 = loop.ctxs[0]
        K, Kbg, Kba, beta = c0.K, c0.Kbg, c0.Kba, c0.bandwidth()
    finally:
        loop.close()
    for r, info in enumerate(infos):
        assert info["status"] == 0 and (info["K"], info["beta"]) == (K, beta), (r, info)
        assert same_bits(packed[r], packed[0]), r
    tot = parts[0].copy()
    for p in parts[1:]:
        tot += p
    assert all(same_bits(x, tot) for x in reduced)
    m = 3 * (Kbg + Kba) + 2
    n = 6 * K + m
    fixed = sr.fixed_mask(K, Kbg, Kba, np.ones(K, np.uint8), 0, 1)
    S_dev, *_ = sr.unpack_system(tot, K, beta, m)
    ref, P, _, bad = cr.selected_inverse(S_dev, K, beta, m, fixed)
    assert bad == -1
    bound = sr.forward_bound(n, cr.kappa(S_dev, fixed))
    err = cr.cov_error(cr.packed_to_dense(packed[0], K, beta, m), ref, P)
    record_property("err_covref", err)
    record_property("bound", bound)
    assert err < bound, (err, bound)
