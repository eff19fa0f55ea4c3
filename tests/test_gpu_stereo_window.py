"""The reference's live frame loop on the device-side window: stereo tracks become bearing factors and new landmarks
(AbstractOptimizer::process(VisualTracks), reference internal/hyper/optimizers/abstract.cpp:243-260), pose measurements
become manifold factors (:266-270), IMU samples inertial factors, and the window slides -- all without a re-bind.

Two contexts run the same sequence: A through hb200_append_stereo_tracks, B through the composed path
(hb200_ingest_stereo -> host -> hb200_append_landmarks + hb200_append_bearing_factors).  Per frame the bookkeeping is
checked against a host restatement of the rules (HostWindow of test_gpu_sliding.py with bearing and manifold lists),
the two contexts against each other bit for bit, new landmarks / bearings against the oracle's ingest, and residuals,
Jacobians, LM records and state against an oracle window built from the host lists.
"""
import dataclasses

import numpy as np
import pytest

import oracle_lib as ol
from hyperslam_b200 import runtime, synthetic
from test_gpu_sliding import HostWindow, rel_err

pytestmark = pytest.mark.gpu


class StereoHostWindow(HostWindow):
    """HostWindow plus the bearing (visual list, kind 1) and manifold lists and the landmark map of a slide."""

    def __init__(self, full, K0):
        super().__init__(full, K0)
        self.b = dict(stamp=np.zeros(0), cam=np.zeros(0, np.int32), gid=np.zeros(0, np.int64), bearing=np.zeros((0, 3)))
        self.m = dict(stamp=np.zeros(0), sensor=np.zeros(0, np.int32), pose=np.zeros((0, 7)))

    @staticmethod
    def _cat(lists, new):
        for key in lists:
            lists[key] = np.concatenate([lists[key], np.asarray(new[key], dtype=lists[key].dtype).reshape((-1,) + lists[key].shape[1:])])

    def add_landmarks(self, gids, xyz):
        self.lm_ids += list(gids)
        self.lm_xyz = np.vstack([self.lm_xyz, np.asarray(xyz).reshape(-1, 3)])

    def add_lists(self, b=None, i=None, m=None):
        for lists, new in ((self.b, b), (self.i, i), (self.m, m)):
            if new is not None:
                self._cat(lists, new)

    def slide(self, lower, drop_inertial=True, drop_manifold=False):
        st = self.knots[:, 7]
        ub = int(np.searchsorted(st, lower, side="right"))
        begin, last_const = max(0, ub - 1 - (self.k - 1) // 2), ub - 1
        last = {}
        for g, t in zip(self.v["gid"].tolist() + self.b["gid"].tolist(), self.v["stamp"].tolist() + self.b["stamp"].tolist()):
            last[g] = max(last.get(g, -np.inf), t)
        keep_set = {g for g in self.lm_ids if g not in last or last[g] >= lower}
        vm = np.array([g in keep_set for g in self.v["gid"].tolist()], dtype=bool)
        bm = np.array([g in keep_set for g in self.b["gid"].tolist()], dtype=bool)
        ib, mb = self.base_of(self.i["stamp"]), self.base_of(self.m["stamp"])
        im = ~(ib + self.k - 1 <= last_const) if drop_inertial else np.ones(ib.size, dtype=bool)
        mm = ~(mb + self.k - 1 <= last_const) if drop_manifold else np.ones(mb.size, dtype=bool)
        vb, bb = self.base_of(self.v["stamp"]), self.base_of(self.b["stamp"])
        mins = [begin] + [int(x[mask].min()) for x, mask in ((vb, vm), (bb, bm), (ib, im), (mb, mm)) if mask.any()]
        shift = max(0, min(min(mins), len(st) - self.k))
        sel = [p for p, g in enumerate(self.lm_ids) if g in keep_set]
        lmap = -np.ones(len(self.lm_ids), dtype=np.int32)
        lmap[sel] = np.arange(len(sel))
        dropped = dict(landmarks=len(self.lm_ids) - len(sel), visual=int((~vm).sum() + (~bm).sum()), inertial=int((~im).sum()),
                       manifold=int((~mm).sum()), knots=shift)
        self.lm_xyz, self.lm_ids = self.lm_xyz[sel], [self.lm_ids[p] for p in sel]
        for lists, mask in ((self.v, vm), (self.b, bm), (self.i, im), (self.m, mm)):
            for key in lists:
                lists[key] = lists[key][mask]
        self.knots = self.knots[shift:]
        self.knot_const = (self.knots[:, 7] <= lower).astype(np.uint8)
        if ub > 0:
            self.gravity_const = 1
        return dropped, lmap

    def counts(self):
        return [self.v["stamp"].size, self.i["stamp"].size, self.b["stamp"].size, self.m["stamp"].size]

    def window(self):
        return dataclasses.replace(super().window(), b_stamp=self.b["stamp"].copy(), b_cam=self.b["cam"].astype(np.int32), b_lm=self.local_lm(self.b["gid"]),
                                   b_bearing=self.b["bearing"].copy(), m_stamp=self.m["stamp"].copy(), m_sensor=self.m["sensor"].astype(np.int32),
                                   m_pose=self.m["pose"].copy())


def error_code(fn, *args):
    try:
        fn(*args)
    except runtime.HB200Error as e:
        return int(str(e).split(":")[0].split()[-1])
    return 0


def assert_same_state(a, b, what):
    sa, sb = a.state(), b.state()
    for key in sa:
        assert np.array_equal(sa[key], sb[key]), (what, key)


def sync_state(src, *ctxs):
    """Carry one context's state into every context and restart the trust region at its initial radius (hb200_optimize
    with 0 iterations): the LM step assembles the system with FP64 atomics, so two contexts agree bit for bit on
    everything but the last bits of an iterated state."""
    s = src.state()
    for ctx in ctxs:
        ctx.optimize(0, s["knots"].copy(), s["gyro_bias"].copy(), s["accel_bias"].copy(), s["gravity"].copy(), s["landmarks"].copy(), records=False)


def frame_loop_setup(order, K0, frames, seed):
    full = synthetic.make_window(order=order, num_knots=K0 + frames + 4, num_landmarks=0, num_imu=1200, seed=seed, bias_dt=1.0)
    full = synthetic.add_bearing_and_pose_factors(full, num_pose=3 * (K0 + frames), seed=seed + 1)
    hw = StereoHostWindow(full, K0)
    lo, hi = hw.valid_range()
    im = (full.i_stamp >= lo) & (full.i_stamp < hi)
    hw.add_lists(i=dict(stamp=full.i_stamp[im], meas=full.i_meas[im]))
    hw.knot_const[:2] = 1
    tracks = synthetic.make_stereo_tracks(full, hi, hi + 0.1 * frames, seed=seed + 2)
    return full, hw, hi, tracks


@pytest.mark.parametrize("order,frames,drop_manifold", [(4, 20, True), (4, 8, False), (6, 6, True)])
def test_stereo_frame_loop_two_paths_one_truth(built, order, frames, drop_manifold):
    K0, width = 14, 9
    full, hw, prev_hi, tracks = frame_loop_setup(order, K0, frames, synthetic.SEED_BASE + 4300 + order)
    A, B = runtime.Context(0), runtime.Context(0)
    for ctx in (A, B):
        ctx.load_window(hw.window())
    cams = full.cameras
    total = dict(landmarks=0, visual=0, inertial=0, manifold=0, knots=0)
    appended_manifold = 0
    for frame in range(frames):
        hw.append_knot()
        for ctx in (A, B):
            ctx.append_knots(1)
        _, hi = hw.valid_range()
        knots = A.state()["knots"]
        assert np.array_equal(knots, hw.knots), frame
        sel_frames = np.unique(tracks["stamp"][(tracks["stamp"] >= prev_hi) & (tracks["stamp"] < hi)])
        for s in sel_frames:   # one VisualTracks message per camera frame
            t = tracks["stamp"] == s
            gids, px0, px1 = tracks["gid"][t], tracks["px0"][t], tracks["px1"][t]
            n = gids.size
            pos = {g: p for p, g in enumerate(hw.lm_ids)}
            given = np.array([pos.get(g, -1) for g in gids.tolist()], dtype=np.int32)
            new = given < 0
            want = given.copy()
            want[new] = len(hw.lm_ids) + np.arange(int(new.sum()))
            stamp, c0, c1 = np.full(n, s), np.zeros(n, np.int32), np.ones(n, np.int32)
            base = int(hw.base_of(np.array([s]))[0])
            OB0, OB1, OL = ol.ingest_stereo_frame(knots[base:base + order], s, cams[0], cams[1], px0, px1)
            # A: on the device
            out, n_new = A.append_stereo_tracks(stamp, c0, c1, px0, px1, given)
            assert np.array_equal(out, want) and n_new == int(new.sum()), frame
            # B: composed
            b0, b1, lm_w, bad = B.ingest_stereo(stamp, c0, c1, px0, px1)
            assert bad == 0
            assert np.abs(b0 - OB0).max() < 1e-12 and np.abs(b1 - OB1).max() < 1e-12, frame
            if new.any():
                assert rel_err(lm_w[new], OL[new]) < 1e-9, frame
            B.append_landmarks(lm_w[new])
            bst, bcam = np.repeat(stamp, 2), np.stack([c0, c1], 1).ravel()
            blm, bear = np.repeat(want, 2), np.stack([b0, b1], 1).reshape(-1, 3)
            B.append_bearing_factors(bst, bcam, blm, bear)
            hw.add_landmarks(gids[new].tolist(), lm_w[new])
            hw.add_lists(b=dict(stamp=bst, cam=bcam, gid=np.repeat(gids, 2), bearing=bear))
        ii = (full.i_stamp >= prev_hi) & (full.i_stamp < hi)
        mi = np.flatnonzero((full.m_stamp >= prev_hi) & (full.m_stamp < hi))[:1] if frame % 3 == 0 else np.zeros(0, np.int64)
        prev_hi = hi
        for ctx in (A, B):
            ctx.append_inertial_factors(full.i_stamp[ii], full.i_meas[ii])
            ctx.append_manifold_factors(full.m_stamp[mi], full.m_sensor[mi], full.m_pose[mi])
        hw.add_lists(i=dict(stamp=full.i_stamp[ii], meas=full.i_meas[ii]), m=dict(stamp=full.m_stamp[mi], sensor=full.m_sensor[mi], pose=full.m_pose[mi]))
        appended_manifold += mi.size
        # --- the window moves on ---
        lower = hw.knots[len(hw.knots) - 1 - width, 7] + 1e-9
        stats = A.slide(lower, drop_inertial=True, drop_manifold=drop_manifold)
        assert B.slide(lower, drop_inertial=True, drop_manifold=drop_manifold) == stats
        dropped, lmap = hw.slide(lower, drop_inertial=True, drop_manifold=drop_manifold)
        for key in total:
            total[key] += dropped[key]
        assert (stats["knots"], stats["landmarks"], stats["visual_factors"], stats["inertial_factors"]) == \
            (len(hw.knots), len(hw.lm_ids), hw.v["stamp"].size + hw.b["stamp"].size, hw.i["stamp"].size), (frame, stats, dropped)
        assert (stats["knots_dropped"], stats["landmarks_dropped"], stats["visual_factors_dropped"], stats["inertial_factors_dropped"]) == \
            (dropped["knots"], dropped["landmarks"], dropped["visual"], dropped["inertial"]), (frame, stats, dropped)
        for ctx in (A, B):
            assert list(ctx.factor_counts()) == hw.counts(), frame
            assert np.array_equal(ctx.landmark_map(), lmap), frame
        assert_same_state(A, B, frame)
        st = A.state()
        assert np.array_equal(st["knots"], hw.knots) and np.array_equal(st["landmarks"], hw.lm_xyz), frame
        # --- residuals and Jacobians: A == B bit for bit, both against the oracle ---
        ow = ol.OracleWindow(hw.window(), radius=1e4)
        assert ow.bad == 0
        for ctx in (A, B):
            ctx.evaluate(jacobians=True)
        oa, ob, oo = A.outputs(), B.outputs(), ow.evaluate()
        assert oa.keys() == ob.keys()
        for key in oa:
            assert np.array_equal(oa[key], ob[key]), (frame, key)
        for key in ("b_r", "m_r", "i_r", "b_Jp", "b_Jl", "m_Jp", "i_Jp"):
            if key in oo and oo[key].size:
                assert rel_err(oa[key], oo[key]) < (1e-9 if key.endswith("_r") else 1e-8), (frame, key)
        # --- two LM iterations on each context against the oracle ---
        # Ten times looser than the pixel sequence of test_gpu_sliding.py: a landmark that entered with the newest camera
        # frame has two bearings 11 cm apart, its depth is weakly determined, and the step's forward error grows with it.
        ra, rb = A.iterate(2), B.iterate(2)
        for a, b in zip(ra, rb):
            o = ow.iterate(apply=True)
            for rec in (a, b):
                assert rec["spd"] == 1 and rec["accepted"] == o["accepted"], (frame, rec, o["accepted"])
                assert abs(rec["cost"] - o["cost"]) <= 1e-6 * abs(o["cost"]), (frame, rec, o["cost"])
                assert abs(rec["cost_new"] - o["cost_new"]) <= 1e-5 * abs(o["cost_new"]), (frame, rec, o["cost_new"])
        so = ow.state()
        for ctx in (A, B):
            st = ctx.state()
            for key in ("knots", "landmarks", "gyro_bias", "accel_bias", "gravity"):
                if so[key].size:
                    assert rel_err(st[key], so[key]) < 1e-5, (frame, key)
        sync_state(A, A, B)
        st = A.state()
        hw.knots, hw.lm_xyz = st["knots"].copy(), st["landmarks"].copy()
        hw.full = dataclasses.replace(hw.full, gyro_bias=st["gyro_bias"].copy(), accel_bias=st["accel_bias"].copy(), gravity=st["gravity"].copy())
    if frames >= 20:
        assert total["knots"] > 3 and total["landmarks"] > 20 and total["visual"] > 100 and total["manifold"] > 0, total
    if not drop_manifold:   # the reference never removes pose residuals: every one stays and holds its leading knots
        assert A.factor_counts()[runtime.MANIFOLD] == appended_manifold > 0 and total["manifold"] == 0, total
    A.close(); B.close()


def test_mixed_visual_list_outputs_and_full_rebind(built):
    """Pixel and bearing appends interleave in one visual list; after a slide each family comes back in bound order and
    agrees with an oracle window of the two lists; a full bind of the same window rebuilds it."""
    full = synthetic.make_window(order=4, num_knots=30, num_landmarks=160, frames_per_landmark=4, num_imu=600, seed=synthetic.SEED_BASE + 4400, bias_dt=1.0)
    hw = StereoHostWindow(full, 12)
    lo, hi = hw.valid_range()
    nv, ni, new_ids = hw.take_new(lo, hi)
    hw.add(nv, ni, new_ids)
    hw.knot_const[:2] = 1
    ctx = runtime.Context(0)
    ctx.load_window(hw.window())
    truth = full.truth
    prev_hi = hi
    for frame in range(6):
        hw.append_knot()
        ctx.append_knots(1)
        _, hi = hw.valid_range()
        nv, ni, new_ids = hw.take_new(prev_hi, hi)
        prev_hi = hi
        ctx.append_landmarks(full.landmarks[new_ids].reshape(-1, 3))
        hw.add(dict(stamp=nv["stamp"][:0], cam=nv["cam"][:0], gid=nv["gid"][:0], pixel=nv["pixel"][:0]), ni, new_ids)
        ctx.append_inertial_factors(ni["stamp"], ni["meas"])
        # alternate runs of pixel and bearing factors, arrival order kept
        for lo_, hi_ in ((0, nv["stamp"].size // 3), (nv["stamp"].size // 3, 2 * nv["stamp"].size // 3), (2 * nv["stamp"].size // 3, nv["stamp"].size)):
            part = {key: val[lo_:hi_] for key, val in nv.items()}
            if not part["stamp"].size:
                continue
            lm = hw.local_lm(part["gid"])
            if (lo_ // max(1, nv["stamp"].size // 3)) % 2 == 0:
                ctx.append_pixel_factors(part["stamp"], part["cam"], lm, part["pixel"])
                hw.add(part, dict(stamp=np.zeros(0), meas=np.zeros((0, 6))), [])
            else:
                _, p_s = synthetic.pixel_model(truth["knots"], 4, full.cameras, truth["landmarks"], part["stamp"], part["cam"], part["gid"])
                bear = p_s / np.linalg.norm(p_s, axis=1, keepdims=True)
                ctx.append_bearing_factors(part["stamp"], part["cam"], lm, bear)
                hw.add_lists(b=dict(stamp=part["stamp"], cam=part["cam"], gid=part["gid"], bearing=bear))
        lower = hw.knots[len(hw.knots) - 1 - 9, 7] + 1e-9
        ctx.slide(lower)
        hw.slide(lower)
        assert list(ctx.factor_counts()) == hw.counts(), frame
    assert hw.v["stamp"].size and hw.b["stamp"].size
    ow = ol.OracleWindow(hw.window())
    ctx.evaluate(jacobians=True)
    got, want = ctx.outputs(), ow.evaluate()
    for key in ("v_r", "b_r", "i_r"):
        assert rel_err(got[key], want[key]) < 1e-9, key
    for key in ("v_Jp", "v_Jl", "b_Jp", "b_Jl", "i_Jp"):
        assert rel_err(got[key], want[key]) < 1e-8, key
    ctx.build_system()
    S0, b0 = ctx.system()
    ctx.bind()   # full re-bind of the device lists where they stand, host sort of the keys, derive
    ctx.evaluate(jacobians=True)
    again = ctx.outputs()
    for key in got:
        assert np.array_equal(got[key], again[key]), key
    ctx.build_system()
    S1, b1 = ctx.system()
    assert rel_err(S1, S0) < 1e-12 and rel_err(b1, b0) < 1e-12   # same terms; FP64 atomics sum them in another order
    ctx.close()


def test_failed_appends_leave_the_window_intact(built):
    full = synthetic.make_window(order=4, num_knots=24, num_landmarks=0, num_imu=400, seed=synthetic.SEED_BASE + 4500, bias_dt=1.0)
    full = synthetic.add_bearing_and_pose_factors(full, num_pose=20, seed=synthetic.SEED_BASE + 4501)
    # camera 2: identity rotation, no distortion -- two views of its principal point are exactly parallel rays
    cam2 = np.concatenate([[0, 0, 0, 1, 0.05, 0, 0], full.cameras[0, 7:11], [0, 0, 0, 0]])
    full = dataclasses.replace(full, cameras=np.vstack([full.cameras, cam2]))
    hw = StereoHostWindow(full, 16)
    lo, hi = hw.valid_range()
    im = (full.i_stamp >= lo) & (full.i_stamp < hi)
    hw.add_lists(i=dict(stamp=full.i_stamp[im], meas=full.i_meas[im]))
    ctx = runtime.Context(0)
    ctx.load_window(hw.window())
    tracks = synthetic.make_stereo_tracks(full, lo + 0.2, hi, seed=synthetic.SEED_BASE + 4502)
    s0 = np.unique(tracks["stamp"])[2]
    t = tracks["stamp"] == s0
    n = int(t.sum())
    args = [np.full(n, s0), np.zeros(n, np.int32), np.ones(n, np.int32), tracks["px0"][t], tracks["px1"][t], -np.ones(n, np.int32)]
    ctx.append_stereo_tracks(*args)
    ctx.append_manifold_factors(full.m_stamp[:1], full.m_sensor[:1], full.m_pose[:1])

    def snapshot():
        return ctx.factor_counts().tolist(), (ctx.K, ctx.L), ctx.state()

    def unchanged(before):
        counts, sizes, st = before
        assert ctx.factor_counts().tolist() == counts and (ctx.K, ctx.L) == sizes
        now = ctx.state()
        for key in st:
            assert np.array_equal(now[key], st[key]), key

    L = ctx.L
    s1 = np.unique(tracks["stamp"])[3]
    t1 = tracks["stamp"] == s1
    m = int(t1.sum())
    good = [np.full(m, s1), np.zeros(m, np.int32), np.ones(m, np.int32), tracks["px0"][t1], tracks["px1"][t1], -np.ones(m, np.int32)]
    bad_cases = []
    a = [x.copy() for x in good]; a[1][m // 2] = 7; bad_cases.append((a, 2))                           # invalid camera
    a = [x.copy() for x in good]; a[0][:] = hi + 1.0; bad_cases.append((a, 2))                        # stamp out of range
    a = [x.copy() for x in good]; a[5][0] = L; bad_cases.append((a, 2))                               # existing-landmark index >= L
    a = [x.copy() for x in good]; a[0][:] = s0 - 0.3; bad_cases.append((a, 3))                        # before the end of the visual list
    a = [x.copy() for x in good]; a[3][1] = np.nan; bad_cases.append((a, 2))                          # non-finite triangulation
    a = [x.copy() for x in good]; a[1][0] = a[2][0] = 2; a[3][0] = a[4][0] = cam2[7:9]                # parallel rays
    _, _, lw, _ = ctx.ingest_stereo(*[x[:1] for x in a[:5]])
    parallel_nonfinite = not np.isfinite(lw).all()
    if parallel_nonfinite:
        bad_cases.append((a, 2))
    for a, code in bad_cases:
        before = snapshot()
        assert error_code(ctx.append_stereo_tracks, *a) == code
        unchanged(before)
    before = snapshot()
    assert error_code(ctx.append_bearing_factors, np.full(2, s1), np.array([0, 9]), np.zeros(2, np.int32), np.ones((2, 3))) == 2
    unchanged(before)
    assert error_code(ctx.append_bearing_factors, np.full(2, s0 - 0.3), np.array([0, 1]), np.zeros(2, np.int32), np.ones((2, 3))) == 3
    unchanged(before)
    assert error_code(ctx.append_manifold_factors, full.m_stamp[1:2], np.array([5]), full.m_pose[1:2]) == 2
    unchanged(before)
    out, n_new = ctx.append_stereo_tracks(*good)
    assert n_new == m and np.array_equal(out, L + np.arange(m)) and ctx.L == L + m
    assert ctx.factor_counts().tolist() == [0, hw.i["stamp"].size, 2 * (n + m), 1]
    ctx.close()
    assert parallel_nonfinite, "two views of one principal point through one camera should triangulate to a non-finite point"
