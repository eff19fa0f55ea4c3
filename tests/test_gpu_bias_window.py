"""Bias splines that grow and slide with the device-side window (hb200_append_bias_knots, HB200_SLIDE_DROP_BIAS).

The reference calls updateSensor whenever an IMU sample falls past a bias spline (abstract.cpp:272-292) and applies its
removal rule (optimizer.cpp:331-341) to every state element.  Here the stereo-inertial frame loop of
test_gpu_stereo_window.py starts from kb bias knots per spline, extends both splines before each frame's IMU samples and
slides with DROP_INERTIAL | DROP_BIAS.  Per frame the device is checked against a host restatement of the rules (sizes,
bias values and stamps bit for bit, dropped counts, bias base maps), against a second context loaded from the restated
window by set_* + bind (residuals and Jacobians bit for bit), and against the oracle (LM records and state).
"""
import dataclasses
import math

import numpy as np
import pytest

import oracle_lib as ol
from hyperslam_b200 import runtime, synthetic
from test_bias_extension import append_count, bias_base, extend
from test_gpu_sliding import rel_err
from test_gpu_solvers import run_case, solver_window
from test_gpu_stereo_window import StereoHostWindow, error_code, sync_state

pytestmark = pytest.mark.gpu

KB = 4


class BiasHostWindow(StereoHostWindow):
    """StereoHostWindow with its own bias splines: extension before the IMU samples, the removal rule on slides."""

    def __init__(self, full, K0, gyro, accel):
        super().__init__(full, K0)
        self.bg, self.ba = gyro.copy(), accel.copy()
        self.bias_dropped = (0, 0)

    def append_bias(self, t):
        ng, na = append_count(self.bg, t), append_count(self.ba, t)
        self.bg, self.ba = extend(self.bg, ng), extend(self.ba, na)
        return ng, na

    @staticmethod
    def _bias_shift(b, lower, kept_stamps):
        st = b[:, 3]
        ub = int(np.searchsorted(st, lower, side="right"))
        mins = [max(0, ub - 1 - (KB - 1) // 2)] + ([int(bias_base(st, kept_stamps).min())] if kept_stamps.size else [])
        return max(0, min(min(mins), len(st) - KB))

    def slide(self, lower, drop_inertial=True, drop_manifold=False, drop_bias=False):
        out = super().slide(lower, drop_inertial, drop_manifold)
        gd = ad = 0
        if drop_bias and drop_inertial:   # self.i now holds exactly the kept inertial factors
            gd, ad = self._bias_shift(self.bg, lower, self.i["stamp"]), self._bias_shift(self.ba, lower, self.i["stamp"])
            self.bg, self.ba = self.bg[gd:], self.ba[ad:]
        self.bias_dropped = (gd, ad)
        return out

    def bias_maps(self):
        return bias_base(self.bg[:, 3], self.i["stamp"]), bias_base(self.ba[:, 3], self.i["stamp"])

    def window(self):
        return dataclasses.replace(super().window(), gyro_bias=self.bg.copy(), accel_bias=self.ba.copy(), bias_const=0)


def start_splines(t0, gyro_dt, accel_dt, full):
    """kb knots per spline whose valid span starts at t0, valued at the perturbed template's first bias knot."""
    out = []
    for dt, src in ((gyro_dt, full.gyro_bias), (accel_dt, full.accel_bias)):
        b = np.zeros((KB, 4))
        b[:, :3] = src[0, :3]
        b[:, 3] = t0 + (np.arange(KB) - (KB - 1) // 2) * dt
        out.append(b)
    return out


def assert_state_unchanged(ctx, before):
    sizes, st, maps = before
    assert (ctx.K, ctx.L, ctx.Kbg, ctx.Kba) == sizes and ctx.bias_knots()["gyro"] == sizes[2] and ctx.bias_knots()["accel"] == sizes[3]
    now = ctx.state()
    for key in st:
        assert np.array_equal(now[key], st[key]), key
    for a, b in zip(ctx.index_maps(), maps):
        assert np.array_equal(a, b)


def test_append_bias_knots_rule_and_errors(built):
    full = synthetic.make_window(order=4, num_knots=80, num_landmarks=0, num_imu=800, seed=synthetic.SEED_BASE + 5200)
    gyro, accel = start_splines(0.3, 0.7, 1.1 / 3.0, full)
    hw = BiasHostWindow(full, 80, gyro, accel)
    ctx = runtime.Context(0)
    ctx.load_window(hw.window())   # no inertial factors yet
    # stamps inside both spans append nothing
    assert ctx.append_bias_knots(0.3) == (0, 0) and ctx.append_bias_knots(0.6) == (0, 0)
    # growing stamps: the device follows the restated rule bit for bit, gyro and accel independently
    seen = set()
    for t in (0.7, 1.0, 1.35, 2.2, 2.2, 4.05, 7.3):
        want = hw.append_bias(t)
        got = ctx.append_bias_knots(t)
        assert got == want, (t, got, want)
        seen.add(got)
        st = ctx.state()
        assert np.array_equal(st["gyro_bias"], hw.bg) and np.array_equal(st["accel_bias"], hw.ba), t
        assert ctx.bias_knots() == dict(gyro=len(hw.bg), accel=len(hw.ba), gyro_dropped=0, accel_dropped=0)
        assert ctx.reduced_size() == 6 * ctx.K + 3 * (len(hw.bg) + len(hw.ba)) + 2
    assert (0, 0) in seen and any(g != a for g, a in seen) and any(g > 1 for g, _ in seen)
    # an inertial factor at the newest stamp now binds, and its bias bases are the oracle's
    im = (full.i_stamp >= 0.3) & (full.i_stamp <= 7.3)
    ctx.append_inertial_factors(full.i_stamp[im], full.i_meas[im])
    hw.add_lists(i=dict(stamp=full.i_stamp[im], meas=full.i_meas[im]))
    ow = ol.OracleWindow(hw.window())
    assert ow.bad == 0
    for got, want in zip(ctx.index_maps()[1:], ow.index_maps()[1:]):
        assert np.array_equal(got, want)
    # failed calls change nothing
    before = ((ctx.K, ctx.L, ctx.Kbg, ctx.Kba), ctx.state(), ctx.index_maps())
    sep = hw.ba[-1, 3] - hw.ba[-2, 3]
    for t, code in ((math.nan, -1), (math.inf, -1), (-math.inf, -1), (hw.ba[-1, 3] + (runtime.BIAS_APPEND_MAX + 3) * sep, -1),
                    (np.nextafter(hw.ba[1, 3], -np.inf), 2), (0.0, 2), (1e300, -1)):
        assert error_code(ctx.append_bias_knots, t) == code, t
        assert_state_unchanged(ctx, before)
    ctx.close()
    # -2: no bias splines; bias splines but no bound window
    bare = runtime.Context(0)
    assert error_code(bare.append_bias_knots, 1.0) == -2
    bare.set_spline(4, full.knots)
    bare.set_bias_splines(4, gyro, accel)
    assert error_code(bare.append_bias_knots, 5.0) == -2
    assert bare.bias_knots()["gyro"] == KB
    bare.close()


def run_bias_loop(order, frames, drop_bias, seed, gyro_dt=0.5, accel_dt=0.6):
    K0, width, dt = 14, 9, 0.1
    full = synthetic.make_window(order=order, num_knots=K0 + frames + 4, num_landmarks=0, num_imu=30 * (K0 + frames + 4), seed=seed, bias_dt=1.0)
    full = synthetic.add_bearing_and_pose_factors(full, num_pose=3 * (K0 + frames), seed=seed + 1)
    lo, hi = StereoHostWindow(full, K0).valid_range()
    hw = BiasHostWindow(full, K0, *start_splines(lo, gyro_dt, accel_dt, full))
    hw.knot_const[:2] = 1
    tracks = synthetic.make_stereo_tracks(full, hi, hi + dt * frames, seed=seed + 2)
    A, B = runtime.Context(0), runtime.Context(0)
    A.load_window(hw.window())
    # the first IMU samples: extend from kb knots, then append them
    im = (full.i_stamp >= lo) & (full.i_stamp < hi)
    assert A.append_bias_knots(full.i_stamp[im].max()) == hw.append_bias(full.i_stamp[im].max())
    A.append_inertial_factors(full.i_stamp[im], full.i_meas[im])
    hw.add_lists(i=dict(stamp=full.i_stamp[im], meas=full.i_meas[im]))
    prev_hi, spans, sizes, dropped_total = hi, [], [], [0, 0]
    for frame in range(frames):
        hw.append_knot()
        A.append_knots(1)
        _, hi = hw.valid_range()
        for s in np.unique(tracks["stamp"][(tracks["stamp"] >= prev_hi) & (tracks["stamp"] < hi)]):
            t = tracks["stamp"] == s
            pos = {g: p for p, g in enumerate(hw.lm_ids)}
            if frame == frames - 1:
                # the last frame only continues tracks: a landmark seen by one stereo pair has two bearing rows, a
                # rank-deficient V_l, and the covariance at the end would refuse it (status 2)
                t &= np.isin(tracks["gid"], list(pos))
                if not t.any():
                    continue
            gids, px0, px1 = tracks["gid"][t], tracks["px0"][t], tracks["px1"][t]
            n = gids.size
            given = np.array([pos.get(g, -1) for g in gids.tolist()], dtype=np.int32)
            new = given < 0
            stamp, c0, c1 = np.full(n, s), np.zeros(n, np.int32), np.ones(n, np.int32)
            b0, b1, lm_w, bad = A.ingest_stereo(stamp, c0, c1, px0, px1)   # what append_stereo_tracks writes, bit for bit
            assert bad == 0
            out, n_new = A.append_stereo_tracks(stamp, c0, c1, px0, px1, given)
            want = given.copy()
            want[new] = len(hw.lm_ids) + np.arange(int(new.sum()))
            assert np.array_equal(out, want) and n_new == int(new.sum()), frame
            hw.add_landmarks(gids[new].tolist(), lm_w[new])
            hw.add_lists(b=dict(stamp=np.repeat(stamp, 2), cam=np.stack([c0, c1], 1).ravel(), gid=np.repeat(gids, 2), bearing=np.stack([b0, b1], 1).reshape(-1, 3)))
        ii = (full.i_stamp >= prev_hi) & (full.i_stamp < hi)
        mi = np.flatnonzero((full.m_stamp >= prev_hi) & (full.m_stamp < hi))[:1] if frame % 3 == 0 else np.zeros(0, np.int64)
        prev_hi = hi
        if ii.any():   # process(InertialMeasurement): updateSensor for the newest sample, then the samples
            t_last = full.i_stamp[ii].max()
            assert A.append_bias_knots(t_last) == hw.append_bias(t_last), frame
            A.append_inertial_factors(full.i_stamp[ii], full.i_meas[ii])
        A.append_manifold_factors(full.m_stamp[mi], full.m_sensor[mi], full.m_pose[mi])
        hw.add_lists(i=dict(stamp=full.i_stamp[ii], meas=full.i_meas[ii]), m=dict(stamp=full.m_stamp[mi], sensor=full.m_sensor[mi], pose=full.m_pose[mi]))
        # --- the window moves on ---
        lower = hw.knots[len(hw.knots) - 1 - width, 7] + 1e-9
        spans.append(hi - lower)
        stats = A.slide(lower, drop_inertial=True, drop_manifold=True, drop_bias=drop_bias)
        dropped, lmap = hw.slide(lower, drop_inertial=True, drop_manifold=True, drop_bias=drop_bias)
        assert (stats["knots"], stats["landmarks"], stats["inertial_factors"]) == (len(hw.knots), len(hw.lm_ids), hw.i["stamp"].size), frame
        assert (stats["knots_dropped"], stats["inertial_factors_dropped"]) == (dropped["knots"], dropped["inertial"]), frame
        assert list(A.factor_counts()) == hw.counts() and np.array_equal(A.landmark_map(), lmap), frame
        bk = A.bias_knots()
        assert bk == dict(gyro=len(hw.bg), accel=len(hw.ba), gyro_dropped=hw.bias_dropped[0], accel_dropped=hw.bias_dropped[1]), (frame, bk)
        assert (A.Kbg, A.Kba) == (len(hw.bg), len(hw.ba))
        dropped_total[0] += bk["gyro_dropped"]; dropped_total[1] += bk["accel_dropped"]
        sizes.append((len(hw.bg), len(hw.ba)))
        st = A.state()
        for key, want in (("knots", hw.knots), ("landmarks", hw.lm_xyz), ("gyro_bias", hw.bg), ("accel_bias", hw.ba)):
            assert np.array_equal(st[key], want), (frame, key)
        _, ib, ig, ia = A.index_maps()
        hg, ha = hw.bias_maps()
        assert np.array_equal(ib, hw.base_of(hw.i["stamp"])) and np.array_equal(ig, hg) and np.array_equal(ia, ha), frame
        assert ig.min() >= 0 and ia.min() >= 0 and ig.max() + KB <= len(hw.bg) and ia.max() + KB <= len(hw.ba)
        # --- residuals and Jacobians: bit for bit against the restated window, set_* + bind on a second context ---
        win = hw.window()
        B.load_window(win)
        A.evaluate(jacobians=True); B.evaluate(jacobians=True)
        oa, ob = A.outputs(), B.outputs()
        assert oa.keys() == ob.keys()
        for key in oa:
            assert np.array_equal(oa[key], ob[key]), (frame, key)
        # --- the oracle: index maps, two LM iterations, state (tolerances of test_gpu_stereo_window.py) ---
        ow = ol.OracleWindow(win, radius=1e4)
        assert ow.bad == 0
        for got, want in zip(A.index_maps()[1:], ow.index_maps()[1:]):
            assert np.array_equal(got, want), frame
        for rec in A.iterate(2):
            o = ow.iterate(apply=True)
            assert rec["spd"] == 1 and rec["accepted"] == o["accepted"], (frame, rec, o["accepted"])
            assert abs(rec["cost"] - o["cost"]) <= 1e-6 * abs(o["cost"]), (frame, rec, o["cost"])
            assert abs(rec["cost_new"] - o["cost_new"]) <= 1e-5 * abs(o["cost_new"]), (frame, rec, o["cost_new"])
        so, st = ow.state(), A.state()
        for key in ("knots", "landmarks", "gyro_bias", "accel_bias", "gravity"):
            if so[key].size:
                assert rel_err(st[key], so[key]) < 1e-5, (frame, key)
        sync_state(A, A)
        st = A.state()
        hw.knots, hw.lm_xyz, hw.bg, hw.ba = st["knots"].copy(), st["landmarks"].copy(), st["gyro_bias"].copy(), st["accel_bias"].copy()
        hw.full = dataclasses.replace(hw.full, gravity=st["gravity"].copy())
    B.close()
    return A, hw, sizes, spans, dropped_total


def bias_bound(order, spans, sep, dt=0.1):
    """Bias knots a slid window can hold.  The kept inertial factors span less than T = (window length) + (k - 1)
    knot separations: the window ends at the valid range's end, and a factor stays while one of its k control points
    lies past the lower bound.  An interval shorter than T touches at most ceil(T / sep) + 1 bias segments; the fewest-knots
    extension ends the spline with the newest sample's segment, and the removal rule starts it at the earliest kept
    factor's base, so at most ceil(T / sep) + kb knots stay."""
    T = max(spans) + (order - 1) * dt
    return math.ceil(T / sep) + KB


def hold_poses(ctx):
    """Every state element constant, gravity constant, biases variable: the covariance then speaks about the bias block
    alone.  (With variable poses the window's newest state element, which only the newest segment's samples reach, fails
    its pivot first in this loop.)"""
    ctx.set_constant(np.ones(ctx.K, np.uint8), gravity_const=1, bias_const=0)


@pytest.mark.parametrize("order,frames", [(4, 30), (6, 30)])
def test_bias_frame_loop_stays_bounded(built, order, frames):
    gyro_dt, accel_dt = 0.5, 0.6
    A, hw, sizes, spans, dropped = run_bias_loop(order, frames, True, synthetic.SEED_BASE + 5300 + order, gyro_dt, accel_dt)
    assert frames * 0.1 >= 5 * max(gyro_dt, accel_dt) - 1e-9   # at least five separations of either spline
    bg_max, ba_max = bias_bound(order, spans, gyro_dt), bias_bound(order, spans, accel_dt)
    m_max = 3 * (bg_max + ba_max) + 2
    assert m_max <= 54, m_max   # BCR's arrow limit (DESIGN 5.2)
    for g, a in sizes:
        assert g <= bg_max and a <= ba_max and 3 * (g + a) + 2 <= m_max, (sizes, bg_max, ba_max)
    assert dropped[0] >= 3 and dropped[1] >= 3, dropped
    # every bias knot is held by a kept inertial factor: the bias block of the covariance exists
    hold_poses(A)
    A.build_covariance()
    info = A.compute_covariance()
    assert info["rc"] == 0 and info["status"] == 0, info
    A.close()


def test_bias_frame_loop_without_drop_grows_and_loses_covariance(built):
    order, frames, gyro_dt = 4, 30, 0.5
    A, hw, sizes, spans, dropped = run_bias_loop(order, frames, False, synthetic.SEED_BASE + 5400, gyro_dt, 0.6)
    assert dropped == [0, 0]
    assert sizes[-1][0] > bias_bound(order, spans, gyro_dt) and sizes[-1][0] > sizes[len(sizes) // 2][0] > sizes[0][0], sizes
    # the earliest bias knots no longer have an inertial factor
    assert bias_base(hw.bg[:, 3], hw.i["stamp"]).min() > 0
    hold_poses(A)
    A.build_covariance()
    info = A.compute_covariance()
    K, nbias = A.K, 3 * (A.Kbg + A.Kba)
    assert info["status"] == 1 and info["bad_dof"] == 6 * K, info   # the first dof of the earliest gyro bias knot
    A.close()


# ---- a growing arrowhead and the chunked band solver --------------------------------------------------------
# Without DROP_BIAS the arrowhead grows by 6 rows per bias separation.  band_solve_kernel<false> moves the corner system
# [m + 1][m | 1] and two m-vectors into its shared memory after the factorisation; from m of about 155 that is more
# than its two chunk views, and past 220 KB the window does not fit the solver at all.
def test_chunked_solver_with_a_corner_wider_than_its_chunk_views(built, record_property):
    run_case(40, 5, 26, 26, "chunked", report=record_property)   # m = 158: corner 204 824 B, chunk views 194 880 B


def test_arrow_too_wide_for_the_chunked_solver(built):
    ctx = runtime.Context(0)
    assert error_code(ctx.load_window, solver_window(40, 28, 28)) == -6   # m = 170: corner 236 696 B
    ctx.close()
