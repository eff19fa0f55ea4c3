"""Device-side sliding-window bookkeeping (SURVEY.md section 8f rank 3) against a host restatement of the reference's
rules + the oracle, over a 20-frame sequence:

  per frame   append one state element by the reference's extrapolation (abstract.cpp:126-136), add the frame's
              landmarks and residual blocks (optimizer.cpp:212-232,253-274,347-358), move the window's lower bound
              (landmarks whose observation range left the window go with their residuals, optimizer.cpp:360-382;
              elements at or before the bound become constant, :322-328; unreferenced leading elements are removed,
              :331-341; gravity constant, abstract.cpp:57-61), then two LM iterations.

The host side keeps plain Python lists and applies the same rules; the oracle is rebuilt from those lists every frame.
Checked per frame: window sizes, the state arrays after the bookkeeping (bit-exact copies), the index maps
(bit-exact), iteration records and the state after the iterations.
"""
import dataclasses

import numpy as np
import pytest

import oracle_lib as ol
from hyperslam_b200 import runtime, synthetic

pytestmark = pytest.mark.gpu


def rel_err(a, b):
    return float(np.abs(np.asarray(a) - np.asarray(b)).max() / (np.abs(np.asarray(b)).max() + 1e-300))


class HostWindow:
    """The reference's window rules on plain arrays (the test's independent restatement)."""

    def __init__(self, full, K0):
        self.full, self.k = full, full.order
        self.knots = full.knots[:K0].copy()
        self.lm_ids = []          # global landmark ids in window order
        self.lm_xyz = np.zeros((0, 3))
        self.v = dict(stamp=np.zeros(0), cam=np.zeros(0, np.int32), gid=np.zeros(0, np.int64), pixel=np.zeros((0, 2)))
        self.i = dict(stamp=np.zeros(0), meas=np.zeros((0, 6)))
        self.knot_const = np.zeros(K0, np.uint8)
        self.gravity_const = 0
        self.upper = None

    def valid_range(self):
        left = (self.k - 1) // 2
        st = self.knots[:, 7]
        return st[left], st[len(st) - (self.k - 1 - left) - 1]   # [first segment start, last segment end)

    def take_new(self, lo, hi):
        f = self.full
        vm = (f.v_stamp >= lo) & (f.v_stamp < hi)
        im = (f.i_stamp >= lo) & (f.i_stamp < hi)
        order_v, order_i = np.argsort(f.v_stamp[vm], kind="stable"), np.argsort(f.i_stamp[im], kind="stable")
        nv = dict(stamp=f.v_stamp[vm][order_v], cam=f.v_cam[vm][order_v], gid=f.v_lm[vm][order_v].astype(np.int64), pixel=f.v_pixel[vm][order_v])
        ni = dict(stamp=f.i_stamp[im][order_i], meas=f.i_meas[im][order_i])
        new_ids = [g for g in dict.fromkeys(nv["gid"].tolist()) if g not in self.lm_ids]
        return nv, ni, new_ids

    def add(self, nv, ni, new_ids):
        self.lm_ids += new_ids
        self.lm_xyz = np.vstack([self.lm_xyz, self.full.landmarks[new_ids].reshape(-1, 3)])
        for key in self.v:
            self.v[key] = np.concatenate([self.v[key], nv[key]])
        for key in self.i:
            self.i[key] = np.concatenate([self.i[key], ni[key]])

    def local_lm(self, gids):
        pos = {g: p for p, g in enumerate(self.lm_ids)}
        return np.array([pos[g] for g in gids.tolist()], dtype=np.int32)

    def append_knot(self):
        st = self.knots[:, 7]
        new = self.knots[-2].copy()
        self.knots[-1, :7] = self.knots[-2, :7]
        new[7] = st[-1] + (st[-1] - st[-2])
        self.knots = np.vstack([self.knots, new])
        self.knot_const = np.append(self.knot_const, 0).astype(np.uint8)

    def base_of(self, stamps):
        st = self.knots[:, 7]
        j = np.searchsorted(st, stamps, side="right") - 1
        return j - (self.k - 1) // 2

    def slide(self, lower, drop_inertial=True):
        st = self.knots[:, 7]
        ub = int(np.searchsorted(st, lower, side="right"))
        begin, last_const = max(0, ub - 1 - (self.k - 1) // 2), ub - 1
        last = {}
        for g, t in zip(self.v["gid"].tolist(), self.v["stamp"].tolist()):
            last[g] = max(last.get(g, -np.inf), t)
        keep_lm = [g for g in self.lm_ids if g not in last or last[g] >= lower]
        keep_set = set(keep_lm)
        vm = np.array([g in keep_set for g in self.v["gid"].tolist()], dtype=bool)
        ib = self.base_of(self.i["stamp"])
        im = ~(ib + self.k - 1 <= last_const) if drop_inertial else np.ones(ib.size, dtype=bool)   # the reference itself never removes inertial residuals
        vb = self.base_of(self.v["stamp"])
        mins = [begin] + ([int(vb[vm].min())] if vm.any() else []) + ([int(ib[im].min())] if im.any() else [])
        shift = max(0, min(min(mins), len(st) - self.k))
        dropped = dict(landmarks=len(self.lm_ids) - len(keep_lm), visual=int((~vm).sum()), inertial=int((~im).sum()), knots=shift)
        sel = [p for p, g in enumerate(self.lm_ids) if g in keep_set]
        self.lm_xyz, self.lm_ids = self.lm_xyz[sel], keep_lm
        for key in self.v:
            self.v[key] = self.v[key][vm]
        for key in self.i:
            self.i[key] = self.i[key][im]
        self.knots = self.knots[shift:]
        self.knot_const = (self.knots[:, 7] <= lower).astype(np.uint8)
        if ub > 0:
            self.gravity_const = 1
        return dropped

    def window(self):
        f = self.full
        return dataclasses.replace(f, knots=self.knots.copy(), landmarks=self.lm_xyz.copy(), v_stamp=self.v["stamp"].copy(), v_cam=self.v["cam"].astype(np.int32),
                                   v_lm=self.local_lm(self.v["gid"]), v_pixel=self.v["pixel"].copy(), i_stamp=self.i["stamp"].copy(), i_meas=self.i["meas"].copy(),
                                   knot_const=self.knot_const.copy(), gravity_const=self.gravity_const, truth=None)


@pytest.mark.parametrize("drop_inertial", [True, False])
def test_sliding_sequence_matches_host_rules_and_oracle(built, drop_inertial):
    K0, frames, width = 14, (20 if drop_inertial else 8), 9
    # bias knots every 1 s: with the default 10 s a sub-second window sits inside one bias segment, its four control points
    # are nearly collinear, and once the trust region reaches its 1e16 cap a 1e-15 change of the knots moves the oracle's own
    # accel-bias solution by up to 7e-7 relative -- any summation order other than the oracle's could then miss the 1e-6 bound
    full = synthetic.make_window(order=4, num_knots=K0 + 20 + 2, num_landmarks=220, frames_per_landmark=5, num_imu=1500, seed=synthetic.SEED_BASE + 1234,
                                 bias_dt=1.0)
    hw = HostWindow(full, K0)
    lo, hi = hw.valid_range()
    nv, ni, new_ids = hw.take_new(lo, hi)
    hw.add(nv, ni, new_ids)
    hw.knot_const[:2] = 1
    ctx = runtime.Context(0)
    ctx.load_window(hw.window())
    prev_hi = hi
    radius = 1e4   # hb200_iterate continues the trust region across calls; the oracle is rebuilt per frame with the same radius
    total_dropped = dict(landmarks=0, visual=0, inertial=0, knots=0)
    for frame in range(frames):
        # --- the message: one more state element, the frame's factors, the window moves on ---
        hw.append_knot()
        ctx.append_knots(1)
        _, hi = hw.valid_range()
        nv, ni, new_ids = hw.take_new(prev_hi, hi)
        prev_hi = hi
        ctx.append_landmarks(full.landmarks[new_ids].reshape(-1, 3))
        hw.add(nv, ni, new_ids)
        ctx.append_pixel_factors(nv["stamp"], nv["cam"], hw.local_lm(nv["gid"]), nv["pixel"])
        ctx.append_inertial_factors(ni["stamp"], ni["meas"])
        lower = hw.knots[len(hw.knots) - 1 - width, 7] + 1e-9
        stats = ctx.slide(lower, drop_inertial=drop_inertial)
        dropped = hw.slide(lower, drop_inertial=drop_inertial)
        for key in total_dropped:
            total_dropped[key] += dropped[key]
        assert (stats["knots"], stats["landmarks"], stats["visual_factors"], stats["inertial_factors"]) == \
            (len(hw.knots), len(hw.lm_ids), hw.v["stamp"].size, hw.i["stamp"].size), (frame, stats, dropped)
        assert stats["knots_dropped"] == dropped["knots"] and stats["landmarks_dropped"] == dropped["landmarks"]
        assert stats["inertial_factors_dropped"] == dropped["inertial"]
        # --- state arrays after the bookkeeping: plain copies, bit-exact ---
        st = ctx.state()
        assert np.array_equal(st["knots"], hw.knots), frame
        assert np.array_equal(st["landmarks"], hw.lm_xyz), frame
        win = hw.window()
        ow = ol.OracleWindow(win, radius=radius)
        assert ow.bad == 0
        for got, want in zip(ctx.index_maps(), ow.index_maps()):
            assert np.array_equal(got, want), frame
        # --- two LM iterations on the slid window ---
        recs = ctx.iterate(2)
        for rec in recs:
            o = ow.iterate(apply=True)
            assert rec["spd"] == 1
            assert abs(rec["cost"] - o["cost"]) <= 1e-7 * abs(o["cost"]), (frame, rec, o["cost"])
            assert abs(rec["cost_new"] - o["cost_new"]) <= 1e-6 * abs(o["cost_new"]), (frame, rec, o["cost_new"])
            assert rec["accepted"] == o["accepted"] == 1, (frame, rec)
        radius = recs[-1]["radius"]
        st, so = ctx.state(), ow.state()
        for key in ("knots", "landmarks", "gyro_bias", "accel_bias", "gravity"):
            assert rel_err(st[key], so[key]) < 1e-6, (frame, key)
        hw.knots, hw.lm_xyz = st["knots"].copy(), st["landmarks"].copy()   # carry the optimised state into the next frame
        # (biases / gravity live in the context and in `full` alike: refresh the template the oracle is built from)
        hw.full = dataclasses.replace(hw.full, gyro_bias=st["gyro_bias"].copy(), accel_bias=st["accel_bias"].copy(), gravity=st["gravity"].copy())
    if drop_inertial:
        assert total_dropped["knots"] > 5 and total_dropped["landmarks"] > 20 and total_dropped["inertial"] > 100, total_dropped
    else:   # old inertial residuals keep the leading state elements alive, as in the reference
        assert total_dropped["knots"] == 0 and total_dropped["inertial"] == 0 and total_dropped["landmarks"] > 20, total_dropped
    ctx.close()
