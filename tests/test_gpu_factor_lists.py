"""A setter on a window that appends and a slide have changed on the device, then hb200_bind.

The factor lists live on the device only: each setter replaces its own family there and hb200_bind binds the lists
where they stand.  Per family: load, iterate, append, slide, set a new (shorter, reordered, perturbed) list and bind;
then a context built fresh from the same final lists, state and constancy must give bit-identical copy-outs, index
maps and deterministic systems.  The families the test does not replace come from its own record of the window, in
bound order.
"""
import dataclasses

import numpy as np
import pytest

from hyperslam_b200 import runtime, synthetic

pytestmark = pytest.mark.gpu

FIELDS = dict(pixel=("v_stamp", "v_cam", "v_lm", "v_pixel"), bearing=("b_stamp", "b_cam", "b_lm", "b_bearing"),
              inertial=("i_stamp", "i_meas"), manifold=("m_stamp", "m_sensor", "m_pose"))


def take(win, family, lo, hi):
    """The family's factors with stamps in [lo, hi), in stamp order (so their bound order)."""
    cols = [getattr(win, f) for f in FIELDS[family]]
    sel = np.nonzero((cols[0] >= lo) & (cols[0] < hi))[0]
    sel = sel[np.argsort(cols[0][sel], kind="stable")]
    return [np.ascontiguousarray(c[sel]) for c in cols]


def set_family(ctx, family, cols):
    getattr(ctx, f"set_{family}_factors")(*cols)


def counts(x):
    """Factor counts per family (HB200_PIXEL / _INERTIAL / _BEARING / _MANIFOLD) of a context or of a record."""
    if isinstance(x, runtime.Context):
        return [int(n) for n in x.factor_counts()]
    return [x[f][0].size for f in ("pixel", "inertial", "bearing", "manifold")]


def new_list(family, cols, rng):
    """A replacement list: the first 80% of the current one, perturbed and in random order."""
    n = (4 * cols[0].size) // 5
    order = rng.permutation(n)
    out = [np.ascontiguousarray(c[:n][order]) for c in cols]
    meas = out[-1].copy()
    if family == "manifold":
        meas[:, 4:] += 1e-3
    else:
        meas += {"pixel": 0.25, "bearing": 1e-3, "inertial": 1e-3}[family]
    out[-1] = meas
    return out


@pytest.mark.parametrize("family", list(FIELDS))
def test_setter_after_append_and_slide_matches_a_fresh_context(built, family):
    K0 = 16
    full = synthetic.make_window(order=4, num_knots=K0 + 2, num_landmarks=160, frames_per_landmark=5, num_imu=700, seed=synthetic.SEED_BASE + 4321)
    full = synthetic.add_bearing_and_pose_factors(full, num_bearing=300, num_pose=60)
    st = full.knots[:, 7]
    lo, hi0, hi1 = st[1], st[K0 - 3], st[K0 - 1] - 1e-6   # valid spans of K0 and K0 + 2 knots (order 4)
    mid = 0.5 * (hi0 + hi1)
    # the loaded window: factors in [lo, hi0), the landmarks they observe
    rec = {f: take(full, f, lo, hi0) for f in FIELDS}
    gids = np.unique(np.concatenate([rec["pixel"][2], rec["bearing"][2]]))
    local = {int(g): i for i, g in enumerate(gids)}
    for f in ("pixel", "bearing"):
        rec[f][2] = np.array([local[int(g)] for g in rec[f][2]], dtype=np.int32)
    knot_const = np.zeros(K0, np.uint8)
    knot_const[:2] = 1
    win = dataclasses.replace(full, knots=full.knots[:K0].copy(), landmarks=full.landmarks[gids].copy(), knot_const=knot_const, truth=None,
                              **{name: col for f in FIELDS for name, col in zip(FIELDS[f], rec[f])})
    ctx = runtime.Context(0)
    ctx.load_window(win)
    ctx.iterate(2)
    # append: two state elements, the new landmarks, pixels in [hi0, mid), bearings in [mid, hi1), inertial and pose factors
    ctx.append_knots(2)
    new = dict(pixel=take(full, "pixel", hi0, mid), bearing=take(full, "bearing", mid, hi1), inertial=take(full, "inertial", hi0, hi1),
               manifold=take(full, "manifold", hi0, hi1))
    fresh = [int(g) for g in np.unique(np.concatenate([new["pixel"][2], new["bearing"][2]])) if int(g) not in local]
    ctx.append_landmarks(full.landmarks[fresh])
    for g in fresh:
        local[g] = len(local)
    for f in ("pixel", "bearing"):
        new[f][2] = np.array([local[int(g)] for g in new[f][2]], dtype=np.int32)
    for f in FIELDS:
        getattr(ctx, f"append_{f}_factors")(*new[f])
        rec[f] = [np.ascontiguousarray(np.concatenate([a, b])) for a, b in zip(rec[f], new[f])]
    # slide: landmarks that left the window go with their visual factors, the rest are renumbered
    lower = st[5] + 1e-9
    stats = ctx.slide(lower, drop_inertial=False)
    assert stats["landmarks_dropped"] > 0 and stats["visual_factors_dropped"] > 0, stats
    lm_map = ctx.landmark_map()
    for f in ("pixel", "bearing"):
        keep = lm_map[rec[f][2]] >= 0
        rec[f] = [np.ascontiguousarray(c[keep]) for c in rec[f]]
        rec[f][2] = np.ascontiguousarray(lm_map[rec[f][2]])
    assert counts(ctx) == counts(rec)
    # the setter under test, then a full bind
    rec[family] = new_list(family, rec[family], np.random.default_rng(7))
    set_family(ctx, family, rec[family])
    ctx.bind()
    assert counts(ctx) == counts(rec)
    # the same window built fresh
    state = ctx.state()
    ref = runtime.Context(0)
    ref.set_spline(full.order, state["knots"])
    ref.set_bias_splines(full.bias_order, state["gyro_bias"], state["accel_bias"])
    ref.set_gravity(state["gravity"])
    ref.set_cameras(full.cameras)
    ref.set_imu(full.imu)
    ref.set_landmarks(state["landmarks"])
    ref.set_pose_sensors(full.pose_sensors)
    for f in ("pixel", "inertial", "manifold"):
        set_family(ref, f, rec[f])
    ref.set_bearing_factors(*rec["bearing"], huber=full.huber_bearing)
    ref.bind()
    ref.set_constant((state["knots"][:, 7] <= lower).astype(np.uint8), gravity_const=1, bias_const=full.bias_const)
    for c in (ctx, ref):   # the same solver state on both: the system is damped by the trust region
        c.set_options(full.huber_pixel, full.imu_loss_scale, 1e4)
        c.set_deterministic(True)
    for got, want in zip(ctx.index_maps(), ref.index_maps()):
        assert np.array_equal(got, want)
    for c in (ctx, ref):
        c.evaluate(jacobians=True)
    got, want = ctx.outputs(), ref.outputs()
    assert got.keys() == want.keys()
    for key in want:
        assert np.array_equal(got[key], want[key]), key
    for c in (ctx, ref):
        c.build_system()
    (S, b), (S_ref, b_ref) = ctx.system(), ref.system()
    assert np.array_equal(S, S_ref) and np.array_equal(b, b_ref)
    ctx.close()
    ref.close()
