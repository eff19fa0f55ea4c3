"""Family weight matrices on the device (hb200_set_weights): the weights branch of ExteroceptiveCost::Evaluate.

* outputs: with a dyadic, non-symmetric, non-triangular matrix set for every family, every residual and Jacobian row the
  device returns equals W times the unweighted row of the same context within C u of the weighted row scale
  sum_j |W_ij| max|row j| (C = 64), in every pass -- evaluate, the fused J^T J pass, the deterministic fused pass, and
  the cost-only sweep (hb200_cost against the loss of the weighted residuals) -- and on
  the window shapes of test_gpu_factor_passes that reach the merged lane-group kernel and the one-factor-per-thread
  kernels (S0, S2-separate, S3).  The inertial bias weights stay bit-identical; the cost is the Huber / ScaledLoss /
  plain sum over the weighted residuals.  hb200_factor_evaluate serves W times its unweighted blocks, calibration blocks
  and the dense inertial bias blocks wg[m] W[:, 0:3] / wa[m] W[:, 3:6] included.
* assembly: the packed system equals asmref of the device's own weighted outputs (the inertial bias columns dense,
  weightref) within asmref's componentwise bound, on both inertial J^T J sizes weights reach (the cfg1-sized window,
  which weights move from the scalar kernel to the tensor-core one, and >= 16 384 factors) and in deterministic mode;
  the gyro-accel bias coupling entries are non-zero.
* equivalence: inertial loss_scale s without a matrix against loss_scale 1 with W = sqrt(s) I (s = 1/4, so every
  product with W is exact): on >= 16 384 inertial factors both run the same tensor-core kernel and, deterministic, the
  packed systems and three LM iterations are bit-identical; on the cfg1 window (scalar kernel against tensor-core kernel)
  they agree within the asmref bound and the parity tolerances.  Scaling the pose and inertial matrices by c = 2 on a
  window with only those families (both losses homogeneous in r) scales Sigma by 1/c^2.
* LM iterations against the oracle: three iterations on a cfg1-shaped window with a general matrix for every family; at
  each iteration's start state the oracle evaluates every factor, W is applied in numpy and weightref assembles the
  damped system: the record's cost, the step (backward error on that system) and an accepted step's cost_new (the
  weighted oracle cost at the new state: the trial instantiations) must match.
* sharded through the all-reduce hook: two contexts with the same matrices; partial systems and their rank-order sum
  against weightref within asmref's bound, records and replicated state bit-identical across ranks and equal to one
  context.
* covariance: Sigma with every family weighted against covref's selected inverse of the device's own undamped weighted
  system, landmark marginals included (test_gpu_covariance.check_e2e).  With weights, two deterministic covariance
  computes and two LM runs are bit-identical.
* weights off: set then clear gives outputs, packed system and LM iterations bit-identical to a context that never set
  a matrix; a change between hb200_build_covariance and hb200_compute_covariance gives -2; a bad kind or a non-finite
  entry gives -1 and changes nothing; after a change the captured iteration uses the new matrix.
"""
import math

import numpy as np
import pytest

import asmref as ar
import oracle_lib as ol
import sysref as sr
import weightref as wr
from hyperslam_b200 import runtime, synthetic
from test_gpu_assembly import IMU_MMA_MIN, num_sms, read_system, valid_span, with_imu
from test_gpu_factor_passes import shape_window
from test_gpu_spline_edges import GOLDEN

pytestmark = pytest.mark.gpu

U = 2.0 ** -53
C_ROW = 64
P, I, B, M = runtime.PIXEL, runtime.INERTIAL, runtime.BEARING, runtime.MANIFOLD
FIXTURES = [p for p in GOLDEN if ("euroc" in p or "bearing_pose" in p)]
SHAPES = ("S0", "S2-separate", "S3")


def _ctx(win, weights=None, det=False):
    ctx = runtime.Context(0)
    ctx.load_window(win)
    if det:
        ctx.set_deterministic(True)
    for kind, W in (weights or {}).items():
        ctx.set_weights(kind, W)
    return ctx


def row_check(got, plain, weights):
    """max over keys of |got - W plain| / (C u scale) (<= 1 passes); bias weights must be bit-identical."""
    ref = wr.weigh_outputs(plain, weights)
    scale = wr.abs_weighted_scale(plain, weights)
    worst = {}
    for key, g in got.items():
        if key in ("i_wg", "i_wa"):
            assert np.array_equal(g, plain[key]), key
            continue
        g, r = np.asarray(g), np.asarray(ref[key])
        s = scale[key]
        s = s.reshape(s.shape + (1,) * (g.ndim - s.ndim))
        err = np.abs(g - r) / (C_ROW * U * np.maximum(s, 1e-300))
        worst[key] = float(err.max()) if err.size else 0.0
    return worst


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("path", FIXTURES, ids=[p.split("/")[-1] for p in FIXTURES])
def test_weighted_outputs_every_pass(built, record_property, path, shape):
    win = shape_window(path, shape, num_sms())[1]
    weights = wr.all_weights(seed=11)
    plain_ctx = _ctx(win)
    plain_ctx.evaluate()
    plain = plain_ctx.outputs()
    plain_ctx.close()
    for tag, det in (("evaluate", False), ("fused", False), ("deterministic", True)):
        ctx = _ctx(win, weights, det=det)
        try:
            ctx.evaluate()
            if tag != "evaluate":
                ctx.build_system()
            got = ctx.outputs()
            worst = row_check(got, plain, weights)
            record_property(tag, worst)
            assert all(v <= 1.0 for v in worst.values()), (tag, worst)
            cost = ctx.cost()
            ref = wr.cost(got, win)
            assert abs(cost - ref) <= 1e-11 * abs(ref), (tag, cost, ref)
        finally:
            ctx.close()


@pytest.mark.parametrize("order", [4, 6])
def test_factor_evaluate_weighted_blocks(built, order):
    """hb200_factor_evaluate: every block of a weighted factor, calibration blocks included, is W times the unweighted
    block; the bias blocks are the dense wg[m] W[:, 0:3] / wa[m] W[:, 3:6]."""
    import test_gpu_calibration as gc
    win = gc.make_window(order, seed_off=order)
    weights = wr.all_weights(seed=5)
    a, b = gc.make_ctx(win), _ctx(win, weights)
    try:
        b.evaluate()
        maps = a.index_maps()
        k, kb = win.order, win.bias_order
        for kind in (P, I, B, M):
            W = weights[kind]
            n = {P: len(win.v_stamp), I: len(win.i_stamp), B: len(win.b_stamp), M: len(win.m_stamp)}[kind]
            assert n > 0, kind
            for f in range(min(n, 4)):
                if kind == M:
                    base = gc.knot_base(win, win.m_stamp[f])
                    blocks = [win.knots[base + m] for m in range(k)] + [win.pose_sensors[win.m_sensor[f]]]
                elif kind == B:
                    base, cam = gc.knot_base(win, win.b_stamp[f]), win.cameras[win.b_cam[f]]
                    blocks = [win.knots[base + m] for m in range(k)] + [cam[:7], cam[7:11], cam[11:15], win.landmarks[win.b_lm[f]]]
                else:
                    blocks = gc.blocks_of(win, kind, f, maps)[0]
                r0, J0 = a.factor_evaluate(kind, f, blocks)
                r1, J1 = b.factor_evaluate(kind, f, blocks)
                assert np.abs(r1 - W @ r0).max() <= C_ROW * U * (np.abs(W) @ np.abs(r0)).max()
                # a Jacobian row's rounding is relative to the row's scale over all its blocks (a control point with a
                # tiny basis weight has a block far below it)
                rows = np.max([np.abs(x).max(1) for x in J0], axis=0)
                bound = C_ROW * U * (np.abs(W) @ rows)[:, None]
                for j, (x0, x1) in enumerate(zip(J0, J1)):
                    if kind == I and k + 5 <= j < k + 5 + 2 * kb:
                        gyro = j < k + 5 + kb
                        wv = x0[0, 0] if gyro else x0[3, 0]
                        want = np.zeros((6, 4))
                        want[:, :3] = wv * (W[:, 0:3] if gyro else W[:, 3:6])
                        assert np.array_equal(x1, want), (kind, f, j)
                        continue
                    assert (np.abs(x1 - W @ x0) <= bound).all(), (kind, f, j)
    finally:
        a.close(); b.close()


def _imu_window(order, ni, seed):
    win = synthetic.make_window(order=order, num_knots=30, num_landmarks=60, num_imu=0, bias_dt=1.0, seed=synthetic.SEED_BASE + 900 + seed)
    lo, hi = valid_span(win)
    u = np.sort(np.random.default_rng(seed).random(ni))
    return with_imu(win, lo + u * (hi - lo) * (1 - 1e-9), seed=seed)


def _cfg1(order=4):
    return synthetic.make_window(order=order, num_knots=50, num_landmarks=300, num_imu=2000, seed=synthetic.SEED_BASE + 950 + order,
                                 constant_knots=2)


@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("case", ["cfg1", "large"])
@pytest.mark.parametrize("order", [4, 6])
def test_weighted_assembly(built, record_property, order, case, det):
    win = _cfg1(order) if case == "cfg1" else _imu_window(order, IMU_MMA_MIN + 100, order)
    weights = wr.all_weights(seed=23)
    radius = 1e4
    ctx = _ctx(win, weights, det=det)
    try:
        ctx.evaluate()
        ctx.build_system()
        buf = read_system(ctx)
        prob = ar.problem(ctx.outputs(), win, ctx.index_maps())
        beta = ctx.bandwidth()
        ran = {name for name, _ in ctx.profile_iteration(reps=1)}
    finally:
        ctx.close()
    ref = wr.assemble(prob, radius, W_inertial=weights[I])
    res = ar.compare(buf, ref, beta)
    record_property("compare", res)
    bad = {k: v for k, v in res.items() if k not in ("nonzero_outside", "finite") and not v <= 1.0}
    assert res["finite"] and res["nonzero_outside"] == 0 and not bad, res
    assert any("inertial_hessian_mma" in n for n in ran) and not any(n.startswith("inertial_hessian_kernel") or n.startswith("inertial_hessian_det") for n in ran), ran
    K, Kbg = ref["K"], ref["Kbg"]
    o_bg, o_ba = 6 * K, 6 * K + 3 * Kbg
    coupling = ref["S"][o_ba:o_ba + 3 * ref["Kba"], o_bg:o_bg + 3 * Kbg]
    assert np.count_nonzero(coupling) > 0   # the gyro-accel bias coupling the unweighted structure lacks


def _records(ctx, n=3):
    return [tuple(r.values()) for r in ctx.iterate(n)]


@pytest.mark.parametrize("order", [4, 6])
def test_loss_scale_equals_sqrt_weight_large(built, order):
    """>= 16 384 inertial factors, deterministic: bit-identical systems and LM iterations."""
    win = _imu_window(order, IMU_MMA_MIN + 100, 40 + order)
    win.imu_loss_scale = 0.25
    a = _ctx(win, det=True)
    win1 = synthetic.Window(**{**win.__dict__, "imu_loss_scale": 1.0})
    b = _ctx(win1, {I: 0.5 * np.eye(6)}, det=True)
    try:
        for c in (a, b):
            c.evaluate(); c.build_system()
        assert np.array_equal(read_system(a), read_system(b))
        assert _records(a) == _records(b)
        assert all(np.array_equal(x, y) for x, y in zip(a.state(), b.state()))
    finally:
        a.close(); b.close()


def test_loss_scale_equals_sqrt_weight_cfg1(built):
    """cfg1: scalar J^T J kernel without a matrix against the tensor-core kernel with one."""
    win = _cfg1(4)
    s = 0.25
    win.imu_loss_scale = s
    win1 = synthetic.Window(**{**win.__dict__, "imu_loss_scale": 1.0})
    a, b = _ctx(win), _ctx(win1, {I: math.sqrt(s) * np.eye(6)})
    try:
        for c in (a, b):
            c.evaluate(); c.build_system()
        prob = ar.problem(b.outputs(), win1, b.index_maps())
        ref = wr.assemble(prob, 1e4, W_inertial=math.sqrt(s) * np.eye(6))
        for c in (a, b):
            res = ar.compare(read_system(c), ref, c.bandwidth())
            bad = {k: v for k, v in res.items() if k not in ("nonzero_outside", "finite") and not v <= 1.0}
            assert res["finite"] and not bad, res
        ra, rb = a.iterate(3), b.iterate(3)
        for x, y in zip(ra, rb):
            for key in ("cost", "cost_new", "model_change"):
                assert abs(x[key] - y[key]) <= 1e-9 * abs(x[key]) + 1e-300, (key, x, y)
            assert x["accepted"] == y["accepted"]
    finally:
        a.close(); b.close()


def test_pose_and_inertial_weight_scale_covariance(built):
    """Pose and inertial factors only (both losses homogeneous in r): W = c I on both scales Sigma by 1 / c^2 (c = 2).
    Both contexts set the matrices (c = 1: the identity), so both run the same kernels and every operation scales by a
    power of two."""
    import covref as cr
    from test_gpu_covariance import e2e_window
    win = e2e_window(4, num_landmarks=0, bearing=0, pose=40, seed=3)
    win.knot_const = np.zeros(win.knots.shape[0], np.uint8)
    win.knot_const[:4] = 1
    win.knot_const[cr.untouched_knots(win)] = 1
    out = []
    for c in (1.0, 2.0):
        ctx = _ctx(win, {M: c * np.eye(6), I: c * np.eye(6)}, det=True)
        try:
            ctx.build_covariance()
            info = ctx.compute_covariance()
            assert info["status"] == 0, info
            out.append(ctx.covariance_packed()[0].copy())
        finally:
            ctx.close()
    assert np.abs(out[1] * 4.0 - out[0]).max() <= 1e-12 * np.abs(out[0]).max()


def test_weighted_covariance_and_lm_are_deterministic(built):
    from test_gpu_covariance import e2e_window
    win = e2e_window(4, seed=5)
    weights = wr.all_weights(seed=31)
    res = []
    for _ in range(2):
        ctx = _ctx(win, weights, det=True)
        try:
            ctx.build_covariance()
            info = ctx.compute_covariance()
            assert info["status"] == 0, info
            res.append((ctx.covariance_packed()[0].copy(), _records(ctx)))
        finally:
            ctx.close()
    assert np.array_equal(res[0][0], res[1][0])
    assert res[0][1] == res[1][1]


def test_weights_off_is_bit_identical(built):
    win = _cfg1(4)
    a = _ctx(win, det=True)
    b = _ctx(win, wr.all_weights(seed=2), det=True)
    try:
        for kind in (P, I, B, M):
            b.set_weights(kind, None)
        for c in (a, b):
            c.evaluate()
        oa, ob = a.outputs(), b.outputs()
        assert all(np.array_equal(oa[k], ob[k]) for k in oa)
        for c in (a, b):
            c.build_system()
        assert np.array_equal(read_system(a), read_system(b))
        assert _records(a) == _records(b)
    finally:
        a.close(); b.close()


def test_set_weights_errors_and_invalidation(built):
    win = _cfg1(4)
    ctx = _ctx(win)
    lib = ctx.lib
    try:
        ctx.evaluate()
        base = ctx.outputs()
        bad = np.eye(6)
        bad[2, 3] = np.nan
        assert lib.hb200_set_weights(ctx.h, 7, runtime._d(np.eye(6))) == -1
        assert lib.hb200_set_weights(ctx.h, -1, None) == -1
        assert lib.hb200_set_weights(ctx.h, I, runtime._d(bad)) == -1
        bad[2, 3] = np.inf
        assert lib.hb200_set_weights(ctx.h, I, runtime._d(bad)) == -1
        ctx.evaluate()
        after = ctx.outputs()
        assert all(np.array_equal(base[k], after[k]) for k in base)
        # a change between build and compute drops the pending build
        ctx.build_covariance()
        ctx.set_weights(P, np.diag([2.0, 0.5]))
        info = runtime.CovarianceInfo()
        assert lib.hb200_compute_covariance(ctx.h, runtime.C.byref(info)) == -2
        # setting the current value again keeps a built system
        ctx.evaluate(); ctx.build_system()
        ctx.set_weights(P, np.diag([2.0, 0.5]))
        ctx.solve()
    finally:
        ctx.close()


def test_graph_follows_a_change(built):
    """An iteration captured before set_weights does not replay the old matrix: the same calls on a context without
    graph capture give bit-identical records (deterministic mode)."""
    win = _cfg1(4)
    W = wr.all_weights(seed=3)
    recs = []
    for use_graph in (True, False):
        ctx = runtime.Context(0, use_graph=use_graph)
        try:
            ctx.load_window(win)
            ctx.set_deterministic(True)
            first = _records(ctx, 1)
            for kind, m in W.items():
                ctx.set_weights(kind, m)
            recs.append((first, _records(ctx, 2)))
        finally:
            ctx.close()
    assert recs[0] == recs[1]
    assert recs[0][1][0][0] != recs[0][0][0][0]   # the weighted cost differs from the unweighted one


# ---- LM iterations against the oracle's factors --------------------------------------------------------------------
def _at_state(win, st):
    return synthetic.Window(**{**win.__dict__, **{k: st[k] for k in ("knots", "gyro_bias", "accel_bias", "gravity", "landmarks")}})


def oracle_weighted(win, st, weights):
    """The oracle's (unweighted) factor outputs at state st, weighted in numpy, and its index maps."""
    ow = ol.OracleWindow(_at_state(win, st))
    return wr.weigh_outputs(ow.evaluate(), weights), ow.index_maps()


def lm_window(order):
    base = synthetic.make_config(1, scale=0.25, order=order, constant_knots=2)
    return synthetic.add_bearing_and_pose_factors(base, num_bearing=200, num_pose=12, seed=synthetic.SEED_BASE + 970 + order)


@pytest.mark.parametrize("order", [4, 6])
def test_lm_iterations_against_weighted_oracle(built, record_property, order):
    """Three LM iterations on a cfg1-shaped window with all four families weighted by general matrices.  At the state each
    iteration starts from, the oracle evaluates every factor (no device code), W is applied in numpy and asmref / weightref
    assemble the damped system at the iteration's radius.  The device's record must match: cost = the weighted oracle
    cost, the step solves the reference system (backward error), and an accepted step's cost_new is the weighted oracle
    cost at the state it left -- the trial (cost-only) instantiations of every family checked against the oracle."""
    win = lm_window(order)
    weights = wr.all_weights(seed=41)
    K, Kbg, Kba = win.knots.shape[0], win.gyro_bias.shape[0], win.accel_bias.shape[0]
    fixed = sr.fixed_mask(K, Kbg, Kba, win.knot_const, win.bias_const, win.gravity_const)
    ctx = _ctx(win, weights)
    radius, accepted = 1e4, 0
    try:
        for it in range(3):
            st = ctx.state()
            out, maps = oracle_weighted(win, st, weights)
            rec = ctx.iterate(1)[0]
            dp, _ = ctx.delta()
            st1 = ctx.state()
            cost = wr.cost(out, win)
            assert abs(rec["cost"] - cost) <= 1e-7 * cost, (it, rec, cost)
            ref = wr.assemble(ar.problem(out, win, maps), radius, W_inertial=weights[I], dtype=np.float64)
            A, rhs = sr.damped_masked(ref["S"], ref["b"], ref["g"], ref["diagH"], fixed, radius)
            bwd = sr.backward_error(A, rhs, dp)
            record_property(f"backward_error_{it}", float(bwd))
            assert bwd < 1e-8, (it, bwd)
            if rec["accepted"]:
                accepted += 1
                out1, _ = oracle_weighted(win, st1, weights)
                cost_new = wr.cost(out1, win)
                assert abs(rec["cost_new"] - cost_new) <= 1e-6 * abs(cost_new), (it, rec, cost_new)
            else:
                assert all(np.array_equal(st[k], st1[k]) for k in st)
            radius = rec["radius"]
    finally:
        ctx.close()
    assert accepted >= 1


# ---- sharded through the all-reduce hook ----------------------------------------------------------------------------
def test_sharded_weights_through_the_hook(built, record_property):
    """Weights are replicated configuration: two contexts holding factor shards of one window, both with the same
    matrices.  Their partial systems against weightref within asmref's bound and, summed in rank order, against the whole
    window's restatement; LM iterations through the hook bit-identical across ranks and equal to one context."""
    from test_gpu_sharded import HostReducer, check_record, on_ranks, open_ranks
    win = synthetic.make_config(1, scale=0.25, num_knots=51, constant_knots=2)
    win = synthetic.add_bearing_and_pose_factors(win, num_bearing=100, num_pose=12, seed=synthetic.SEED_BASE + 990)
    weights = wr.all_weights(seed=43)
    win.weights = weights
    world = 2
    shards = [win.shard(r, world) for r in range(world)]
    for s_ in shards:
        s_.weights = weights
    ctxs, own, beta = open_ranks(shards)
    try:
        bufs, refs = [], []
        for c, s_ in zip(ctxs, shards):
            c.evaluate()
            c.build_system()
            bufs.append(read_system(c))
            refs.append(wr.assemble(ar.problem(c.outputs(), s_, c.index_maps()), 1e4, W_inertial=weights[I]))
            res = ar.compare(bufs[-1], refs[-1], beta)
            assert res["finite"] and res["nonzero_outside"] == 0 and all(v <= 1.0 for k, v in res.items() if k not in ("nonzero_outside", "finite")), res
        res = ar.compare_summed_buffers(bufs, refs, beta)
        record_property("partial_sum", res)
        assert res["finite"] and all(v <= 1.0 for k, v in res.items() if k not in ("nonzero_outside", "finite")), res
        red = HostReducer(world)
        red.attach(ctxs)
        recs = on_ranks(red, ctxs, lambda r, c: c.iterate(3))
        states = [c.state() for c in ctxs]
    finally:
        for c in ctxs:
            c.close()
    keys = ("cost", "cost_new", "rho", "radius", "accepted", "spd")
    assert [[x[k] for k in keys] for x in recs[1]] == [[x[k] for k in keys] for x in recs[0]]
    for key in ("knots", "gyro_bias", "accel_bias", "gravity"):
        assert np.array_equal(states[1][key], states[0][key]), key
    single = runtime.Context(0)
    try:
        single.load_window(win)
        srecs = single.iterate(3)
    finally:
        single.close()
    for a, b in zip(recs[0], srecs):
        check_record(a, b)


# ---- covariance against covref of the device's own weighted system ----------------------------------------------------
@pytest.mark.parametrize("order", [4, 6])
def test_weighted_covariance_against_covref(built, record_property, order):
    """Sigma with every family weighted = covref's selected inverse of the device's own undamped weighted system, landmark
    marginals included, as test_gpu_covariance checks it unweighted (its asmref leg, which knows no dense bias columns, is
    replaced by weightref's)."""
    from test_gpu_covariance import check_e2e, e2e_window
    win = e2e_window(order, seed=60 + order)
    win.weights = wr.all_weights(seed=47)
    check_e2e(win, record_property, asm=False)
