"""Marginal covariances on the device (need an H100): hb200_build_covariance / hb200_compute_covariance /
hb200_get_covariance / hb200_interpolate_covariance against tests/covref.py.

* injected systems: build, overwrite the packed buffer with a synthetic band + arrow system (tests/sysref.py), compute;
  the band / arrow / corner entries equal covref's long-double selected inverse within 8 n eps kappa(A_hat) (metric
  |dSigma_ij| / sqrt(Sigma_ii Sigma_jj)), constant dofs are exactly 0, two computes are bit-identical, the widest window
  that fits shared memory runs and the first one past it gets -6;
* end to end on windows with pixel, bearing, pose and IMU factors: the covariance of the device's own undamped system
  (read back between build and compute) and of asmref's long-double restatement at mu = 0, the landmark marginals, and
  the kernels that ran (schur_group_kernel on the K = 500 window with 8192 landmarks);
* a build made stale by a change of the window (landmarks, an evaluation, constants) is refused with -2;
* failures (gauge not fixed, biases without IMU factors, a single-observation landmark) are reported with finite outputs
  and leave the previous results in place (packed, landmark blocks and both interpolations, bit for bit); an unobserved
  landmark gets a zero block;
* the linearisation point of a build is committed only by a successful compute: a repeated compute, failed computes and
  a return to an earlier window give every reader what it should see (deterministic assembly, bit for bit);
* the interpolated pose covariance equals J(t) Sigma J(t)^T of covref within 1e-11 in the correlation metric, also where
  the knot increments straddle the small-angle switches of the SO(3) coefficients;
* the LM path is untouched: iterate() with a covariance computed in between differs from a plain run by no more than
  twice the spread of three plain runs (the assembly's atomics), hb200_get_system refuses after the covariance build, the iteration's kernel list is
  unchanged.
"""
import numpy as np
import pytest

import asmref as ar
import covref as cr
import sysref as sr
from hyperslam_b200 import runtime, synthetic

pytestmark = pytest.mark.gpu

SMEM_LIMIT = 220 * 1024


def cov_smem_bytes(beta, m):
    """cov_smem_doubles (hb200_cov.cuh) in bytes."""
    w = 6 * (beta + 1) + m
    return 8 * (w * (w | 1) + 18 * w + 108)


def read_system(ctx):
    import torch
    ptr, count = ctx.system_device_ptr()

    class _Arr:
        __cuda_array_interface__ = dict(shape=(count,), typestr="<f8", data=(ptr, False), version=2)
    ctx.synchronize()
    out = torch.as_tensor(_Arr(), device="cuda").cpu().numpy().copy()
    torch.cuda.synchronize()
    return out


def inject(ctx, buf):
    import torch
    ptr, count = ctx.system_device_ptr()
    assert count == buf.size

    class _Arr:
        __cuda_array_interface__ = dict(shape=(count,), typestr="<f8", data=(ptr, False), version=2)
    ctx.synchronize()
    torch.as_tensor(_Arr(), device="cuda").copy_(torch.from_numpy(buf))
    torch.cuda.synchronize()


def solver_window(K, Kbg, Kba, knot_const=(), seed=0):
    """Order-4 window with K knots, a few pose factors, no landmarks or IMU factors, bias splines of Kbg / Kba knots."""
    base = synthetic.make_window(order=4, num_knots=K, num_landmarks=0, num_imu=0, seed=synthetic.SEED_BASE + 1900 + seed, noise=False)
    win = synthetic.add_bearing_and_pose_factors(base, num_pose=8, seed=synthetic.SEED_BASE + 1950 + seed)

    def bias(Kb):
        a = np.zeros((Kb, 4))
        a[:, 3] = win.knots[0, 7] + np.arange(Kb) * 1.0
        return a
    win.gyro_bias, win.accel_bias = bias(Kbg), bias(Kba)
    kc = np.zeros(K, dtype=np.uint8)
    kc[list(knot_const)] = 1
    win.knot_const, win.bias_const, win.gravity_const = kc, 0, 0
    return win


def run_injected(K, beta, Kbg, Kba, seed, report, force_dense=False):
    m = 3 * (Kbg + Kba) + 2
    n = 6 * K + m
    win = solver_window(K, Kbg, Kba, knot_const=(0, K // 2, K - 1), seed=seed)
    ctx = runtime.Context(0, force_dense=force_dense)
    try:
        ctx.load_window(win)
        ctx.set_min_bandwidth(beta)
        assert ctx.bandwidth() == beta
        ctx.build_covariance()
        S, b, g, dH = sr.make_system(K, beta, m, seed=seed)
        inject(ctx, sr.pack_system(S, b, g, dH, K, beta, m))
        l0 = ctx.launch_count
        info = ctx.compute_covariance()
        assert ctx.launch_count - l0 == 1          # cov_selinv_kernel alone (no landmarks)
        assert info["status"] == 0 and (info["K"], info["beta"], info["m"], info["L"]) == (K, beta, m, 0), info
        packed, _, _ = ctx.covariance_packed()
        info2 = ctx.compute_covariance()
        packed2, _, _ = ctx.covariance_packed()
    finally:
        ctx.close()
    assert np.array_equal(packed.view(np.int64), packed2.view(np.int64))
    assert info2["min_pivot_ratio"] == info["min_pivot_ratio"]
    fixed = sr.fixed_mask(K, Kbg, Kba, win.knot_const)
    ref, P, minpiv, bad = cr.selected_inverse(S, K, beta, m, fixed)
    assert bad == -1
    got = cr.packed_to_dense(packed, K, beta, m)
    assert np.isfinite(packed).all()
    assert np.all(got[fixed] == 0) and np.all(got[:, fixed] == 0)
    # padding rows of the band (past the last pose dof) are 0
    Lay = sr.layout(K, beta, m)
    idx, row, _ = sr._band_slots(Lay)
    pad = np.ones(Lay["oA"], bool)
    pad[idx] = False
    assert np.all(packed[:Lay["oA"]][pad] == 0)
    kap = cr.kappa(S, fixed)
    err = cr.cov_error(got, ref, P)
    bound = sr.forward_bound(n, kap)
    for k, v in dict(n=n, err=err, bound=bound, kappa=kap, min_pivot=info["min_pivot_ratio"], ref_min_pivot=minpiv).items():
        report(k, v)
    assert err < bound, (err, bound, kap)
    assert abs(info["min_pivot_ratio"] - minpiv) <= 1e-6 * minpiv + 1e-12
    return info


SHAPES = [(K, beta, Kbg, Kba) for beta in (3, 5, 12) for Kbg, Kba in ((4, 4), (9, 8)) for K in sorted({beta + 1, 2 * beta + 3, 40})]
SHAPES += [(40, 8, 9, 8), (500, 8, 9, 8)]


@pytest.mark.parametrize("K,beta,Kbg,Kba", SHAPES, ids=[f"b{b}-m{3 * (g + a) + 2}-K{K}" for K, b, g, a in SHAPES])
def test_injected_system(built, record_property, K, beta, Kbg, Kba):
    run_injected(K, beta, Kbg, Kba, seed=1000 * K + 10 * beta + Kbg, report=record_property,
                 force_dense=(beta == 12 and Kbg == 9))


def widest_beta(m):
    return max(b for b in range(1, 40) if cov_smem_bytes(b, m) <= SMEM_LIMIT)


def test_widest_window_and_first_past_it(built, record_property):
    """m = 53: the widest band that fits one CTA's shared memory runs (dense LM solver: the band solvers' own plans do
    not take such wide bands); one more block column gets -6."""
    Kbg, Kba = 9, 8
    m = 53
    beta = widest_beta(m)
    record_property("widest_beta", beta)
    record_property("smem_bytes", cov_smem_bytes(beta, m))
    run_injected(beta + 4, beta, Kbg, Kba, seed=77, report=record_property, force_dense=True)
    win = solver_window(beta + 5, Kbg, Kba, knot_const=(0,), seed=78)
    ctx = runtime.Context(0, force_dense=True)
    try:
        ctx.load_window(win)
        ctx.set_min_bandwidth(beta + 1)
        with pytest.raises(runtime.HB200Error, match="hb200 error -6"):
            ctx.build_covariance()
    finally:
        ctx.close()


# ---- end to end -----------------------------------------------------------------------------------------------------
def e2e_window(order, num_knots=50, num_landmarks=1000, num_imu=2000, bias_const=0, bearing=1000, pose=20, seed=0, frames=5):
    base = synthetic.make_window(order=order, num_knots=num_knots, num_landmarks=num_landmarks, num_imu=num_imu, frames_per_landmark=frames,
                                 seed=synthetic.SEED_BASE + 2000 + seed)
    win = synthetic.add_bearing_and_pose_factors(base, num_bearing=bearing, num_pose=pose, seed=synthetic.SEED_BASE + 2050 + seed)
    win.knot_const = np.zeros(num_knots, np.uint8)
    win.knot_const[:order] = 1
    win.knot_const[cr.untouched_knots(win)] = 1
    win.bias_const = bias_const
    return win


def device_covariance(ctx):
    """build, read the undamped system, compute; returns (system buffer, info, packed, landmarks, launches of the compute)."""
    ctx.build_covariance()
    buf = read_system(ctx)
    l0 = ctx.launch_count
    info = ctx.compute_covariance()
    launches = ctx.launch_count - l0
    packed, lm, _ = ctx.covariance_packed() if info["status"] == 0 else (None, None, None)
    return buf, info, packed, lm, launches


def check_e2e(win, report, asm=True):
    ctx = runtime.Context(0)
    try:
        ctx.load_window(win)
        buf, info, packed, lm, launches = device_covariance(ctx)
        out = ctx.outputs()
        maps = ctx.index_maps()
        beta = ctx.bandwidth()
        knots = ctx.state()["knots"]
        kernels = {nm for nm, _ in ctx.profile_iteration(reps=1)}   # the assembly kernels the build shares with the LM step
    finally:
        ctx.close()
    K, Kbg, Kba, L = win.knots.shape[0], win.gyro_bias.shape[0], win.accel_bias.shape[0], win.landmarks.shape[0]
    m = 3 * (Kbg + Kba) + 2
    n = 6 * K + m
    assert info["status"] == 0, info
    assert launches == (2 if L else 1)     # cov_selinv_kernel + cov_landmark_kernel
    fixed = sr.fixed_mask(K, Kbg, Kba, win.knot_const, win.bias_const, win.gravity_const)
    S_dev, *_ = sr.unpack_system(buf, K, beta, m)
    ref, P, minpiv, bad = cr.selected_inverse(S_dev, K, beta, m, fixed)
    assert bad == -1
    kap = cr.kappa(S_dev, fixed)
    got = cr.packed_to_dense(packed, K, beta, m)
    fam = sr.families(K, Kbg, Kba)
    err = cr.cov_error(got, ref, P)
    bound = sr.forward_bound(n, kap)
    for k, v in dict(n=n, beta=beta, kappa=kap, min_pivot=info["min_pivot_ratio"], threshold=cr.MIN_PIVOT, err_own=err, bound_own=bound).items():
        report(k, v)
    print(f"K {K} order {win.order} bias_const {win.bias_const}: min pivot ratio {info['min_pivot_ratio']:.3e} (threshold {cr.MIN_PIVOT:.0e}), "
          f"kappa {kap:.3e}, err {err:.3e} / {bound:.3e}")
    assert err < bound
    assert np.all(got[fixed] == 0) and np.all(got[:, fixed] == 0)
    assert info["min_pivot_ratio"] > 100 * cr.MIN_PIVOT
    res = dict(got=got, ref=ref, knots=knots, beta=beta, kappa=kap, fixed=fixed, lm=lm, kernels=kernels)
    p = ar.problem(out, win, maps)
    # landmark marginals from the device's own Sigma and factor outputs
    lm_ref = cr.landmark_marginals(p, ref)
    seen = np.abs(lm_ref).reshape(L, -1).max(1) > 0
    errs = np.array([cr.cov_error(lm[l], lm_ref[l]) for l in np.nonzero(seen)[0]])
    report("err_landmarks", float(errs.max()))
    assert np.isfinite(lm).all() and np.all(lm[~seen] == 0)
    assert errs.max() < 10 * bound, (errs.max(), bound)
    if asm:
        a = ar.assemble(p, np.inf)
        keep = ~fixed   # (untouched knots have a zero diagonal)
        eS = sr.entry_error(S_dev[np.ix_(keep, keep)], a["S"].astype(np.float64)[np.ix_(keep, keep)])
        ref_a, _, _, bad_a = cr.selected_inverse(a["S"], K, beta, m, fixed)
        assert bad_a == -1
        err_a = cr.cov_error(got, ref_a, P)
        bound_a = kap * (n * eS + 8 * n * sr.EPS)
        report("err_asmref", err_a)
        report("bound_asmref", bound_a)
        assert err_a < bound_a, (err_a, bound_a, eS)
    return res


@pytest.mark.parametrize("order", [4, 6])
def test_e2e_cfg1_shaped(built, record_property, order):
    res = check_e2e(e2e_window(order, seed=order), record_property)
    # interpolated covariance: knot stamps, mid-segment, segment boundaries, both ends of the valid span, outside
    win = e2e_window(order, seed=order)
    kt = win.knots[:, 7]
    left = (order - 1) // 2
    # the span hb200_interpolate accepts (segment_base): kt[left] <= t < kt[K - k + left + 1]
    lo, hi = kt[left], kt[len(kt) - order + left + 1]
    inside = np.concatenate([[lo, np.nextafter(hi, -np.inf)], kt[left + 1:left + 6], 0.5 * (kt[10:15] + kt[11:16]), kt[20:22] + 1e-12])
    stamps = np.concatenate([inside, [np.nextafter(lo, -np.inf), hi]])
    ctx = runtime.Context(0)
    try:
        ctx.load_window(win)
        ctx.build_covariance()
        assert ctx.compute_covariance()["status"] == 0
        cov, bad = ctx.interpolate_covariance(stamps)
    finally:
        ctx.close()
    assert bad == 2 and np.all(cov[-2:] == 0)
    # J(t) is evaluated independently here (numpy, from the knots) and on the device (from the knot table); measured on an
    # H100: 1.2e-12 .. 1.7e-12 over runs at orders 4 and 6 (the assembly's atomics change the last bits of Sigma)
    worst = 0.0
    for i, t in enumerate(inside):
        want = cr.interpolated(res["knots"], order, t, res["got"])
        worst = max(worst, cr.cov_error(cov[i], want))
    record_property("err_interpolated", worst)
    print(f"order {order}: interpolated covariance, correlation error {worst:.3e}")
    assert worst < 1e-11, worst


NEAR_STATIONARY = [1.05e-4, 1.2e-4, 0.0, 1e-9, 5e-8, 2e-7, 1.05e-3, 5e-5, 1.3e-4, 9e-4, 1.1e-4]


@pytest.mark.parametrize("order", [4, 6])
def test_interpolated_covariance_near_stationary(built, record_property, order):
    """J(t) Sigma J(t)^T where the platform barely turns: knots 10..20 step by the increments above (0 = identical knots),
    which put lambda_j d_j and d_j on both sides of the small-angle switches of the SO(3) coefficients."""
    win = e2e_window(order, num_knots=30, num_landmarks=300, num_imu=600, bearing=100, pose=10, seed=40 + order)
    rng = np.random.default_rng(order)
    for i, inc in enumerate(NEAR_STATIONARY, start=10):
        axis = rng.normal(size=3)
        R = synthetic.quat_to_rot(win.knots[i - 1, None, :4])[0] @ synthetic.so3_exp(inc * axis[None] / np.linalg.norm(axis))[0]
        q = win.knots[i - 1, :4] if inc == 0 else synthetic.rot_to_quat(R[None])[0]
        win.knots[i, :4] = q if np.dot(q, win.knots[i - 1, :4]) >= 0 else -q
    kt = win.knots[:, 7]
    inside = np.concatenate([kt[10:21], kt[10:21] + 0.3 * (kt[11:22] - kt[10:21]), np.nextafter(kt[11:22], -np.inf)])
    ctx = runtime.Context(0)
    try:
        ctx.load_window(win)
        ctx.build_covariance()
        info = ctx.compute_covariance()
        assert info["status"] == 0, info
        packed, _, _ = ctx.covariance_packed()
        beta, knots = ctx.bandwidth(), ctx.state()["knots"]
        cov, bad = ctx.interpolate_covariance(inside)
    finally:
        ctx.close()
    assert bad == 0
    K, m = win.knots.shape[0], 3 * (win.gyro_bias.shape[0] + win.accel_bias.shape[0]) + 2
    got = cr.packed_to_dense(packed, K, beta, m)
    worst = max(cr.cov_error(cov[i], cr.interpolated(knots, order, t, got)) for i, t in enumerate(inside))
    record_property("err_interpolated", worst)
    assert worst < 1e-11, worst


def test_e2e_bias_const(built, record_property):
    """bias_const = 1, as in the reference's live configuration."""
    check_e2e(e2e_window(4, bias_const=1, seed=11), record_property)


def test_e2e_large_window_group_path(built, record_property):
    """K = 500 with 8192 landmarks: the Schur complement runs in schur_group_kernel; band, arrow, corner and landmark blocks
    compared on the device's own system (the long-double assembly of a 3000-dof window is left to test_gpu_assembly)."""
    win = e2e_window(4, num_knots=500, num_landmarks=8192, num_imu=4000, bearing=0, pose=40, seed=21, frames=3)
    res = check_e2e(win, record_property, asm=False)
    assert res["lm"].shape == (8192, 3, 3)
    assert "schur_group_kernel" in res["kernels"] and "schur_kernel" not in res["kernels"], res["kernels"]


def test_stale_build_is_refused(built, record_property):
    """Anything that changes the window between build and compute -- new landmarks, a new evaluation, other constants --
    makes the compute refuse (-2) instead of reading factor outputs of another shape."""
    win = e2e_window(4, num_knots=30, num_landmarks=200, num_imu=800, bearing=100, pose=10, seed=51)
    ctx = runtime.Context(0)
    try:
        ctx.load_window(win)
        ctx.build_covariance()
        ctx.set_landmarks(np.vstack([win.landmarks, win.landmarks[:1] + 1.0]))
        with pytest.raises(runtime.HB200Error, match="hb200 error -2"):
            ctx.compute_covariance()
        ctx.load_window(win)
        ctx.build_covariance()
        ctx.evaluate()
        with pytest.raises(runtime.HB200Error, match="hb200 error -2"):
            ctx.compute_covariance()
        ctx.build_covariance()
        ctx.set_constant(win.knot_const, 1, 0)
        with pytest.raises(runtime.HB200Error, match="hb200 error -2"):
            ctx.compute_covariance()
        ctx.build_covariance()
        assert ctx.compute_covariance()["status"] == 0
    finally:
        ctx.close()


# ---- failures ---------------------------------------------------------------------------------------------------------
def failure_window(pose=10):
    return e2e_window(4, num_knots=30, num_landmarks=200, num_imu=800, bearing=100, pose=pose, seed=31)


def gauge_free_window():
    """No constant knots, no pose factors (yaw and translation free): the compute fails with status 1."""
    win = failure_window(pose=0)
    win.knot_const = cr.untouched_knots(win).astype(np.uint8)
    return win


def readers(ctx, stamps):
    """Everything a reader sees of the committed covariance: packed Sigma, landmark blocks, both interpolations."""
    packed, lm, _ = ctx.covariance_packed()
    pose, bad_pose = ctx.interpolate_covariance(stamps)
    state, bad_state = ctx.interpolate_state_covariance(stamps)
    return packed, lm, pose, state, bad_pose, bad_state


def assert_same_readers(a, b):
    """Bit for bit."""
    for x, y in zip(a[:4], b[:4]):
        assert x.shape == y.shape and np.array_equal(x.view(np.int64), y.view(np.int64))
    assert a[4:] == b[4:]


def test_failures_keep_previous_results(built, record_property):
    good = failure_window()
    stamps = good.knots[6:20, 7] + 0.013
    ctx = runtime.Context(0)
    try:
        ctx.load_window(good)
        ctx.build_covariance()
        info0 = ctx.compute_covariance()
        assert info0["status"] == 0
        keep = readers(ctx, stamps)
        record_property("accepted_min_pivot", info0["min_pivot_ratio"])

        def same_as_before():
            assert_same_readers(readers(ctx, stamps), keep)

        ctx.load_window(gauge_free_window())
        ctx.build_covariance()
        info = ctx.compute_covariance()
        record_property("gauge_free_pivot", info["min_pivot_ratio"])
        print(f"gauge free: status {info['status']} bad dof {info['bad_dof']} pivot {info['min_pivot_ratio']:.3e}; "
              f"accepted min pivot {info0['min_pivot_ratio']:.3e}")
        assert info["status"] == 1 and info["bad_dof"] >= 0 and info["rc"] == runtime.COV_NOT_POSITIVE_DEFINITE
        assert np.isfinite(info["min_pivot_ratio"]) and abs(info["min_pivot_ratio"]) < 0.1 * cr.MIN_PIVOT
        same_as_before()
        # variable biases without IMU factors
        noimu = e2e_window(4, num_knots=30, num_landmarks=200, num_imu=0, bearing=100, pose=10, seed=31)
        ctx.load_window(noimu)
        ctx.build_covariance()
        info = ctx.compute_covariance()
        K, Kbg, Kba = 30, noimu.gyro_bias.shape[0], noimu.accel_bias.shape[0]
        record_property("no_imu_bad_dof", info["bad_dof"])
        assert info["status"] == 1 and 6 * K <= info["bad_dof"] < 6 * K + 3 * (Kbg + Kba), info
        same_as_before()
        # one landmark seen by a single pixel factor
        single = e2e_window(4, num_knots=30, num_landmarks=200, num_imu=800, bearing=0, pose=10, seed=31)
        o = np.nonzero(single.v_lm == 7)[0]
        keepv = np.ones(single.v_stamp.size, bool)
        keepv[o[1:]] = False
        for key in ("v_stamp", "v_cam", "v_lm", "v_pixel"):
            setattr(single, key, np.ascontiguousarray(getattr(single, key)[keepv]))
        ctx.load_window(single)
        ctx.build_covariance()
        info = ctx.compute_covariance()
        assert info["status"] == 2 and info["degenerate_landmarks"] == 1 and info["rc"] == runtime.COV_DEGENERATE_LANDMARKS, info
        assert all(np.isfinite(v) for v in info.values() if isinstance(v, float))
        same_as_before()
        # an unobserved landmark: no failure, zero block, counted
        unobs = e2e_window(4, num_knots=30, num_landmarks=200, num_imu=800, bearing=0, pose=10, seed=31)
        keepv = unobs.v_lm != 5
        for key in ("v_stamp", "v_cam", "v_lm", "v_pixel"):
            setattr(unobs, key, np.ascontiguousarray(getattr(unobs, key)[keepv]))
        ctx.load_window(unobs)
        ctx.build_covariance()
        info = ctx.compute_covariance()
        assert info["status"] == 0 and info["unobserved_landmarks"] == 1, info
        _, lm, _ = ctx.covariance_packed()
        assert np.all(lm[5] == 0) and np.isfinite(lm).all() and (np.abs(lm[[4, 6]]) > 0).all()
    finally:
        ctx.close()


def test_linearisation_point_slots(built):
    """A build freezes its linearisation point beside the committed one and only a successful compute commits it:
    window A, then B (A after two iterations) computed twice, two failed build + compute rounds, and A again, which must
    equal a fresh context's A.  Deterministic assembly, so every comparison is bit for bit."""
    win_a = failure_window()
    stamps = win_a.knots[6:20, 7] + 0.013

    def computed(ctx):
        ctx.build_covariance()
        info = ctx.compute_covariance()
        assert info["status"] == 0, info
        return info

    ctx = runtime.Context(0)
    try:
        ctx.set_deterministic(True)
        ctx.load_window(win_a)
        computed(ctx)
        at_a = readers(ctx, stamps)
        ctx.iterate(2)
        info_b = computed(ctx)
        at_b = readers(ctx, stamps)
        assert not np.array_equal(at_b[0], at_a[0]) and not np.array_equal(at_b[3], at_a[3])
        assert ctx.compute_covariance() == info_b            # no build in between: the same point again
        assert_same_readers(readers(ctx, stamps), at_b)
        ctx.load_window(gauge_free_window())
        for _ in range(2):
            ctx.build_covariance()
            info = ctx.compute_covariance()
            assert info["status"] == 1, info
            assert [info[k] for k in ("K", "beta", "m", "L")] == [info_b[k] for k in ("K", "beta", "m", "L")]
            assert_same_readers(readers(ctx, stamps), at_b)
        ctx.load_window(win_a)
        info_a = computed(ctx)
        again = readers(ctx, stamps)
    finally:
        ctx.close()
    fresh = runtime.Context(0)
    try:
        fresh.set_deterministic(True)
        fresh.load_window(win_a)
        assert computed(fresh) == info_a
        assert_same_readers(again, readers(fresh, stamps))
    finally:
        fresh.close()


# ---- the LM path is untouched -----------------------------------------------------------------------------------------
def test_non_interference(built, record_property):
    win = e2e_window(4, num_knots=30, num_landmarks=300, num_imu=800, bearing=100, pose=10, seed=41)
    ctx = runtime.Context(0)
    try:
        ctx.load_window(win)
        kernels0 = [nm for nm, _ in ctx.profile_iteration(reps=1)]
        ctx.load_window(win)
        ctx.snapshot()

        def run():
            rec = ctx.iterate(3)
            st = ctx.state()
            ctx.restore()
            return np.array([[r[k] for k in ("cost", "cost_new", "model_change", "rho", "radius")] for r in rec]), st

        plain = [run() for _ in range(3)]
        ctx.build_covariance()
        with pytest.raises(runtime.HB200Error, match="hb200 error -2"):
            ctx.system()
        assert ctx.compute_covariance()["status"] == 0
        b, sb = run()
        kernels1 = [nm for nm, _ in ctx.profile_iteration(reps=1)]
    finally:
        ctx.close()
    # the assembly accumulates with floating-point atomics, so plain runs may differ in the last bits; the run with a
    # covariance in between must stay within twice the spread of three plain runs (0 when they agree bit for bit)
    a1, s1 = plain[0]
    spread = lambda f: max(f(x, y) for i, x in enumerate(plain) for y in plain[i + 1:])
    noise = spread(lambda x, y: np.abs(x[0] - y[0]).max())
    record_property("run_to_run", float(noise))
    record_property("with_covariance", float(np.abs(b - a1).max()))
    assert np.abs(b - a1).max() <= 2 * noise
    for k in ("knots", "gyro_bias", "accel_bias", "gravity", "landmarks"):
        assert np.abs(sb[k] - s1[k]).max() <= 2 * spread(lambda x, y: np.abs(x[1][k] - y[1][k]).max()), k
    assert kernels1 == kernels0
    assert not any(nm.startswith("cov_") for nm in kernels1)
