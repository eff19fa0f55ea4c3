"""The reduced-system solvers, tested directly across their plan boundaries (need an H100).

Each case binds a small window without landmarks (so the landmark back-substitution does not run and only the
solve is under test) with K knots and the chosen numbers of gyro and accel bias knots (m = 3 Kbg + 3 Kba + 2;
unequal counts give m = 5 mod 6), sets the band half-width with set_min_bandwidth, builds the system, then
overwrites the packed band-only buffer with a synthetic SPD band + arrow system graded like the real one
(tests/sysref.py) and solves it.  Every case asserts:

* which solver kernel ran (from profile_iteration) and the plan ensure_system made for that shape;
* hb200_get_system == the damped, masked restatement of the injected buffer, within one rounding per entry;
* the equilibrated normwise backward error of dp is below n eps, and constant dofs get exactly 0;
* the forward error of D^-1 dp, per dof family, is below 8 n eps kappa(A_hat) against a long-double-refined reference;
* the band and BCR solvers return bit-identical dp when the same buffer is solved twice.
"""
import numpy as np
import pytest

import sysref as sr
from hyperslam_b200 import runtime, synthetic

pytestmark = pytest.mark.gpu

SOLVER_KERNELS = {"band_solve_kernel", "band_solve_kernel<false>", "bcr_solve_kernel", "cholesky_kernel"}
BWD_C = 1.0   # backward error bound: BWD_C * n * eps
_SMS = []


def num_sms():
    if not _SMS:
        import torch
        _SMS.append(torch.cuda.get_device_properties(0).multi_processor_count)
    return _SMS[0]


def solver_window(K, Kbg, Kba, knot_const=(), bias_const=0, gravity_const=0, seed=0):
    """Order-4 window with K knots, a few pose factors and no landmarks or IMU factors; bias splines of Kbg / Kba
    knots (they carry no factor, only their dofs)."""
    base = synthetic.make_window(order=4, num_knots=K, num_landmarks=0, num_imu=0, seed=synthetic.SEED_BASE + 900 + seed, noise=False)
    win = synthetic.add_bearing_and_pose_factors(base, num_pose=8, seed=synthetic.SEED_BASE + 950 + seed)

    def bias(Kb):
        a = np.zeros((Kb, 4))
        a[:, 3] = win.knots[0, 7] + np.arange(Kb) * 1.0
        return a
    win.gyro_bias, win.accel_bias = bias(Kbg), bias(Kba)
    kc = np.zeros(K, dtype=np.uint8)
    kc[list(knot_const)] = 1
    win.knot_const, win.bias_const, win.gravity_const = kc, int(bias_const), int(gravity_const)
    return win


def inject(ctx, buf):
    """Overwrite the context's packed system with buf (device memory shared through __cuda_array_interface__)."""
    import torch
    ptr, count = ctx.system_device_ptr()
    assert count == buf.size

    class _Arr:
        __cuda_array_interface__ = dict(shape=(count,), typestr="<f8", data=(ptr, False), version=2)
    ctx.synchronize()
    torch.as_tensor(_Arr(), device="cuda").copy_(torch.from_numpy(buf))
    torch.cuda.synchronize()


def solve_injected(ctx, win, beta, radius, seed, report=None, determinism=True):
    """Build, inject a synthetic system of the context's shape, solve (twice) and check it.  Returns the measured errors."""
    K, Kbg, Kba = win.knots.shape[0], win.gyro_bias.shape[0], win.accel_bias.shape[0]
    m = 3 * (Kbg + Kba) + 2
    n = 6 * K + m
    ctx.evaluate()
    ctx.build_system()
    S, b, g, dH = sr.make_system(K, beta, m, seed=seed)
    inject(ctx, sr.pack_system(S, b, g, dH, K, beta, m))
    fixed = sr.fixed_mask(K, Kbg, Kba, win.knot_const, win.bias_const, win.gravity_const)
    A, rhs = sr.damped_masked(S, b, g, dH, fixed, radius)
    ctx.solve()
    dp, _ = ctx.delta()
    ctx.solve()
    dp2, _ = ctx.delta()
    # densify: what the solvers factor, one rounding per entry (the damping add)
    Ag, rg = ctx.system()
    assert np.all(np.abs(Ag - A) <= sr.EPS * np.abs(A)), np.abs(Ag - A).max()
    assert np.all(np.abs(rg - rhs) <= sr.EPS * np.abs(rhs))
    # the step
    assert np.all(dp[fixed] == 0.0)
    bwd = sr.backward_error(A, rhs, dp)
    assert bwd < BWD_C * n * sr.EPS, (bwd, n * sr.EPS)
    ref = sr.Reference(A, rhs, K, beta)
    kappa = ref.kappa()
    fwd = sr.forward_error(dp, ref, sr.families(K, Kbg, Kba))
    bound = sr.forward_bound(n, kappa)
    assert all(v < bound for v in fwd.values()), (fwd, bound, kappa)
    if determinism:
        assert np.array_equal(dp.view(np.int64), dp2.view(np.int64))
    out = dict(n=n, bwd=bwd, bwd_bound=BWD_C * n * sr.EPS, fwd=fwd["all"], fwd_bound=bound, kappa=kappa)
    if report is not None:
        for k, v in out.items():
            report(k, v)
    return out


def solver_ran(ctx):
    ran = {name for name, _ in ctx.profile_iteration(reps=1)} & SOLVER_KERNELS
    assert len(ran) == 1, ran
    return ran.pop()


def run_case(K, beta_req, Kbg, Kba, path, radius=1e4, force_dense=False, seed=0, report=None, **mask):
    win = solver_window(K, Kbg, Kba, seed=seed, **mask)
    m = 3 * (Kbg + Kba) + 2
    ctx = runtime.Context(0, force_dense=force_dense)
    try:
        ctx.load_window(win, radius=radius)
        ctx.set_min_bandwidth(beta_req)
        beta = ctx.bandwidth()
        assert beta == sr.effective_beta(4, K, beta_req)
        plan = sr.solver_plan(K, beta, m, num_sms(), force_dense)
        assert plan["path"] == path, plan
        if path in ("cluster", "chunked"):
            Kt, Kb, bs = plan["Kt"], plan["Kb"], plan["bs"]
            if K >= 2 * beta + 4:   # two-sided: chains of Kt and Kb columns meet at a separator of beta columns
                assert bs == beta and Kt + Kb + bs == K and 0 <= Kt - Kb <= 1
            else:                   # one-sided: chain 1 idle
                assert (Kt, Kb, bs) == (K, 0, 0)
        errs = solve_injected(ctx, win, beta, radius, seed=1000 * K + 10 * beta + m, report=report, determinism=(path != "dense"))
        assert solver_ran(ctx) == plan["kernel"]
        return plan, errs
    finally:
        ctx.close()


# ---- resident 2-CTA cluster band solver, and the first shape past its shared-memory budget ----------------
BIAS_KNOTS = [(4, 4), (5, 4), (8, 8), (9, 8)]   # m = 26, 29, 50, 53


def _cluster_cases():
    out = []
    for beta in (3, 4, 5, 6, 8, 12):
        for Kbg, Kba in BIAS_KNOTS:
            m = 3 * (Kbg + Kba) + 2
            kmax = sr.max_resident_K(beta, m)
            for K in sorted({beta + 1, 2 * beta + 3, 2 * beta + 4, 2 * beta + 5, kmax, kmax + 1}):
                path = "cluster" if K <= kmax else ("bcr" if 6 * beta <= sr.BCR_MAX_NB else "chunked")
                out.append(pytest.param(K, beta, Kbg, Kba, path, id=f"b{beta}-m{m}-K{K}-{path}"))
    return out


@pytest.mark.parametrize("K,beta,Kbg,Kba,path", _cluster_cases())
def test_band_cluster_solver(built, record_property, K, beta, Kbg, Kba, path):
    run_case(K, beta, Kbg, Kba, path, report=record_property)


def test_beta_clamped_to_window(built, record_property):
    """A requested half-width past the window clamps to K - 1."""
    run_case(9, 12, 5, 4, "cluster", report=record_property)


# ---- block cyclic reduction -----------------------------------------------------------------------------
# fewest super-blocks it can see is 4 (narrower windows are resident); 6 beta = 48 with the widest arrow it
# takes (m = 53; m = 54 is not 2 mod 3); a window with nsb > 2 x SM count
@pytest.mark.parametrize("K,beta,Kbg,Kba,nsb", [
    pytest.param(29, 8, 9, 8, 4, id="nsb4-b8-m53-K29"),
    pytest.param(33, 8, 9, 8, 5, id="nsb5-b8-m53-K33"),
    pytest.param(64, 8, 8, 8, 8, id="nsb8-b8-m50-K64"),
    pytest.param(65, 8, 8, 8, 9, id="nsb9-b8-m50-K65"),
    pytest.param(80, 5, 5, 4, 16, id="nsb16-b5-m29-K80"),
    pytest.param(83, 5, 4, 4, 17, id="nsb17-b5-m26-K83"),
    pytest.param(800, 3, 4, 4, 267, id="nsb267-b3-m26-K800"),
])
def test_bcr_solver(built, record_property, K, beta, Kbg, Kba, nsb):
    plan, _ = run_case(K, beta, Kbg, Kba, "bcr", report=record_property)
    assert plan["nsb"] == nsb
    if nsb > 2 * num_sms():
        assert plan["ctas"] == num_sms()


def test_arrow_past_bcr_limit(built, record_property):
    """m = 56 > 54 at 6 beta = 48: the chunked band solver takes it."""
    run_case(64, 8, 9, 9, "chunked", report=record_property)


# ---- chunked band solver: last chunk of the chain phase full / a single column --------------------------
@pytest.mark.parametrize("K,beta,Kbg,Kba,last", [
    pytest.param(35, 12, 4, 4, "full", id="b12-m26-K35-full"),
    pytest.param(37, 12, 4, 4, "single", id="b12-m26-K37-single"),
    pytest.param(34, 5, 10, 9, "full", id="b5-m59-K34-full"),
    pytest.param(36, 5, 10, 9, "single", id="b5-m59-K36-single"),
])
def test_chunked_band_solver(built, record_property, K, beta, Kbg, Kba, last):
    plan, _ = run_case(K, beta, Kbg, Kba, "chunked", report=record_property)
    assert plan["last_chunk"] == (plan["chunk"] if last == "full" else 1)


# ---- dense cooperative Cholesky -------------------------------------------------------------------------
@pytest.mark.parametrize("K,beta,Kbg,Kba,force_dense", [
    pytest.param(80, 40, 9, 8, False, id="auto-n533"),        # n > 512 and 12 (beta + 1) > 6 K
    pytest.param(4, 3, 4, 4, True, id="forced-n50"),
    pytest.param(10, 3, 5, 4, True, id="forced-n89"),
    pytest.param(20, 5, 9, 8, True, id="forced-n173"),
])
def test_dense_solver(built, record_property, K, beta, Kbg, Kba, force_dense):
    run_case(K, beta, Kbg, Kba, "dense", force_dense=force_dense, report=record_property)


# ---- constant-dof masks and damping on every path -----------------------------------------------------------
PATH_SHAPES = {"cluster": (30, 5, 5, 4), "bcr": (80, 5, 5, 4), "chunked": (37, 12, 4, 4), "dense": (80, 40, 9, 8)}
MASKS = {
    "knots-start-middle-end": dict(knot_const=None),
    "bias_const": dict(bias_const=1),
    "gravity_const": dict(gravity_const=1),
    "all-radius1e16": dict(knot_const=None, bias_const=1, gravity_const=1, radius=1e16),
    "none-radius1e16": dict(radius=1e16),
}


@pytest.mark.parametrize("mask", list(MASKS))
@pytest.mark.parametrize("path", list(PATH_SHAPES))
def test_masks_and_damping(built, record_property, path, mask):
    K, beta, Kbg, Kba = PATH_SHAPES[path]
    kw = dict(MASKS[mask])
    if "knot_const" in kw:
        kw["knot_const"] = (0, 1, K // 2, K - 1)
    run_case(K, beta, Kbg, Kba, path, seed=7, report=record_property, **kw)


# ---- re-planning on one context ---------------------------------------------------------------------------
def test_replanning_on_one_context(built, record_property):
    """set_min_bandwidth moves one context between the cluster solver and BCR at different CTA counts and back;
    every solve after a change is checked (covers the grid-barrier counter reset when bcr_ctas changes)."""
    K, Kbg, Kba = 60, 5, 4
    m = 3 * (Kbg + Kba) + 2
    win = solver_window(K, Kbg, Kba, seed=3)
    ctx = runtime.Context(0)
    try:
        ctx.load_window(win)
        seen = []
        for i, beta in enumerate((3, 8, 5, 3, 8)):
            ctx.set_min_bandwidth(beta)
            assert ctx.bandwidth() == beta
            plan = sr.solver_plan(K, beta, m, num_sms())
            solve_injected(ctx, win, beta, 1e4, seed=77 + i)
            seen.append((plan["path"], plan.get("ctas")))
        assert seen == [("cluster", None), ("bcr", 4), ("bcr", 6), ("cluster", None), ("bcr", 4)]
        assert solver_ran(ctx) == "bcr_solve_kernel"
    finally:
        ctx.close()
