"""CPU checks of tests/sysref.py: the packed-layout restatement, the damped / masked system, the reference solve,
and that the equilibrated metrics reject step and system errors the global-maximum comparisons let through."""
import numpy as np
import pytest

import oracle_lib as ol
import sysref as sr
from hyperslam_b200 import synthetic


@pytest.mark.parametrize("K,beta,m", [(4, 3, 26), (13, 3, 29), (20, 5, 50), (27, 12, 53)])
def test_pack_unpack_round_trip(K, beta, m):
    S, b, g, dH = sr.make_system(K, beta, m, seed=K)
    L = sr.layout(K, beta, m)
    assert L["n"] == 6 * K + m and L["total"] == L["os"] + 8
    assert all(L[k] % 2 == 0 for k in ("ob", "oD", "og", "os"))
    buf = sr.pack_system(S, b, g, dH, K, beta, m, scal=np.arange(8.0))
    S2, b2, g2, dH2, scal = sr.unpack_system(buf, K, beta, m)
    assert np.array_equal(S2, S) and np.array_equal(b2, b) and np.array_equal(g2, g) and np.array_equal(dH2, dH)
    assert np.array_equal(scal, np.arange(8.0))
    # sys_index: S[row][col] (row >= col) of the band, the arrow and the corner
    h = 6 + 6 * beta
    for row, col in ((0, 0), (5, 0), (6 * beta + 5, 0), (6 * K - 1, 6 * K - 6), (6 * K, 3), (6 * K + m - 1, 6 * K - 1), (6 * K + m - 1, 6 * K)):
        c = col // 6
        if row < 6 * K:
            idx = (c * h + (row - 6 * c)) * 6 + (col - 6 * c)
        elif col < 6 * K:
            idx = L["oA"] + (row - 6 * K) * 6 * K + col
        else:
            idx = L["oC"] + (row - 6 * K) * m + (col - 6 * K)
        assert buf[idx] == S[row, col]
    if K > beta + 1:
        with pytest.raises(AssertionError):   # entries outside the block band have no slot
            S3 = S.copy(); S3[6 * (beta + 1), 0] = S3[0, 6 * (beta + 1)] = 1.0
            sr.pack_system(S3, b, g, dH, K, beta, m)


def test_damped_masked_matches_direct_statement():
    K, beta, m = 9, 3, 29
    S, b, g, dH = sr.make_system(K, beta, m, seed=3)
    dH[7], dH[8], dH[9] = 0.0, 1e-9, 1e40
    Kbg, Kba = 5, 4
    kc = np.zeros(K, dtype=np.uint8); kc[[0, 4, K - 1]] = 1
    for radius in (1e4, 1e16):
        for bias_const, gravity_const in ((0, 0), (1, 0), (0, 1)):
            fixed = sr.fixed_mask(K, Kbg, Kba, kc, bias_const, gravity_const)
            A, rhs = sr.damped_masked(S, b, g, dH, fixed, radius)
            n = S.shape[0]
            want = S.copy()
            for i in range(n):
                want[i, i] = S[i, i] + (1.0 / radius) * min(max(dH[i], 1e-6), 1e32)
            for i in range(n):
                if fixed[i]:
                    want[i, :] = 0.0; want[:, i] = 0.0
            for i in range(n):
                if fixed[i]:
                    want[i, i] = 1.0
            assert np.array_equal(A, want)
            assert np.array_equal(rhs, np.array([0.0 if fixed[i] else b[i] - g[i] for i in range(n)]))
            assert fixed.sum() == 18 + (3 * (Kbg + Kba) if bias_const else 0) + (2 if gravity_const else 0)


@pytest.mark.parametrize("K,beta,m,radius", [(4, 3, 26, 1e4), (9, 3, 29, 1e16), (12, 4, 50, 1e4)])
def test_reference_agrees_with_mpmath(K, beta, m, radius):
    S, b, g, dH = sr.make_system(K, beta, m, seed=11 * K)
    fixed = sr.fixed_mask(K, (m - 2) // 6, (m - 2) // 3 - (m - 2) // 6, np.r_[1, np.zeros(K - 1)])
    A, rhs = sr.damped_masked(S, b, g, dH, fixed, radius)
    ref = sr.Reference(A, rhs, K, beta)
    x = sr.mp_solve(A, rhs, dps=40)
    fam = sr.families(K, (m - 2) // 6, (m - 2) // 3 - (m - 2) // 6)
    assert sr.forward_error(x, ref, fam)["all"] < 4 * sr.EPS
    assert sr.backward_error(A, rhs, ref.x) < sr.EPS
    assert np.all(ref.x[fixed] == 0.0)
    # the raw system spans the real system's scale range; the equilibrated one is moderately conditioned
    d = np.diag(A)[~fixed]
    assert d.min() / d.max() < 1e-8
    assert 1e2 < ref.kappa() < 1e8


# ---- the equilibrated metrics against the assertions they supersede ----------------------------------------
def _old_assertions_pass(S, b, dp, S0, b0, dp0):
    """What test_system_and_step_parity asserted before: global-maximum relative errors and residual."""
    rel = lambda a, c: np.abs(a - c).max() / np.abs(c).max()
    return bool(rel(S, S0) < 1e-9 and rel(b, b0) < 1e-9 and np.abs(S0 @ dp - b0).max() / np.abs(b0).max() < 1e-7 and rel(dp, dp0) < 1e-5)


@pytest.fixture(scope="module")
def k4_system():
    win = synthetic.make_window(seed=synthetic.SEED_BASE + 200, constant_knots=2, order=4, num_knots=20, num_landmarks=120, num_imu=400)
    o = ol.OracleWindow(win).iterate(apply=False)
    K, Kbg, Kba = 20, win.gyro_bias.shape[0], win.accel_bias.shape[0]
    ref = sr.Reference(o["S"], o["b"], K)
    return dict(S=o["S"], b=o["b"], dp=o["delta_p"], K=K, fam=sr.families(K, Kbg, Kba), ref=ref, kappa=ref.kappa())


def _mutate(v, sl, f):
    v = v.copy(); v[sl] *= f
    return v


MUTATIONS = {   # name -> (what is changed, slice in the k4 system, factor)
    "gyro_bias_step_0.05pct": ("dp", "gyro_bias", 1.0005),
    "pose_step_knot7_1e-7": ("dp", slice(42, 48), 1.0 + 1e-7),
    "pose_step_knot17_1e-6": ("dp", slice(102, 108), 1.0 + 1e-6),
    "gyro_bias_block_S_10pct": ("S", "gyro_bias", 1.1),
    "gyro_bias_block_b_10pct": ("b", "gyro_bias", 1.1),
}


@pytest.mark.parametrize("name", list(MUTATIONS))
def test_metrics_reject_mutations_the_old_assertions_pass(k4_system, name):
    s = k4_system
    S0, b0, dp0, fam = s["S"], s["b"], s["dp"], s["fam"]
    n = S0.shape[0]
    # the oracle's own step passes the new checks
    assert sr.backward_error(S0, b0, dp0) < n * sr.EPS
    assert sr.forward_error(dp0, s["ref"], fam)["all"] < sr.forward_bound(n, s["kappa"])
    what, sl, f = MUTATIONS[name]
    sl = fam[sl] if isinstance(sl, str) else sl
    if what == "S":
        blk = slice(sl.start, sl.start + 3)
        S = S0.copy(); S[blk, blk] *= f
        assert _old_assertions_pass(S, b0, dp0, S0, b0, dp0)
        assert sr.entry_error(S, S0) > 1e3 * 1e-12
        assert sr.entry_error(S, S0, fam)[("gyro_bias", "gyro_bias")] > 0.05
    elif what == "b":
        blk = slice(sl.start, sl.start + 3)
        b = _mutate(b0, blk, f)
        assert _old_assertions_pass(S0, b, dp0, S0, b0, dp0)
        assert sr.rhs_error(b, b0, S0) > 1e3 * 1e-12
        assert sr.rhs_error(b, b0, S0, fam)["gyro_bias"] > 1e-6
    else:
        dp = _mutate(dp0, sl, f)
        assert _old_assertions_pass(S0, b0, dp, S0, b0, dp0)
        assert sr.backward_error(S0, b0, dp) > 1e4 * n * sr.EPS
        if name.startswith("gyro"):
            assert sr.forward_error(dp, s["ref"], fam)["gyro_bias"] > 10 * sr.forward_bound(n, s["kappa"])


def test_solver_plan_matches_documented_boundaries():
    """The shapes DESIGN §4 quotes for the solver selection."""
    assert {b: sr.max_resident_K(b, 26) for b in (3, 5, 8)} == {3: 71, 5: 57, 8: 42}
    assert sr.solver_plan(27, 12, 26, 132)["path"] == "cluster" and sr.solver_plan(27, 12, 26, 132)["Kb"] == 0
    assert sr.solver_plan(28, 12, 26, 132)["path"] == "chunked"
    assert sr.solver_plan(72, 3, 26, 132)["path"] == "bcr"
    p = sr.solver_plan(800, 3, 26, 132)
    assert p["path"] == "bcr" and p["nsb"] > 2 * 132 and p["ctas"] == 132
    assert sr.solver_plan(80, 40, 53, 132)["path"] == "dense"
    # block cyclic reduction never sees fewer than 4 super-blocks: narrower windows are resident
    assert min(sr.solver_plan(K, b, m, 132).get("nsb", 99) for b in range(3, 9) for m in (26, 53) for K in range(b + 1, 120)) == 4
