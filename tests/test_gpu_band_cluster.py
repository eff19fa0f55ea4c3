"""The resident band solver's cross-CTA protocol on the 2-CTA cluster (need an H100).

Chain 0 runs on CTA 0, chain 1 on CTA 1, each CTA with only its own chain in shared memory: chain 1's separator copy
crosses into CTA 0's receive buffer, CTA 0 loads CTA 1's corner partial and SPD flag, and the corner and separator
solutions cross back into CTA 1.  These tests put the hard cases where those crossings are: pivot failures on either
chain, in the separator and in the corner (the SPD flag CTA 0 reports, read from the debug record), and constant dofs and
zero diag(H) entries (the damping clamp) in the separator and at the ends of both chains.
"""
import ctypes as C

import numpy as np
import pytest

import sysref as sr
from test_gpu_solvers import inject, solver_ran, solver_window
from hyperslam_b200 import runtime

pytestmark = pytest.mark.gpu

K, BETA, KBG, KBA = 30, 5, 4, 4     # chain 0: block columns 0-12, separator 13-17, chain 1: 18-29; m = 26
M = 3 * (KBG + KBA) + 2


def open_ctx(monkeypatch, win, beta, radius):
    monkeypatch.setenv("HB200_BAND_TIMING", "1")   # allocates the debug record at bind
    ctx = runtime.Context(0)
    ctx.load_window(win, radius=radius)
    ctx.set_min_bandwidth(beta)
    assert ctx.bandwidth() == beta
    return ctx


def spd_flag(ctx):
    buf = (C.c_longlong * 144)()
    assert ctx.lib.hb200_debug_band_timing(ctx.h, buf) == 0
    return buf[70]


def test_plan_of_the_shape():
    Kt, Kb, bs = sr.band_plan(K, BETA)
    assert (Kt, Kb, bs) == (13, 12, 5)
    assert sr.solver_plan(K, BETA, M, 132)["path"] == "cluster"


# dof of a negative pivot: inside chain 0, chain 1 (the reversed chain on CTA 1), the separator, the corner; and a
# window too short for two chains (CTA 1 idle)
@pytest.mark.parametrize("k,dof", [
    pytest.param(K, 6 * 4 + 2, id="chain0"),
    pytest.param(K, 6 * 24 + 1, id="chain1"),
    pytest.param(K, 6 * 15 + 3, id="separator"),
    pytest.param(K, 6 * K + 7, id="corner"),
    pytest.param(None, None, id="spd"),
    pytest.param(12, 6 * 9, id="one_chain"),
])
def test_pivot_failure_clears_spd_flag(built, monkeypatch, k, dof):
    Kw = k or K
    win = solver_window(Kw, KBG, KBA, seed=5)
    ctx = open_ctx(monkeypatch, win, BETA, radius=1e16)
    try:
        ctx.evaluate()
        ctx.build_system()
        S, b, g, dH = sr.make_system(Kw, BETA, M, seed=17)
        if dof is not None:
            S[dof, dof] = -abs(S[dof, dof]) - 1.0
        inject(ctx, sr.pack_system(S, b, g, dH, Kw, BETA, M))
        ctx.solve()
        ctx.synchronize()
        assert spd_flag(ctx) == (1 if dof is None else 0)
        assert solver_ran(ctx) == "band_solve_kernel"
    finally:
        ctx.close()


def test_masks_and_zero_diagonals_at_the_crossings(built, monkeypatch, record_property):
    """Constant knots and zero diag(H) entries at the last column of chain 0, both ends and the middle of the separator,
    and the first and last columns of chain 1; the step is checked against the damped, masked system and repeated
    solves are bit-identical."""
    knots = (0, 12, 13, 15, 17, 18, 29)
    win = solver_window(K, KBG, KBA, knot_const=knots, seed=8)
    radius = 1e4
    ctx = open_ctx(monkeypatch, win, BETA, radius)
    try:
        ctx.evaluate()
        ctx.build_system()
        S, b, g, dH = sr.make_system(K, BETA, M, seed=23, zero_diagH=0)
        dH[[6 * c + j for c, j in ((11, 5), (12, 0), (13, 4), (14, 1), (16, 2), (17, 5), (18, 3), (19, 0))]] = 0.0
        inject(ctx, sr.pack_system(S, b, g, dH, K, BETA, M))
        fixed = sr.fixed_mask(K, KBG, KBA, win.knot_const, win.bias_const, win.gravity_const)
        A, rhs = sr.damped_masked(S, b, g, dH, fixed, radius)
        ctx.solve()
        dp, _ = ctx.delta()
        ctx.solve()
        dp2, _ = ctx.delta()
        assert spd_flag(ctx) == 1
        assert np.all(dp[fixed] == 0.0)
        n = A.shape[0]
        bwd = sr.backward_error(A, rhs, dp)
        assert bwd < n * sr.EPS, (bwd, n * sr.EPS)
        ref = sr.Reference(A, rhs, K, BETA)
        kappa = ref.kappa()
        fwd = sr.forward_error(dp, ref, sr.families(K, KBG, KBA))
        bound = sr.forward_bound(n, kappa)
        assert all(v < bound for v in fwd.values()), (fwd, bound, kappa)
        assert np.array_equal(dp.view(np.int64), dp2.view(np.int64))
        record_property("bwd", bwd)
        assert solver_ran(ctx) == "band_solve_kernel"
    finally:
        ctx.close()
