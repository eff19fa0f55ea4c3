"""weightref (CPU): the inertial bias columns of a weighted window and the weighted assembly of asmref.

With the oracle's unweighted outputs of a window, W applied in numpy gives what the device returns with W set (up to
rounding; with the dyadic matrices here every product is exact).  The weighted inertial family of weightref must then
be exactly W J_full, J_full the unweighted dense rows [Jp | wg[m] [I3 ; 0] | wa[m] [0 ; I3] | Jg], and its J^T (rho') J
the dense product of that explicitly formed matrix.  asmref itself is unchanged: without a matrix weightref.assemble is
asmref.assemble bit for bit.
"""
import numpy as np
import pytest

import asmref as ar
import oracle_lib as ol
import weightref as wr
from hyperslam_b200 import runtime, synthetic


@pytest.fixture(scope="module")
def case():
    win = synthetic.make_window(order=4, num_knots=12, num_landmarks=30, num_imu=80, seed=synthetic.SEED_BASE + 4242)
    o = ol.OracleWindow(win)
    out = o.evaluate()
    maps = o.index_maps()
    return win, out, maps


def unweighted_rows(out, k, kb):
    F = out["i_r"].shape[0]
    J = np.zeros((F, 6, 6 * k + 6 * kb + 2))
    J[:, :, :6 * k] = out["i_Jp"]
    for m in range(kb):
        for c in range(3):
            J[:, c, 6 * k + 3 * m + c] = out["i_wg"][:, m]
            J[:, 3 + c, 6 * k + 3 * kb + 3 * m + c] = out["i_wa"][:, m]
    J[:, :, 6 * k + 6 * kb:] = out["i_Jg"]
    return J


def test_dyadic_matrices_are_general():
    for kind, W in wr.all_weights(seed=1).items():
        d = runtime.Context.WEIGHT_SIDES[kind]
        assert W.shape == (d, d) and np.all(np.isfinite(W))
        if d > 1:
            assert not np.allclose(W, W.T) and not np.allclose(W, np.tril(W)) and not np.allclose(W, np.triu(W))


def test_weighted_inertial_rows_are_W_times_full_rows(case):
    win, out, maps = case
    W = wr.dyadic_matrix(6, 3)
    k, kb = win.order, win.bias_order
    weighted = wr.weigh_outputs(out, {runtime.INERTIAL: W})
    got = wr.inertial_rows(weighted, W, k, kb)
    want = np.einsum("ij,fjc->fic", W, unweighted_rows(out, k, kb))
    assert np.array_equal(got, want)   # dyadic W: every product and short sum is exact
    # the gyro-accel bias coupling the unweighted rows lack
    JtJ = np.einsum("fic,fid->cd", got, got)
    o = 6 * k
    assert np.count_nonzero(JtJ[o + 3 * kb:o + 6 * kb, o:o + 3 * kb]) > 0
    assert np.count_nonzero(np.einsum("fic,fid->cd", unweighted_rows(out, k, kb), unweighted_rows(out, k, kb))[o + 3 * kb:o + 6 * kb, o:o + 3 * kb]) == 0


def test_weighted_family_in_asmref(case):
    win, out, maps = case
    W = wr.dyadic_matrix(6, 4)
    k, kb = win.order, win.bias_order
    weighted = wr.weigh_outputs(out, {runtime.INERTIAL: W})
    p = ar.problem(weighted, win, maps)
    with wr._weighted_families(W):
        fams = ar._families(p, np.float64)
    J, r, w, _, cols = fams["inertial"]
    assert np.array_equal(J, wr.inertial_rows(weighted, W, k, kb))
    # J^T (rho') J of the family restated densely over the reduced system's columns
    n = 6 * p["K"] + 3 * (p["Kbg"] + p["Kba"]) + 2
    dense = np.zeros((n, n))
    for f in range(J.shape[0]):
        Jf = np.zeros((6, n))
        Jf[:, cols[f]] = J[f]
        dense += w[f] * Jf.T @ Jf
    ref = wr.assemble(p, 1e4, W_inertial=W, dtype=np.float64)
    ref0 = ar.assemble(ar.problem({**weighted, "i_Jp": 0 * weighted["i_Jp"], "i_Jg": 0 * weighted["i_Jg"], "i_wg": 0 * out["i_wg"],
                                   "i_wa": 0 * out["i_wa"]}, win, maps), 1e4, dtype=np.float64)
    o = 6 * p["K"]
    # the bias and gravity rows have no landmark terms: there the difference is the inertial family alone
    np.testing.assert_allclose((ref["S"] - ref0["S"])[o:, o:], dense[o:, o:], rtol=1e-12, atol=1e-12 * np.abs(dense).max())


def test_without_matrix_assemble_is_asmref(case):
    win, out, maps = case
    p = ar.problem(out, win, maps)
    a = ar.assemble(p, 1e4, dtype=np.float64)
    b = wr.assemble(p, 1e4, W_inertial=None, dtype=np.float64)
    assert all(np.array_equal(a[key], b[key]) for key in ("S", "b", "g", "diagH"))
