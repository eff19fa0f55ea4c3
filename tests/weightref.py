"""Family weight matrices in the test restatements (test infrastructure, CPU only).

The device applies a family's matrix W to the residual and every Jacobian block it stores (hb200_set_weights), so the
copied-out r and J of the pixel, bearing and pose families, and of the inertial pose and gravity blocks, are already
weighted: asmref assembles them unchanged.  The inertial bias blocks are not stored; the copy-out keeps the basis weights
wg / wa, and the bias Jacobian of gyro knot m is wg[m] W[:, 0:3] (accel knot m: wa[m] W[:, 3:6]) instead of the
unweighted wg[m] [I3 ; 0] / wa[m] [0 ; I3].  `assemble` is asmref.assemble with those dense bias columns.
"""
from __future__ import annotations

import contextlib
import threading

import numpy as np

import asmref as ar
from hyperslam_b200 import runtime

SIDES = runtime.Context.WEIGHT_SIDES


def dyadic_matrix(d, seed):
    """A non-symmetric, non-triangular d x d matrix of small dyadic entries (k / 8, k in [-12, 12], diagonal >= 5/8 in
    magnitude): products with it and their short sums are exact far more often than not, so W x restated in numpy and
    the device's W x differ by rounding of x alone."""
    rng = np.random.default_rng(seed)
    W = rng.integers(-12, 13, size=(d, d)).astype(np.float64) / 8.0
    for i in range(d):
        W[i, i] = (5 + rng.integers(0, 8)) / 8.0 * (1 if rng.random() < 0.5 else -1)
    if d > 1:   # neither triangular nor symmetric
        W[0, d - 1], W[d - 1, 0] = 0.375, -1.25
    return W


def all_weights(seed=0):
    return {kind: dyadic_matrix(d, seed + kind) for kind, d in SIDES.items()}


def inertial_bias_columns(J, wg, wa, W, k, kb):
    """Overwrite the bias columns of the dense inertial rows J (F, 6, 6k + 6kb + 2) with wg[m] W[:, 0:3] / wa[m] W[:, 3:6]."""
    W = np.asarray(W, dtype=J.dtype)
    for m in range(kb):
        J[:, :, 6 * k + 3 * m:6 * k + 3 * m + 3] = wg[:, m, None, None].astype(J.dtype) * W[None, :, 0:3]
        J[:, :, 6 * k + 3 * kb + 3 * m:6 * k + 3 * kb + 3 * m + 3] = wa[:, m, None, None].astype(J.dtype) * W[None, :, 3:6]
    return J


_LOCK = threading.RLock()   # the family builder is swapped module-wide: one weighted assembly at a time


@contextlib.contextmanager
def _weighted_families(W_inertial):
    """asmref's family builder with the inertial bias columns built from W_inertial, for the duration of the block.
    asmref itself stays the unweighted restatement its own tests check."""
    _LOCK.acquire()
    orig = ar._families

    def families(p, dt):
        fams = orig(p, dt)
        if W_inertial is not None and "inertial" in fams:
            J, r, w, terms, cols = fams["inertial"]
            o = p["out"]
            fams["inertial"] = (inertial_bias_columns(J, o["i_wg"], o["i_wa"], W_inertial, p["order"], p["bias_order"]), r, w, terms, cols)
        return fams

    ar._families = families
    try:
        yield
    finally:
        ar._families = orig
        _LOCK.release()


def assemble(prob, radius, W_inertial=None, **kw):
    """asmref.assemble of the device's own (weighted) outputs, the inertial bias columns built from W_inertial."""
    with _weighted_families(W_inertial):
        return ar.assemble(prob, radius, **kw)


def inertial_rows(out, W, k, kb):
    """Dense weighted inertial Jacobian rows [Jp | gyro bias | accel bias | gravity] (F, 6, 6k + 6kb + 2) of `out`."""
    F = out["i_r"].shape[0]
    J = np.zeros((F, 6, 6 * k + 6 * kb + 2))
    J[:, :, :6 * k] = out["i_Jp"]
    J[:, :, 6 * k + 6 * kb:] = out["i_Jg"]
    return inertial_bias_columns(J, out["i_wg"], out["i_wa"], W, k, kb)


def weigh_outputs(out, weights):
    """W applied in numpy to unweighted outputs (Context.outputs() / OracleWindow.evaluate() layout): what the device
    returns with those matrices set, up to rounding.  Bias weights stay as they are."""
    res = dict(out)
    P, I, B, M = runtime.PIXEL, runtime.INERTIAL, runtime.BEARING, runtime.MANIFOLD
    if P in weights:
        for key in ("v_r", "v_Jp", "v_Jl"):
            if key in out:
                res[key] = np.einsum("ij,fj...->fi...", weights[P], out[key])
    if I in weights:
        for key in ("i_r", "i_Jp", "i_Jg"):
            if key in out:
                res[key] = np.einsum("ij,fj...->fi...", weights[I], out[key])
    if B in weights:
        for key in ("b_r", "b_Jp", "b_Jl"):
            if key in out:
                res[key] = weights[B][0, 0] * out[key]
    if M in weights:
        for key in ("m_r", "m_Jp"):
            if key in out:
                res[key] = np.einsum("ij,fj...->fi...", weights[M], out[key])
    return res


def abs_weighted_scale(out, weights):
    """Per output row, sum_j |W_ij| max|row j of out|: the scale a weighted row's rounding error is measured in."""
    P, I, B, M = runtime.PIXEL, runtime.INERTIAL, runtime.BEARING, runtime.MANIFOLD
    fam = {"v": P, "i": I, "b": B, "m": M}
    res = {}
    for key, a in out.items():
        if key in ("i_wg", "i_wa"):
            continue
        W = weights.get(fam[key[0]])
        a = np.abs(np.asarray(a, dtype=np.float64))
        if key[0] == "b":
            row = a if a.ndim == 1 else a.max(-1)
            res[key] = (abs(W[0, 0]) if W is not None else 1.0) * row
            continue
        row = a if a.ndim == 2 else a.max(-1)          # (F, R)
        Wa = np.abs(W) if W is not None else np.eye(row.shape[1])
        res[key] = np.einsum("ij,fj->fi", Wa, row)
    return res


def cost(out, win, weights=None):
    """1/2 sum rho(|r|^2) of (already weighted) outputs: Huber for visual factors, ScaledLoss for inertial, none for pose."""
    def huber(s, d):
        return np.where(s <= d * d, s, 2 * d * np.sqrt(s) - d * d)
    c = 0.5 * huber((out["v_r"] ** 2).sum(1), win.huber_pixel).sum()
    c += 0.5 * win.imu_loss_scale * (out["i_r"] ** 2).sum()
    if "b_r" in out:
        c += 0.5 * huber(out["b_r"] ** 2, win.huber_bearing).sum()
    if "m_r" in out:
        c += 0.5 * (out["m_r"] ** 2).sum()
    return float(c)
