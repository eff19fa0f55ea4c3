"""Long-double assembly of the reduced system from the device's own per-factor outputs (test infrastructure, CPU only).

Input: the residuals and Jacobians a context copies out (`Context.outputs()`), the knot / bias bases of every factor,
the landmark of every visual factor, the loss settings and the trust-region radius.  Output: what hb200_build_system
leaves in the raw packed buffer (sysref.layout), restated in np.longdouble:

  S      = J^T W J - sum_l Y_l Y_l^T            over the band, arrow and corner (lower triangle)
  b slot = sum_l Y_l z_l                        (the solvers use b - g)
  g      = J^T W r          diagH = diag(J^T W J) (before the Schur complement)          scal[0] = cost

with, per landmark, V_l = sum w Jl^T Jl damped by mu clamp(diag V_l, 1e-6, 1e32), V_l = L L^T (Cholesky, every pivot
floored at mu d_j: V + mu D >= mu D bounds it from below in exact arithmetic), Y_l = W_l L^-T and z_l = L^-1 g_l.
Weights: Huber rho' of |r|^2 for pixel / bearing factors (from the device's own r), the inertial ScaledLoss, none for
pose factors.

Every entry also gets a componentwise bound gamma_ij M_ij with gamma_ij = C_BOUND m_ij u (u = 2^-53, m_ij = number of
summands the entry receives) and M the same sums over absolute values.  For the landmark terms M also carries the
first-order effect of perturbing W_l and V_l by their own rounding, |W| |L^-T| |Y|^T and |Y| |L^-1| |V| |L^-T| |Y|^T:
V_l of a short-baseline track is ill-conditioned along the depth, and two correct summation orders of V_l differ there
by more than rounding of the result.  Because the reference starts from the device's Jacobians, summation order and
that sensitivity are the only legitimate differences left.
"""
from __future__ import annotations

import dataclasses

import numpy as np

import sysref as sr
from hyperslam_b200 import synthetic

LD = np.longdouble
U = 2.0 ** -53
C_BOUND = 2.0            # gamma_ij = C_BOUND * m_ij * u
DAMP_LO, DAMP_HI = sr.DAMP_LO, sr.DAMP_HI


def huber(s, delta):
    """(weight rho'(s), rho(s)) of the Huber loss on s = |r|^2 with threshold delta (ceres::HuberLoss)."""
    d = LD(delta)
    inl = s <= d * d
    rt = np.sqrt(np.where(inl, 1, s))
    return np.where(inl, 1, d / rt), np.where(inl, s, 2 * d * rt - d * d)


def problem(out, win, maps):
    """Everything assemble() needs from a bound window: `out` = Context.outputs() (or OracleWindow.evaluate()),
    `win` the synthetic.Window it was loaded from, `maps` = index_maps() (pixel, inertial, gyro-bias, accel-bias bases)."""
    vb, ib, ig, ia = maps
    k = win.order
    seg = lambda t: synthetic.segment(win.knots[:, 7], k, np.asarray(t, dtype=np.float64))[0] if np.size(t) else np.zeros(0, np.int64)
    return dict(out=out, order=k, bias_order=win.bias_order, K=win.knots.shape[0], Kbg=win.gyro_bias.shape[0], Kba=win.accel_bias.shape[0],
                L=win.landmarks.shape[0], vb=np.asarray(vb), ib=np.asarray(ib), ig=np.asarray(ig), ia=np.asarray(ia),
                bb=seg(win.b_stamp), mb=seg(win.m_stamp), v_lm=np.asarray(win.v_lm), b_lm=np.asarray(win.b_lm),
                huber_pixel=win.huber_pixel, huber_bearing=win.huber_bearing, imu_scale=win.imu_loss_scale)


def _families(p, dt):
    """Per family: (J (F, R, C), r (F, R), w (F), cost terms (F), global column of every J column (F, C))."""
    o, k, kb = p["out"], p["order"], p["bias_order"]
    K, Kbg, Kba = p["K"], p["Kbg"], p["Kba"]
    o_bg, o_ba, o_g = 6 * K, 6 * K + 3 * Kbg, 6 * K + 3 * Kbg + 3 * Kba
    pose = lambda base: 6 * np.asarray(base, dtype=np.int64)[:, None] + np.arange(6 * k)[None, :]
    fams = {}
    if len(p["vb"]):
        r = o["v_r"].astype(dt)
        w, rho = huber((r * r).sum(1), p["huber_pixel"])
        fams["pixel"] = (o["v_Jp"].astype(dt), r, w.astype(dt), (rho / 2).astype(dt), pose(p["vb"]))
    if len(p["bb"]):
        r = o["b_r"].astype(dt)[:, None]
        w, rho = huber(r[:, 0] * r[:, 0], p["huber_bearing"])
        fams["bearing"] = (o["b_Jp"].astype(dt)[:, None, :], r, w.astype(dt), (rho / 2).astype(dt), pose(p["bb"]))
    if len(p["mb"]):
        r = o["m_r"].astype(dt)
        fams["manifold"] = (o["m_Jp"].astype(dt), r, np.ones(len(r), dt), (r * r).sum(1) / 2, pose(p["mb"]))
    if len(p["ib"]):
        F = len(p["ib"])
        nc = 6 * k + 6 * kb + 2
        J = np.zeros((F, 6, nc), dt)
        J[:, :, :6 * k] = o["i_Jp"]
        for m in range(kb):
            for c in range(3):
                J[:, c, 6 * k + 3 * m + c] = o["i_wg"][:, m]
                J[:, 3 + c, 6 * k + 3 * kb + 3 * m + c] = o["i_wa"][:, m]
        J[:, :, 6 * k + 6 * kb:] = o["i_Jg"]
        cols = np.concatenate([pose(p["ib"]), o_bg + 3 * np.asarray(p["ig"], np.int64)[:, None] + np.arange(3 * kb)[None, :],
                               o_ba + 3 * np.asarray(p["ia"], np.int64)[:, None] + np.arange(3 * kb)[None, :],
                               np.broadcast_to(o_g + np.arange(2), (F, 2))], axis=1)
        r = o["i_r"].astype(dt)
        w = np.full(F, p["imu_scale"], dt)
        fams["inertial"] = (J, r, w, w * (r * r).sum(1) / 2, cols)
    return fams


def _chol3(V, Dl, mu):
    """Cholesky of the damped 3 x 3 blocks V (L, 3, 3) with pivots floored at mu d_j: (L10, L20, L21, 1/L00, 1/L11, 1/L22)."""
    p0 = np.maximum(V[:, 0, 0], mu * Dl[:, 0])
    i0 = 1 / np.sqrt(p0)
    l10, l20 = V[:, 1, 0] * i0, V[:, 2, 0] * i0
    p1 = np.maximum(V[:, 1, 1] - l10 * l10, mu * Dl[:, 1])
    i1 = 1 / np.sqrt(p1)
    l21 = (V[:, 2, 1] - l20 * l10) * i1
    p2 = np.maximum(V[:, 2, 2] - l20 * l20 - l21 * l21, mu * Dl[:, 2])
    return l10, l20, l21, i0, i1, 1 / np.sqrt(p2)


def _lsolve(f, x):
    """L^-1 x for x (L, ..., 3) with the factors of _chol3 (broadcast over the middle axes)."""
    l10, l20, l21, i0, i1, i2 = (a.reshape((-1,) + (1,) * (x.ndim - 2)) for a in f)
    y0 = x[..., 0] * i0
    y1 = (x[..., 1] - l10 * y0) * i1
    y2 = (x[..., 2] - l20 * y0 - l21 * y1) * i2
    return np.stack([y0, y1, y2], -1)


def _adjugate_inverse(V):
    """The explicit adjugate inverse the landmark elimination used to take (kept to show what the bound rejects)."""
    a, b, c, d, e, f = V[:, 0, 0], V[:, 0, 1], V[:, 0, 2], V[:, 1, 1], V[:, 1, 2], V[:, 2, 2]
    c00, c01, c02 = d * f - e * e, c * e - b * f, b * e - c * d
    idt = 1 / (a * c00 + b * c01 + c * c02)
    return np.stack([np.stack([c00, c01, c02], -1), np.stack([c01, a * f - c * c, b * c - a * e], -1),
                     np.stack([c02, b * c - a * e, a * d - b * b], -1)], -2) * idt[:, None, None]


def assemble(p, radius, dtype=LD, seed=None, weights=None, skip_landmarks=(), adjugate_landmarks=()):
    """The raw packed system of problem p at the given radius.  Returns a dict of dense S (n x n, symmetric), b, g, diagH,
    cost and their bounds (*_bound = gamma * M).

    dtype / seed: a float64 assembly with the factors of every family in a random order (the bound's own check);
    weights: {family: weight array} replacing the loss weights; skip_landmarks: landmarks whose Schur term is left out;
    adjugate_landmarks: landmarks eliminated through the explicit adjugate inverse instead (mutations the bound must reject)."""
    dt = dtype
    K, Kbg, Kba, k = p["K"], p["Kbg"], p["Kba"], p["order"]
    n = 6 * K + 3 * (Kbg + Kba) + 2
    mu = dt(1) / dt(radius)
    S, MS, cS = np.zeros((n, n), dt), np.zeros((n, n)), np.zeros((n, n))
    g, Mg, cg = np.zeros(n, dt), np.zeros(n), np.zeros(n)
    cost, Mcost, ccost = dt(0), 0.0, 0.0
    rng = np.random.default_rng(seed) if seed is not None else None
    fams = _families(p, dt)
    for name, (J, r, w, c, cols) in fams.items():
        if weights and name in weights:
            w = np.asarray(weights[name], dt)
        R = J.shape[1]
        order = rng.permutation(len(w)) if rng is not None else np.arange(len(w))
        J, r, w, c, cols = J[order], r[order], w[order], c[order], cols[order]
        cost += c.sum()
        Mcost += float(np.abs(c).sum())
        ccost += len(c)
        ucols, grp = np.unique(cols, axis=0, return_inverse=True)
        grp = grp.ravel()
        for q in range(len(ucols)):
            sel = grp == q
            Jw, Jq = J[sel] * w[sel, None, None], J[sel]
            ix = np.ix_(ucols[q], ucols[q])
            S[ix] += np.einsum("frc,frd->cd", Jw, Jq)
            A = np.abs(Jq).astype(np.float64)
            MS[ix] += np.einsum("frc,frd->cd", A * np.abs(w[sel, None, None]).astype(np.float64), A)
            cS[ix] += sel.sum() * (R + 3)
            g[ucols[q]] += np.einsum("frc,fr->c", Jw, r[sel])
            Mg[ucols[q]] += np.einsum("frc,fr->c", A * np.abs(w[sel, None, None]).astype(np.float64), np.abs(r[sel]).astype(np.float64))
            cg[ucols[q]] += sel.sum() * (R + 3)
    diagH, MdH, cdH = np.diagonal(S).copy(), np.diagonal(MS).copy(), np.diagonal(cS).copy()
    b, Mb, cb = np.zeros(n, dt), np.zeros(n), np.zeros(n)
    # landmark elimination
    L = p["L"]
    obs = []
    if "pixel" in fams:
        J, r, w, _, _ = fams["pixel"]
        wv = np.asarray(weights["pixel"], dt) if weights and "pixel" in weights else w
        obs.append((J, p["out"]["v_Jl"].astype(dt), r, wv, np.asarray(p["vb"]), np.asarray(p["v_lm"])))
    if "bearing" in fams:
        J, r, w, _, _ = fams["bearing"]
        wv = np.asarray(weights["bearing"], dt) if weights and "bearing" in weights else w
        obs.append((J, p["out"]["b_Jl"].astype(dt)[:, None, :], r, wv, np.asarray(p["bb"]), np.asarray(p["b_lm"])))
    if L and obs:
        lo = np.full(L, np.iinfo(np.int64).max)
        hi = np.full(L, -1)
        nobs = np.zeros(L, np.int64)
        for _, _, _, _, base, lm in obs:
            np.minimum.at(lo, lm, base)
            np.maximum.at(hi, lm, base)
            np.add.at(nobs, lm, 1)
        seen = nobs > 0
        lo = np.where(seen, lo, 0)
        span = np.where(seen, hi - lo + k, 0)
        RW = 6 * int(span.max())
        W, V, gl = np.zeros((L, RW, 3), dt), np.zeros((L, 3, 3), dt), np.zeros((L, 3), dt)
        MW, MV = np.zeros((L, RW, 3)), np.zeros((L, 3, 3))
        for Jp, Jl, r, w, base, lm in obs:
            wJl = Jl * w[:, None, None]
            np.add.at(V, lm, np.einsum("fra,frb->fab", wJl, Jl))
            np.add.at(gl, lm, np.einsum("fra,fr->fa", wJl, r))
            aJl = np.abs(wJl).astype(np.float64)
            np.add.at(MV, lm, np.einsum("fra,frb->fab", aJl, np.abs(Jl).astype(np.float64)))
            off = base - lo[lm]
            for q in np.unique(off):
                s = off == q
                np.add.at(W[:, 6 * q:6 * q + 6 * k], lm[s], np.einsum("fra,frc->fac", Jp[s], wJl[s]))
                np.add.at(MW[:, 6 * q:6 * q + 6 * k], lm[s], np.einsum("fra,frc->fac", np.abs(Jp[s]).astype(np.float64), aJl[s]))
        Dl = np.clip(np.diagonal(V, axis1=1, axis2=2), dt(DAMP_LO), dt(DAMP_HI))
        Vd = V + mu * (Dl[:, :, None] * np.eye(3, dtype=dt))
        f = _chol3(Vd, Dl, mu)
        Y, z = _lsolve(f, W), _lsolve(f, gl[:, None, :])[:, 0]
        adj = np.zeros(L, bool)
        adj[list(adjugate_landmarks)] = True
        if adj.any():   # W V^-1 W^T through the adjugate inverse: Y z -> W Vi g, Y Y^T -> (W Vi) W^T (Y stands for W Vi here)
            Vi = _adjugate_inverse(Vd[adj])
            WV = np.einsum("lra,lab->lrb", W[adj], Vi)
        # |L^-1| and the first-order bound of the landmark terms
        Li = _lsolve(f, np.broadcast_to(np.eye(3, dtype=dt), (L, 3, 3)).copy())    # rows: L^-1 e_j -> (L^-1)^T
        Li = np.swapaxes(Li, 1, 2)                                                  # L^-1
        aLi = np.abs(Li).astype(np.float64)
        MVd = MV + np.abs(mu * Dl).astype(np.float64)[:, :, None] * np.eye(3)
        G = np.einsum("lab,lbc,ldc->lad", aLi, MVd, aLi)                            # |L^-1| |V| |L^-T|
        aY, az = np.abs(Y).astype(np.float64), np.abs(z).astype(np.float64)
        Yt = np.einsum("lrb,lab->lra", MW, aLi)                                     # |W| |L^-T|
        zt = np.einsum("lb,lab->la", np.abs(gl).astype(np.float64), aLi)
        keep = seen.copy()
        keep[list(skip_landmarks)] = False
        for c0 in np.unique(lo[keep]):
            sel = keep & (lo == c0)
            r0 = 6 * int(c0)
            wd = min(RW, 6 * K - r0)
            Ys, zs = Y[sel, :wd], z[sel]
            rows = slice(r0, r0 + wd)
            sa = sel & ~adj
            if sa.any():
                S[rows, rows] -= np.einsum("lra,lsa->rs", Y[sa, :wd], Y[sa, :wd])
                b[rows] += np.einsum("lra,la->r", Y[sa, :wd], z[sa])
            sj = sel[adj]
            if sj.any():
                WVs, Ws = WV[sj, :wd], W[sel & adj, :wd]
                S[rows, rows] -= np.einsum("lra,lsa->rs", WVs, Ws)
                b[rows] += np.einsum("lra,la->r", WVs, gl[sel & adj])
            aYs, Ytl = aY[sel, :wd], Yt[sel, :wd]
            MS[rows, rows] += (np.einsum("lra,lsa->rs", aYs, aYs) + 2 * np.einsum("lra,lsa->rs", Ytl, aYs)
                               + np.einsum("lra,lab,lsb->rs", aYs, G[sel], aYs))
            Mb[rows] += (np.einsum("lra,la->r", aYs, az[sel]) + np.einsum("lra,la->r", Ytl, az[sel]) + np.einsum("lra,la->r", aYs, zt[sel])
                         + np.einsum("lra,lab,lb->r", aYs, G[sel], az[sel]))
            m = (2 * nobs[sel] + 12).astype(np.float64)     # W, V and g_l sums, the factorisation and the 3-term products
            occ = (np.abs(W[sel, :wd]).sum(-1) > 0).astype(np.float64)
            cS[rows, rows] += np.einsum("l,lr,ls->rs", m, occ, occ)
            cb[rows] += np.einsum("l,lr->r", m, occ)
    S = np.tril(S) + np.tril(S, -1).T
    MS, cS = np.maximum(MS, MS.T), np.maximum(cS, cS.T)
    gam = lambda c: C_BOUND * (c + 1) * U
    return dict(S=S, b=b, g=g, diagH=diagH, cost=cost, S_bound=gam(cS) * MS, b_bound=gam(cb) * Mb, g_bound=gam(cg) * Mg,
                diagH_bound=gam(cdH) * MdH, cost_bound=gam(ccost) * Mcost, n=n, K=K, Kbg=Kbg, Kba=Kba)


# ---- comparison with the raw packed buffer ----------------------------------------------------------------
def packed(ref, beta):
    """(values, bounds) in the raw packed layout: lower-triangle slots only.  Every other slot (upper half of the diagonal
    blocks and of the corner, rows past the last pose dof, padding) has value 0 and bound 0."""
    K, n = ref["K"], ref["n"]
    m = n - 6 * K
    Lay = sr.layout(K, beta, m)
    val, bnd = np.zeros(Lay["total"], LD), np.zeros(Lay["total"])
    idx, row, col = sr._band_slots(Lay)
    low = row >= col
    idx, row, col = idx[low], row[low], col[low]
    val[idx], bnd[idx] = ref["S"][row, col], ref["S_bound"][row, col]
    np_ = 6 * K
    val[Lay["oA"]:Lay["oC"]] = ref["S"][np_:, :np_].ravel()
    bnd[Lay["oA"]:Lay["oC"]] = ref["S_bound"][np_:, :np_].ravel()
    tri = np.tril(np.ones((m, m), bool))
    val[Lay["oC"]:Lay["oC"] + m * m] = np.where(tri, ref["S"][np_:, np_:], 0).ravel()
    bnd[Lay["oC"]:Lay["oC"] + m * m] = np.where(tri, ref["S_bound"][np_:, np_:], 0).ravel()
    for key, o in (("b", "ob"), ("diagH", "oD"), ("g", "og")):
        val[Lay[o]:Lay[o] + n], bnd[Lay[o]:Lay[o] + n] = ref[key], ref[key + "_bound"]
    val[Lay["os"]], bnd[Lay["os"]] = ref["cost"], ref["cost_bound"]
    return val, bnd, Lay


def compare(buf, ref, beta):
    """Worst |buf - ref| / bound per part of the packed buffer (S band, arrow, corner, b, g, diagH, cost), and the number of
    slots that must be exactly zero and are not.  A part passes when its ratio is <= 1."""
    val, bnd, Lay = packed(ref, beta)
    return _ratios(np.asarray(buf, dtype=np.float64), val, bnd, bnd == 0, Lay, ref["n"])


def _ratios(buf, val, bnd, zero, Lay, n):
    assert buf.size == val.size
    err = np.abs(buf.astype(LD) - val).astype(np.float64)
    parts = dict(band=slice(0, Lay["oA"]), arrow=slice(Lay["oA"], Lay["oC"]), corner=slice(Lay["oC"], Lay["ob"]),
                 b=slice(Lay["ob"], Lay["ob"] + n), diagH=slice(Lay["oD"], Lay["oD"] + n), g=slice(Lay["og"], Lay["og"] + n),
                 cost=slice(Lay["os"], Lay["os"] + 1))
    out = {}
    for key, s in parts.items():
        e, bb, z = err[s], bnd[s], zero[s]
        out[key] = float((e[~z] / bb[~z]).max()) if (~z).any() else 0.0
    out["nonzero_outside"] = int(np.count_nonzero(buf[:Lay["os"]][zero[:Lay["os"]]] != 0.0))   # (scal[1:] is not the assembly's)
    out["finite"] = bool(np.isfinite(buf).all())
    return out


def check(buf, ref, beta):
    res = compare(buf, ref, beta)
    bad = {k: v for k, v in res.items() if k not in ("nonzero_outside", "finite") and not v <= 1.0}
    assert res["finite"] and res["nonzero_outside"] == 0 and not bad, res
    return res


# ---- sharded systems ----------------------------------------------------------------------------------------
SHARD_FIELDS = dict(pixel=("v_stamp", "v_cam", "v_lm", "v_pixel"), bearing=("b_stamp", "b_cam", "b_lm", "b_bearing"),
                    inertial=("i_stamp", "i_meas"), pose=("m_stamp", "m_sensor", "m_pose"))


def partition(win, ranks, world):
    """The factor shards of `win` for `world` ranks: ranks[family][f] = rank of factor f, for every family of SHARD_FIELDS.
    State (knots, biases, gravity, landmarks, calibration) is replicated in every shard."""
    out = []
    for r in range(world):
        kw = {}
        for fam, keys in SHARD_FIELDS.items():
            sel = np.asarray(ranks[fam]) == r
            assert sel.size == getattr(win, keys[0]).shape[0], fam
            kw.update({key: np.ascontiguousarray(getattr(win, key)[sel]) for key in keys})
        out.append(dataclasses.replace(win, **kw))
    return out


def compare_shard_sum(refs, full):
    """Long-double sum of the shard references against the reference of the whole window: worst |sum - full| / bound per
    part (S, b, g, diagH, cost) with bound = the sum of the shard bounds + the full window's bound, and the number of entries
    that differ where every bound is 0.  A partition that keeps each landmark's observations on one rank passes (<= 1)."""
    out = dict(nonzero_outside=0)
    for key in ("S", "b", "g", "diagH", "cost"):
        err = np.abs(sum(r[key] for r in refs) - full[key]).astype(np.float64)
        bnd = sum(r[key + "_bound"] for r in refs) + full[key + "_bound"]
        err, bnd = np.atleast_1d(err), np.atleast_1d(bnd)
        z = bnd == 0
        out[key] = float((err[~z] / bnd[~z]).max()) if (~z).any() else 0.0
        out["nonzero_outside"] += int(np.count_nonzero(err[z]))
    return out


def compare_summed_buffers(bufs, refs, beta):
    """Partial packed buffers (one per rank, all at half-width beta) summed in rank order in float64, as the reduction does,
    against the long-double sum of their references.  Bound per slot: the sum of the shard bounds + (N - 1) u sum_r |buf_r|
    (the float64 sum of N terms).  Slots where every shard's bound is 0 must be exactly 0.  Same keys as compare()."""
    vals, bnds = [], []
    for r in refs:
        v, b, Lay = packed(r, beta)
        vals.append(v)
        bnds.append(b)
    bufs = [np.asarray(b, dtype=np.float64) for b in bufs]
    tot = bufs[0].copy()
    for b in bufs[1:]:
        tot = tot + b
    own = sum(bnds)
    bnd = own + (len(bufs) - 1) * U * sum(np.abs(b) for b in bufs)
    return _ratios(tot, sum(vals), bnd, own == 0, Lay, refs[0]["n"])
