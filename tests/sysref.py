"""Reference tools for the reduced-system solvers (test infrastructure, CPU only).

* the packed band-only system buffer (`hb::SysLayout`, hyperslam_b200/csrc/hb200_types.cuh) and its inverse;
* what the solvers factor: the damped, masked system (densify_kernel, and the band / BCR gathers);
* a reference solve: symmetric diagonal equilibration, float64 band + arrow Cholesky, iterative refinement with
  residuals in long double;
* the equilibrated error metrics the solver and parity tests assert on;
* the solver selection of `ensure_system` (hb200_api.cu), restated so a test can say which path it reaches;
* a generator of synthetic band + arrow SPD systems graded like the real ones.

The reduced system's dof families differ by up to nine orders of magnitude on the diagonal (the bias and gravity
blocks sit at 1e-9 .. 1e-6 of max|S| on a typical window), so errors measured against the global maximum say
nothing about the small families.  Every metric here is taken after scaling by D = diag(A)^-1/2.
"""
from __future__ import annotations

import numpy as np
import scipy.linalg as sla
import scipy.sparse.linalg as spla

EPS = float(np.finfo(np.float64).eps)
DAMP_LO, DAMP_HI = 1e-6, 1e32       # clamp of diag(H) in the LM damping term (densify_kernel, band / BCR gathers)
SMEM_LIMIT = 220 * 1024             # shared-memory budget ensure_system plans against (bytes)
BCR_MAX_NB = 48                     # kBcrMaxNb (hb200_bcr.cuh): 6 beta <= 48
BCR_MAX_M = 54                      # widest arrow block cyclic reduction takes (ensure_system)
FAMILIES = ("pose", "gyro_bias", "accel_bias", "gravity")


# ---- packed layout -----------------------------------------------------------------------------------------
def layout(K, beta, m):
    """hb::sys_layout (hb200_types.cuh): offsets in doubles of the band-only packed system.
      P [K][h][6]  block column c holds rows 6c .. 6c+h-1 of columns 6c .. 6c+5, h = 6 + 6 beta (lower triangle)
      A [m][6K]    arrow rows            C [m][m]  corner
      b, diagH, g [n] each (even offsets)           scal [8]"""
    h, np_ = 6 + 6 * beta, 6 * K
    n = np_ + m
    oA = K * h * 6
    oC = oA + m * np_
    ob = (oC + m * m + 1) & ~1
    oD = (ob + n + 1) & ~1
    og = (oD + n + 1) & ~1
    os_ = (og + n + 1) & ~1
    return dict(K=K, beta=beta, m=m, h=h, np=np_, n=n, oA=oA, oC=oC, ob=ob, oD=oD, og=og, os=os_, total=os_ + 8)


def _band_slots(L):
    """(packed index, row, col) of every P slot that holds a matrix entry (row < 6K; rows past it are padding)."""
    K, h = L["K"], L["h"]
    c, r, a = np.meshgrid(np.arange(K), np.arange(h), np.arange(6), indexing="ij")
    row, col = 6 * c + r, 6 * c + a
    idx = (c * h + r) * 6 + a
    keep = row < L["np"]
    return idx[keep], row[keep], col[keep]


def pack_system(S, b, g, diagH, K, beta, m, scal=None):
    """Dense symmetric S (zero outside the block band of half-width beta and the arrow) -> packed buffer.
    Slots of the diagonal blocks above the diagonal get the symmetric value; padding rows are zero."""
    L = layout(K, beta, m)
    S = np.asarray(S, dtype=np.float64)
    np_, n = L["np"], L["n"]
    assert S.shape == (n, n)
    blk = np.arange(np_) // 6
    far = np.abs(blk[:, None] - blk[None, :]) > beta
    assert not np.any(S[:np_, :np_][far]), "S has entries outside the block band"
    buf = np.zeros(L["total"])
    idx, row, col = _band_slots(L)
    buf[idx] = S[row, col]
    buf[L["oA"]:L["oC"]] = S[np_:, :np_].ravel()
    buf[L["oC"]:L["oC"] + m * m] = S[np_:, np_:].ravel()
    buf[L["ob"]:L["ob"] + n] = b
    buf[L["oD"]:L["oD"] + n] = diagH
    buf[L["og"]:L["og"] + n] = g
    if scal is not None:
        buf[L["os"]:L["os"] + 8] = scal
    return buf


def unpack_system(buf, K, beta, m):
    """Packed buffer -> (S, b, g, diagH, scal); S is read from the lower triangle only and symmetrised."""
    L = layout(K, beta, m)
    np_, n = L["np"], L["n"]
    buf = np.asarray(buf, dtype=np.float64)
    assert buf.size == L["total"]
    S = np.zeros((n, n))
    idx, row, col = _band_slots(L)
    low = row >= col
    S[row[low], col[low]] = buf[idx[low]]
    S[np_:, :np_] = buf[L["oA"]:L["oC"]].reshape(m, np_)
    C = buf[L["oC"]:L["oC"] + m * m].reshape(m, m)
    S[np_:, np_:] = np.tril(C)
    S = np.tril(S) + np.tril(S, -1).T
    seg = lambda o: buf[o:o + n].copy()
    return S, seg(L["ob"]), seg(L["og"]), seg(L["oD"]), buf[L["os"]:L["os"] + 8].copy()


# ---- what the solvers factor ----------------------------------------------------------------------------
def fixed_mask(K, Kbg, Kba, knot_const=None, bias_const=0, gravity_const=0):
    """Constant-dof mask of update_fixed (hb200_api.cu): 6 per constant knot, every bias dof, both gravity dofs."""
    n = 6 * K + 3 * Kbg + 3 * Kba + 2
    f = np.zeros(n, dtype=bool)
    if knot_const is not None:
        f[:6 * K] = np.repeat(np.asarray(knot_const, dtype=bool), 6)
    if bias_const:
        f[6 * K:n - 2] = True
    if gravity_const:
        f[n - 2:] = True
    return f


def damped_masked(S, b, g, diagH, fixed, radius):
    """A = S + mu clamp(diagH, 1e-6, 1e32) on the diagonal (mu = 1 / radius), rows and columns of constant dofs
    replaced by the identity; rhs = b - g with constant entries 0."""
    fixed = np.asarray(fixed, dtype=bool)
    A = np.array(S, dtype=np.float64)
    i = np.arange(A.shape[0])
    A[i, i] += (1.0 / radius) * np.minimum(np.maximum(diagH, DAMP_LO), DAMP_HI)
    A[fixed, :] = 0.0
    A[:, fixed] = 0.0
    A[fixed, fixed] = 1.0
    rhs = np.where(fixed, 0.0, np.asarray(b) - np.asarray(g))
    return A, rhs


def families(K, Kbg, Kba):
    o = 6 * K
    return dict(pose=slice(0, o), gyro_bias=slice(o, o + 3 * Kbg), accel_bias=slice(o + 3 * Kbg, o + 3 * Kbg + 3 * Kba),
                gravity=slice(o + 3 * Kbg + 3 * Kba, o + 3 * Kbg + 3 * Kba + 2))


# ---- reference solve ------------------------------------------------------------------------------------
def lower_symmetric(A):
    """The symmetric matrix the solvers see: A's lower triangle mirrored."""
    A = np.asarray(A, dtype=np.float64)
    return np.tril(A) + np.tril(A, -1).T


def equilibrate(A):
    """D = diag(A)^-1/2 and A_hat = D A D."""
    d = 1.0 / np.sqrt(np.diag(A))
    return d, A * d[:, None] * d[None, :]


class BandArrowCholesky:
    """float64 Cholesky of an SPD band + arrow matrix: banded factor of the pose block (lower half-bandwidth
    6 beta + 5), then the dense Schur complement of the arrow."""

    def __init__(self, A, np_, beta):
        hb = min(6 * beta + 5, max(np_ - 1, 0))
        P = A[:np_, :np_]
        self.np, self.B = np_, A[np_:, :np_]
        ab = np.zeros((hb + 1, np_))
        for d in range(hb + 1):
            ab[d, :np_ - d] = np.diagonal(P, -d)
        self.cb = sla.cholesky_banded(ab, lower=True)
        self.Z = sla.cho_solve_banded((self.cb, True), self.B.T)
        self.cs = sla.cho_factor(A[np_:, np_:] - self.B @ self.Z, lower=True)

    def solve(self, r):
        zp = sla.cho_solve_banded((self.cb, True), r[:self.np])
        xm = sla.cho_solve(self.cs, r[self.np:] - self.B @ zp)
        return np.concatenate([zp - self.Z @ xm, xm])


def residual_ld(A, x, b, rows=512):
    """b - A x accumulated in long double."""
    xl = np.asarray(x, dtype=np.longdouble)
    r = np.empty(A.shape[0], dtype=np.longdouble)
    for lo in range(0, A.shape[0], rows):
        r[lo:lo + rows] = np.asarray(b[lo:lo + rows], dtype=np.longdouble) - A[lo:lo + rows].astype(np.longdouble) @ xl
    return r


def block_bandwidth(A, K):
    """Block half-bandwidth of the pose part of A (6 x 6 control-point blocks)."""
    r, c = np.nonzero(A[:6 * K, :6 * K])
    return int(np.abs(r // 6 - c // 6).max()) if r.size else 0


class Reference:
    """Reference solution of A x = rhs: float64 band + arrow Cholesky of the equilibrated matrix, then iterative
    refinement of x in long double with long-double residuals of the unrounded A (equilibration itself rounds,
    which would cost kappa * eps).  Holds D, A_hat, y = D^-1 x and x.  beta defaults to the band A has."""

    def __init__(self, A, rhs, K, beta=None, refine=4):
        self.A, self.rhs = lower_symmetric(A), np.asarray(rhs, dtype=np.float64)
        beta = block_bandwidth(self.A, K) if beta is None else beta
        self.d, self.Ah = equilibrate(self.A)
        self.fac = BandArrowCholesky(self.Ah, 6 * K, beta)
        x = (self.d * self.fac.solve(self.d * self.rhs)).astype(np.longdouble)
        for _ in range(refine):
            r = residual_ld(self.A, x, self.rhs)
            x = x + self.d * self.fac.solve(self.d * r.astype(np.float64))
        self.x_ld = x
        self.x = x.astype(np.float64)
        self.y = (x / self.d).astype(np.float64)

    def kappa(self):
        """1-norm condition number of A_hat (= its inf-norm one: A_hat is symmetric); ||A_hat^-1||_1 estimated."""
        n = self.Ah.shape[0]
        inv = spla.LinearOperator((n, n), matvec=self.fac.solve, rmatvec=self.fac.solve, dtype=np.float64)
        return float(np.abs(self.Ah).sum(axis=0).max() * spla.onenormest(inv, t=4))


def mp_solve(A, rhs, dps=50):
    """mpmath LU solve at dps digits (small n only): cross-check of the reference itself."""
    import mpmath
    with mpmath.workdps(dps):
        x = mpmath.lu_solve(mpmath.matrix(A.tolist()), mpmath.matrix(list(rhs)))
        return np.array([float(v) for v in x])


# ---- metrics ----------------------------------------------------------------------------------------------
def entry_error(A, A_ref, fam=None):
    """max |A - A_ref|_ij / sqrt(A_ref_ii A_ref_jj); per pair of dof families when fam is given."""
    d = 1.0 / np.sqrt(np.abs(np.diag(A_ref)))
    E = np.abs(np.asarray(A) - A_ref) * d[:, None] * d[None, :]
    if fam is None:
        return float(E.max())
    return {(p, q): float(E[fam[p], fam[q]].max()) for p in fam for q in fam if fam[p].stop > fam[p].start and fam[q].stop > fam[q].start}


def rhs_error(b, b_ref, A_ref, fam=None):
    """max |D (b - b_ref)| / ||D b_ref||_inf with D = diag(A_ref)^-1/2; per dof family when fam is given."""
    d = 1.0 / np.sqrt(np.abs(np.diag(A_ref)))
    e = np.abs(d * (np.asarray(b) - b_ref)) / (np.abs(d * b_ref).max() + 1e-300)
    if fam is None:
        return float(e.max())
    return {f: float(e[s].max()) for f, s in fam.items() if s.stop > s.start}


def backward_error(A, rhs, x):
    """Normwise backward error of the equilibrated system: ||A_hat y - b_hat|| / (||A_hat|| ||y|| + ||b_hat||), inf-norms,
    y = D^-1 x; the residual D (rhs - A x) is taken in long double on the unrounded A.  A is read from its lower
    triangle, as the solvers read it."""
    A = lower_symmetric(A)
    d, Ah = equilibrate(A)
    x = np.asarray(x, dtype=np.float64)
    r = np.abs(d * residual_ld(A, x, rhs)).max()
    return float(r / (np.abs(Ah).sum(axis=1).max() * np.abs(x / d).max() + np.abs(d * rhs).max()))


def forward_error(x, ref, fam):
    """||y - y_ref||_inf over each dof family (and 'all') divided by ||y_ref||_inf, y = D^-1 x."""
    e = (np.abs(np.asarray(x, dtype=np.longdouble) - ref.x_ld) / ref.d).astype(np.float64) / np.abs(ref.y).max()
    out = {f: float(e[s].max()) for f, s in fam.items() if s.stop > s.start}
    out["all"] = float(e.max())
    return out


def forward_bound(n, kappa, c=8.0):
    return c * n * EPS * kappa


# ---- solver selection (ensure_system, hb200_api.cu) ------------------------------------------------------
def band_plan(K, beta):
    """hb::band_plan (hb200_band.cuh): (Kt, Kb, bs) block columns of chain 0 / chain 1 / separator."""
    if K >= 2 * beta + 4:
        Kt = (K - beta + 1) // 2
        return Kt, K - beta - Kt, beta
    return K, 0, 0


def band_workspace_bytes(K, beta, m):
    """hb::band_workspace_doubles (hb200_band.cuh) in bytes."""
    Kt, Kb, bs = band_plan(K, beta)
    h = 6 + 6 * beta
    n0, n1 = Kt + bs, (Kb + bs if Kb else 0)
    d = (n0 + n1) * h * 6 + (m + 1) * 6 * (n0 + n1) + (n0 + n1) * 48 + 6 * (n0 + n1)
    d += (m + 1) * (m | 1) + 2 * m
    d += 6 * K + m + (6 * K + m) // 8 + 1
    return 8 * (d + 8)


def bcr_smem_bytes(K, beta, m):
    nb = 6 * beta
    p1 = nb * (nb | 1) + nb + 1 + nb * (((2 * nb + m + 1 + 11) // 16) * 16 + 4) + (m + 1) * m
    p2 = 3 * nb * nb + 2 * nb * m + 2 * nb
    mp = ((m + 5) // 6) * 6
    p3 = mp * (mp | 1) + 3 * (mp + 1) + 8
    p4 = nb * (m + 1)
    p5 = 2 * (nb + 1) + 2 * nb + m + 2 + nb * (nb | 1)
    return 8 * max(p1, p2, p3, p4, p5)


def effective_beta(order, K, min_beta, max_track_rows=0):
    return min(max(order - 1, max_track_rows // 6 - 1, min_beta), max(K - 1, 0))


def solver_plan(K, beta, m, num_sms, force_dense=False):
    """Which reduced-system solver ensure_system picks, and how it splits the work.
    path: 'cluster' (band_solve_kernel<true>), 'bcr' (bcr_solve_kernel), 'chunked' (band_solve_kernel<false>), 'dense'."""
    n = 6 * K + m
    Kt, Kb, bs = band_plan(K, beta)
    p = dict(n=n, beta=beta, m=m, Kt=Kt, Kb=Kb, bs=bs, ws=band_workspace_bytes(K, beta, m))
    if force_dense or not (n <= 512 or 12 * (beta + 1) <= 6 * K):
        p.update(path="dense", kernel="cholesky_kernel")
        return p
    if p["ws"] <= SMEM_LIMIT:
        p.update(path="cluster", kernel="band_solve_kernel")
        return p
    if 6 * beta <= BCR_MAX_NB and m <= BCR_MAX_M and bcr_smem_bytes(K, beta, m) <= SMEM_LIMIT:
        nsb = (K + beta - 1) // beta
        p.update(path="bcr", kernel="bcr_solve_kernel", nsb=nsb, ctas=max(1, min(num_sms, (nsb + 1) // 2)))
        return p
    colbytes = ((6 + 6 * beta) * 6 + 6 * (m + 1) + 48) * 8
    cols = max(beta + 2, min((200 * 1024) // (2 * colbytes), K + beta))
    ch = cols - beta                                             # columns eliminated per chunk (run_chunked)
    last = max(Kt, Kb) - ch * ((max(Kt, Kb) - 1) // ch)          # columns in the last chunk of the chain phase
    p.update(path="chunked", kernel="band_solve_kernel<false>", chunk_cols=cols, chunk=ch, last_chunk=last,
             chunk_smem=2 * colbytes * cols)
    return p


def max_resident_K(beta, m, limit=400):
    """Largest K whose two-chain workspace fits SMEM_LIMIT (every K above it does not)."""
    fits = [K for K in range(beta + 1, limit) if band_workspace_bytes(K, beta, m) <= SMEM_LIMIT]
    return max(fits)


# ---- synthetic systems ------------------------------------------------------------------------------------
def make_system(K, beta, m, seed=0, kappa=1e5, zero_diagH=3, rows_per_block=3):
    """Synthetic SPD band + arrow system (S, b, g, diagH) with graded dof scales.

    S = G (J^T J + alpha I) G.  Every row of J spans exactly beta + 1 consecutive control-point blocks (so the
    outermost band block is never zero) plus random arrow columns; alpha sets kappa(A_hat) near `kappa`.
    G grades the families like the real system: diag(S) of the pose dofs near 1, gyro / accel bias near
    1e-9 / 1e-7, gravity near 1e-5.  diagH = diag(S) times a factor in [1, 3], with `zero_diagH` entries zeroed
    and one set below 1e-6 so that the damping clamp acts."""
    rng = np.random.default_rng(seed)
    np_, n = 6 * K, 6 * K + m
    w, rows = 6 * (beta + 1), 6 * rows_per_block
    M = np.zeros((n, n))
    for s in range(K - beta):                       # rows starting at control point s: J_s = [pose block | arrow]
        cols = np.r_[6 * s:6 * s + w, np_:n]
        Js = np.concatenate([rng.standard_normal((rows, w)), rng.standard_normal((rows, m)) * (rng.random((rows, m)) < 0.3)], axis=1)
        M[np.ix_(cols, cols)] += Js.T @ Js
    M += (np.abs(M).sum(axis=1).max() / kappa) * np.eye(n)
    Kb3 = (m - 2) // 2
    scale = np.concatenate([10.0 ** rng.uniform(-0.5, 0.0, np_), 10.0 ** rng.uniform(-4.7, -4.3, Kb3),
                            10.0 ** rng.uniform(-3.7, -3.3, m - 2 - Kb3), 10.0 ** rng.uniform(-2.7, -2.3, 2)])
    S = lower_symmetric(M * scale[:, None] * scale[None, :])
    b = rng.standard_normal(n) * np.sqrt(np.diag(S))
    g = rng.standard_normal(n) * np.sqrt(np.diag(S))
    diagH = np.diag(S) * rng.uniform(1.0, 3.0, n)
    z = rng.choice(n, size=zero_diagH + 1, replace=False)
    diagH[z[:-1]] = 0.0
    diagH[z[-1]] = 1e-9
    return S, b, g, diagH


# ---- system / step parity against the oracle -------------------------------------------------------------------
SYS_EQ_TOL = 1e-9   # equilibrated entry / rhs error of an assembled system against the oracle's, per dof family


def check_system_and_step(S, b, dp, S_ref, b_ref, K, Kbg, Kba, tol=SYS_EQ_TOL):
    """Assert an assembled (damped, masked) system and its step against the oracle's system:
    * equilibrated entry and rhs errors per block family below tol;
    * the step's equilibrated backward error on the system it was solved from (S, b) below n eps (solve error alone);
    * its per-family forward error against the reference solution of the oracle's system below
      kappa (n e_S + e_b + 8 n eps) (assembly error plus solve error, amplified by the condition number).
    Returns the measured values."""
    fam = families(K, Kbg, Kba)
    n = S.shape[0]
    eS, eb = entry_error(S, S_ref, fam), rhs_error(b, b_ref, S_ref, fam)
    for key, v in list(eS.items()) + list(eb.items()):
        assert v < tol, (key, v)
    bwd = backward_error(S, b, dp)
    assert bwd < n * EPS, bwd
    ref = Reference(S_ref, b_ref, K)
    kappa = ref.kappa()
    fwd = forward_error(dp, ref, fam)
    bound = kappa * (n * max(eS.values()) + max(eb.values()) + 8 * n * EPS)
    assert all(v < bound for v in fwd.values()), (fwd, bound)
    return dict(entry=max(eS.values()), rhs=max(eb.values()), bwd=bwd, bwd_bound=n * EPS, fwd=fwd["all"], fwd_bound=bound, kappa=kappa,
                **{f"entry_{p}_{q}": v for (p, q), v in eS.items()}, **{f"rhs_{f}": v for f, v in eb.items()},
                **{f"fwd_{f}": v for f, v in fwd.items()})


def bias_values(state):
    """Bias spline knots without their stamp column (the stamps dwarf the values they would be compared with)."""
    return {k: state[k][:, :3] for k in ("gyro_bias", "accel_bias")}
