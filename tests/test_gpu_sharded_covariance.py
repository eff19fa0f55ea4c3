"""Marginal covariances on sharded contexts, on one GPU (need an H100): N contexts on device 0, each holding a
landmark-owner shard of the same window, reduce their undamped partial systems through the all-reduce callback
(hb200_set_allreduce) with the reducer of tests/test_gpu_sharded.py, which here also keeps every rank's input buffer.

Per partition (orders 4 and 6, two and three ranks, compact shards, a rank that owns no landmark; pixel, bearing, pose and
IMU factors):
* Sigma (band, arrow, corner), status and pivot are bit-identical across ranks;
* Sigma equals tests/covref.py's selected inverse of the rank-order float64 sum of the captured partials within
  sysref.forward_bound(n, kappa), and that sum is the reduced buffer every rank inverted, bit for bit;
* Sigma equals covref of asmref's long-double whole-window system (from one context's factor outputs) within the bound
  check_e2e of tests/test_gpu_covariance.py uses;
* landmark blocks read from their owners match covref's marginals within 10x the bound; non-owned blocks are exactly 0;
  L and unobserved_landmarks are rank-local;
* interpolated covariances are bit-identical across ranks and within 1e-11 of covref.
Failures: a single-observation landmark on one rank makes every rank report status 2 with the same count and keep its
previous results; a window without a gauge makes every rank report status 1 with the same bad_dof.
Deterministic contexts: iterate(2) -> covariance -> iterate(2) equals iterate(4) bit for bit, two build + compute pairs
are bit-identical, and hb200_get_system refuses (-2) after the covariance build.
"""
import numpy as np
import pytest

import asmref as ar
import covref as cr
import sysref as sr
from hyperslam_b200 import runtime
from test_gpu_covariance import e2e_window, read_system
from test_gpu_sharded import HostReducer, on_ranks, open_ranks, shard_by_owner

pytestmark = pytest.mark.gpu


class KeepingReducer(HostReducer):
    """HostReducer that keeps a copy of each rank's input buffer of the last reduction (taken on the rank's stream before
    the sum is copied back)."""

    def __init__(self, n):
        super().__init__(n)
        self.inputs = [None] * n

    def hook(self, rank, stream):
        torch = self.torch
        ext = torch.cuda.ExternalStream(stream, device=self.dev)
        inner = super().hook(rank, stream)

        def allreduce(ptr, count, s):
            with torch.cuda.stream(ext):
                self.inputs[rank] = self._wrap(ptr, count).clone()
            return inner(ptr, count, s)
        return allreduce

    def captured(self):
        self.torch.cuda.synchronize()
        return [b.cpu().numpy().copy() for b in self.inputs]


def shape(win):
    K, Kbg, Kba = win.knots.shape[0], win.gyro_bias.shape[0], win.accel_bias.shape[0]
    m = 3 * (Kbg + Kba) + 2
    return K, m, 6 * K + m, sr.fixed_mask(K, Kbg, Kba, win.knot_const, win.bias_const, win.gravity_const)


def stamps_of(win):
    kt, k = win.knots[:, 7], win.order
    left = (k - 1) // 2
    lo, hi = kt[left], kt[len(kt) - k + left + 1]
    return np.concatenate([[lo, np.nextafter(hi, -np.inf)], kt[left + 1:left + 5], 0.5 * (kt[6:10] + kt[7:11])])


def covariance_on_ranks(red, ctxs, stamps):
    """build + compute on every rank (collective), then each rank's results."""
    infos = on_ranks(red, ctxs, lambda r, c: (c.build_covariance(), c.compute_covariance())[1])
    out = []
    for c, info in zip(ctxs, infos):
        res = dict(info=info, reduced=read_system(c))
        if info["status"] == 0:
            res["packed"], res["lm"], _ = c.covariance_packed()
            res["interp"], res["bad"] = c.interpolate_covariance(stamps)
        out.append(res)
    return out


def same_bits(a, b):
    return np.array_equal(np.asarray(a, np.float64).view(np.int64), np.asarray(b, np.float64).view(np.int64))


CASES = {"k4-n2-scattered": (4, 2, "scattered", False), "k6-n3-compact": (6, 3, "scattered", True),
         "k4-n3-empty-rank": (4, 3, "two", False), "k6-n2-compact": (6, 2, "blocks", True)}


@pytest.mark.parametrize("case", list(CASES))
def test_sharded_covariance(built, record_property, case):
    order, world, owners, compact = CASES[case]
    win = e2e_window(order, num_knots=30, num_landmarks=300, num_imu=800, bearing=150, pose=10, seed=60 + order + world)
    K, m, n, fixed = shape(win)
    L = win.landmarks.shape[0]
    rng = np.random.default_rng(6000 + order + world)
    if owners == "scattered":
        owner = rng.integers(0, world, L)
    elif owners == "two":       # the last rank owns no landmark: no visual factor there
        owner = rng.integers(0, world - 1, L)
    else:
        owner = np.searchsorted([(L * r) // world for r in range(world + 1)], np.arange(L), side="right") - 1
    shards, index = shard_by_owner(win, owner, world, compact=compact)
    stamps = stamps_of(win)
    ctxs, _, beta = open_ranks(shards)
    try:
        red = KeepingReducer(world)
        red.attach(ctxs)
        res = covariance_on_ranks(red, ctxs, stamps)
        parts = red.captured()
        probs = [ar.problem(c.outputs(), s, c.index_maps()) for c, s in zip(ctxs, shards)]
        knots = ctxs[0].state()["knots"]
    finally:
        for c in ctxs:
            c.close()
    single = runtime.Context(0)
    try:
        single.load_window(win)
        single.set_min_bandwidth(beta)
        single.evaluate()
        p_full = ar.problem(single.outputs(), win, single.index_maps())
    finally:
        single.close()

    info0 = res[0]["info"]
    assert info0["status"] == 0, info0
    for r in range(world):
        info = res[r]["info"]
        for key in ("status", "bad_dof", "min_pivot_ratio", "degenerate_landmarks", "K", "beta", "m"):
            assert info[key] == info0[key], (r, key, info, info0)
        assert same_bits(res[r]["packed"], res[0]["packed"]), r
        assert same_bits(res[r]["interp"], res[0]["interp"]), r
        held = shards[r].landmarks.shape[0]
        seen = np.zeros(held, bool)
        seen[shards[r].v_lm] = True
        seen[shards[r].b_lm] = True
        assert (info["L"], info["unobserved_landmarks"]) == (held, int((~seen).sum())), (r, info)
    assert (info0["K"], info0["beta"], info0["m"]) == (K, beta, m)

    # the rank-order float64 sum of the partials is what every rank inverted
    tot = parts[0].copy()
    for p in parts[1:]:
        tot += p
    for r in range(world):
        assert same_bits(res[r]["reduced"], tot), r
    S_dev, *_ = sr.unpack_system(tot, K, beta, m)
    ref, P, _, bad = cr.selected_inverse(S_dev, K, beta, m, fixed)
    assert bad == -1
    kap = cr.kappa(S_dev, fixed)
    bound = sr.forward_bound(n, kap)
    got = cr.packed_to_dense(res[0]["packed"], K, beta, m)
    err = cr.cov_error(got, ref, P)
    # against asmref's long-double system of the whole window
    a = ar.assemble(p_full, np.inf)
    keep = ~fixed
    eS = sr.entry_error(S_dev[np.ix_(keep, keep)], a["S"].astype(np.float64)[np.ix_(keep, keep)])
    ref_a, _, _, bad_a = cr.selected_inverse(a["S"], K, beta, m, fixed)
    assert bad_a == -1
    err_a = cr.cov_error(got, ref_a, P)
    bound_a = kap * (n * eS + 8 * n * sr.EPS)
    for k, v in dict(n=n, beta=beta, kappa=kap, err_own=err, bound_own=bound, err_asmref=err_a, bound_asmref=bound_a).items():
        record_property(k, v)
    print(f"{case}: kappa {kap:.3e}, err {err:.3e} / {bound:.3e}, asmref {err_a:.3e} / {bound_a:.3e}")
    assert err < bound, (err, bound)
    assert err_a < bound_a, (err_a, bound_a, eS)
    assert np.all(got[fixed] == 0) and np.all(got[:, fixed] == 0)

    # landmark blocks from their owners; held, non-owned blocks are exactly zero
    worst = 0.0
    for r in range(world):
        mine = owner[index[r]] == r
        lm = res[r]["lm"]
        assert np.isfinite(lm).all() and np.all(lm[~mine] == 0), r
        lm_ref = cr.landmark_marginals(probs[r], ref)
        for l in np.nonzero(mine)[0]:
            if np.abs(lm_ref[l]).max() > 0:
                worst = max(worst, cr.cov_error(lm[l], lm_ref[l]))
            else:
                assert np.all(lm[l] == 0)
    record_property("err_landmarks", worst)
    assert worst < 10 * bound, (worst, bound)

    # interpolated pose covariances
    assert res[0]["bad"] == 0
    werr = max(cr.cov_error(res[0]["interp"][i], cr.interpolated(knots, order, t, got)) for i, t in enumerate(stamps))
    record_property("err_interpolated", werr)
    assert werr < 1e-11, werr


# ---- failures ---------------------------------------------------------------------------------------------------------
def load_ranks(ctxs, shards):
    """Load new shards into open contexts and agree on the half-width again (what open_ranks does at creation)."""
    for c, s in zip(ctxs, shards):
        c.load_window(s)
    beta = max(c.bandwidth() for c in ctxs)
    for c in ctxs:
        c.set_min_bandwidth(beta)


def test_failures_on_every_rank(built, record_property):
    world = 3
    good = e2e_window(4, num_knots=30, num_landmarks=200, num_imu=800, bearing=100, pose=10, seed=31)
    L = good.landmarks.shape[0]
    owner = np.random.default_rng(31).integers(0, world, L)
    stamps = stamps_of(good)
    ctxs, _, _ = open_ranks(shard_by_owner(good, owner, world)[0])
    try:
        red = HostReducer(world)
        red.attach(ctxs)
        res0 = covariance_on_ranks(red, ctxs, stamps)
        assert all(r["info"]["status"] == 0 for r in res0)
        keep = [c.covariance_packed() for c in ctxs]

        def same_as_before():
            for c, k in zip(ctxs, keep):
                now = c.covariance_packed()
                assert same_bits(now[0], k[0]) and same_bits(now[1], k[1])

        # one landmark seen by a single pixel factor: degenerate on its owner only, reported by every rank
        single = e2e_window(4, num_knots=30, num_landmarks=200, num_imu=800, bearing=0, pose=10, seed=31)
        o = np.nonzero(single.v_lm == 7)[0]
        keepv = np.ones(single.v_stamp.size, bool)
        keepv[o[1:]] = False
        for key in ("v_stamp", "v_cam", "v_lm", "v_pixel"):
            setattr(single, key, np.ascontiguousarray(getattr(single, key)[keepv]))
        load_ranks(ctxs, shard_by_owner(single, owner, world)[0])
        infos = on_ranks(red, ctxs, lambda r, c: (c.build_covariance(), c.compute_covariance())[1])
        record_property("degenerate_owner", int(owner[7]))
        for info in infos:
            assert info["status"] == 2 and info["rc"] == runtime.COV_DEGENERATE_LANDMARKS and info["degenerate_landmarks"] == 1, info
        same_as_before()
        # no gauge: no constant knots but the untouched ones, no pose factors
        nogauge = e2e_window(4, num_knots=30, num_landmarks=200, num_imu=800, bearing=100, pose=0, seed=31)
        nogauge.knot_const = cr.untouched_knots(nogauge).astype(np.uint8)
        load_ranks(ctxs, shard_by_owner(nogauge, owner, world)[0])
        infos = on_ranks(red, ctxs, lambda r, c: (c.build_covariance(), c.compute_covariance())[1])
        record_property("gauge_free_bad_dof", infos[0]["bad_dof"])
        for info in infos:
            assert info["status"] == 1 and info["rc"] == runtime.COV_NOT_POSITIVE_DEFINITE and info["bad_dof"] >= 0, info
            assert (info["bad_dof"], info["min_pivot_ratio"]) == (infos[0]["bad_dof"], infos[0]["min_pivot_ratio"])
        same_as_before()
    finally:
        for c in ctxs:
            c.close()


# ---- deterministic contexts: the LM loop around a covariance ---------------------------------------------------------
def test_deterministic_lm_around_covariance(built):
    world = 2
    win = e2e_window(4, num_knots=30, num_landmarks=300, num_imu=800, bearing=150, pose=10, seed=71)
    L = win.landmarks.shape[0]
    owner = np.random.default_rng(71).integers(0, world, L)
    shards, _ = shard_by_owner(win, owner, world)
    stamps = stamps_of(win)
    keys = ("cost", "cost_new", "model_change", "rho", "radius", "accepted", "spd")

    def run(with_cov):
        ctxs, _, _ = open_ranks(shards)
        try:
            for c in ctxs:
                c.set_deterministic(True)
            red = HostReducer(world)
            red.attach(ctxs)
            covs = None
            if with_cov:
                recs = on_ranks(red, ctxs, lambda r, c: c.iterate(2))
                covs = [covariance_on_ranks(red, ctxs, stamps) for _ in range(2)]
                for c in ctxs:
                    with pytest.raises(runtime.HB200Error, match="hb200 error -2"):
                        c.system()
                more = on_ranks(red, ctxs, lambda r, c: c.iterate(2))
                recs = [a + b for a, b in zip(recs, more)]
            else:
                recs = on_ranks(red, ctxs, lambda r, c: c.iterate(4))
            states = [c.state() for c in ctxs]
        finally:
            for c in ctxs:
                c.close()
        return [[[x[k] for k in keys] for x in rr] for rr in recs], states, covs

    recs_a, states_a, covs = run(True)
    recs_b, states_b, _ = run(False)
    assert recs_a == recs_b
    for sa, sb in zip(states_a, states_b):
        for key in sa:
            assert same_bits(sa[key], sb[key]), key
    first, second = covs
    for r in range(world):
        assert first[r]["info"]["status"] == 0
        assert first[r]["info"] == second[r]["info"]
        for key in ("reduced", "packed", "lm", "interp"):
            assert same_bits(first[r][key], second[r][key]), (r, key)
