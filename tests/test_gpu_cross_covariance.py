"""Covariance blocks outside the selected inverse's pattern on the device (need an H100): hb200_set_covariance_blocks /
hb200_get_covariance_blocks against tests/crosscovref.py and tests/covref.py.

* far knot pairs equal covref.dense_inverse_ld of the device's own undamped system within sysref.forward_bound(n, kappa)
  (the bound check_e2e of tests/test_gpu_covariance.py uses); landmark x knot / bias / gravity and landmark x landmark
  blocks equal the long-double formulas on that inverse and the device's factor outputs within 10x the bound; the
  largest normalised reference entry among them is >= 1e3 x the bound (a march that returned zeros would fail);
* pairs in the pattern are bit-identical to hb200_get_covariance, (b, a) is exactly the transpose of (a, b), constant
  dofs are 0, an unobserved landmark gets status 2 and a zero block;
* snapshot: iterations, failed computes and a registration without a compute leave the committed blocks as they are; a
  bad index makes the compute return -1 and launch nothing;
* a compute without requests launches two kernels; in deterministic mode a context that registered and cleared a list
  gives Sigma and the landmark blocks bit for bit as one that never registered; two computes are bit-identical in both
  assembly modes;
* sharded on one GPU (2 contexts, the all-reduce callback): knot, bias and gravity pairs are bit-identical across ranks
  and match the dense inverse of the rank-order sum; landmark pairs come from their owner, status 1 elsewhere;
* hyper::Covariance with Options::full_pattern (host binary cross_covariance_test) accepts the pairs the default options
  refuse, and its tangent and ambient blocks match the C-ABI blocks through covref.ceres_tangent / covref.ambient.
"""
import os
import subprocess

import numpy as np
import pytest

import asmref as ar
import covref as cr
import crosscovref as xr
import sysref as sr
from hyperslam_b200 import runtime
from test_gpu_covariance import e2e_window, failure_window, gauge_free_window, read_system
from test_gpu_host_covariance import dump_window
from test_gpu_sharded import HostReducer, on_ranks, open_ranks, shard_by_owner

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KN, BG, BA, GR, LM = runtime.COV_KNOT, runtime.COV_GYRO_BIAS, runtime.COV_ACCEL_BIAS, runtime.COV_GRAVITY, runtime.COV_LANDMARK


def same_bits(a, b):
    return np.array_equal(np.asarray(a, np.float64).view(np.int64), np.asarray(b, np.float64).view(np.int64))


def dofs(kind, i, K, Kbg, Kba):
    o = 6 * K
    return {KN: 6 * i + np.arange(6), BG: o + 3 * i + np.arange(3), BA: o + 3 * Kbg + 3 * i + np.arange(3),
            GR: o + 3 * (Kbg + Kba) + np.arange(2)}[kind]


def requests(K, Kbg, Kba, L, beta, rng, n_lm=40):
    """Far knot pairs (both orders), pairs in the pattern, landmark x knot / bias / gravity and landmark pairs."""
    req = []
    for i in range(0, K, 3):
        for j in range(i + beta + 1, K, 4):
            req.append((KN, i, KN, j) if (i + j) % 2 else (KN, j, KN, i))
    req += [(KN, 5, KN, 5), (KN, 5, KN, 5 + beta), (KN, 5 + beta, KN, 5), (KN, 7, BG, 1), (BA, 2, KN, 9), (GR, 0, GR, 0), (BG, 0, BA, Kba - 1)]
    ls = rng.integers(0, L, (n_lm, 2))
    ks = rng.integers(0, K, n_lm)
    for q in range(n_lm):
        l, m, j = int(ls[q, 0]), int(ls[q, 1]), int(ks[q])
        req.append((LM, l, KN, j) if q % 2 else (KN, j, LM, l))
        req.append((LM, l, LM, m if m != l else (m + 1) % L))
    req += [(LM, 3, BG, 0), (BA, Kba - 1, LM, 4), (LM, 5, GR, 0), (GR, 0, LM, 6), (LM, 7, LM, 7)]
    req += [(kb, ib, ka, ia) for ka, ia, kb, ib in req[-12:]]   # reversed: exact transposes
    return np.array(req, np.int32)


def compute(ctx, req):
    """register, build, read the system, compute; (system, info, launches, packed, lm, blocks, status)."""
    ctx.set_covariance_blocks(req)
    ctx.build_covariance()
    buf = read_system(ctx)
    l0 = ctx.launch_count
    info = ctx.compute_covariance()
    launches = ctx.launch_count - l0
    assert info["status"] == 0, info
    packed, lm, _ = ctx.covariance_packed()
    blocks, st = ctx.covariance_blocks()
    return buf, info, launches, packed, lm, blocks, st


def reference_blocks(req, p, Sig, lm_ref, K, Kbg, Kba):
    """Long-double blocks of each request from a full Sigma (the dense inverse) and the factor outputs, and the square
    roots of the diagonals of both sides (for the normalised error)."""
    terms = xr.landmark_terms(p)
    dg = np.sqrt(np.abs(np.diagonal(Sig)).astype(np.float64))
    out = []
    for ka, ia, kb, ib in req:
        flip = ka != LM and kb == LM
        if flip:
            ka, ia, kb, ib = kb, ib, ka, ia
        if ka == LM and kb == LM:
            want = lm_ref[ia] if ia == ib else xr.landmark_pair(terms, Sig, ia, ib)
            da, db = np.sqrt(np.abs(np.diag(lm_ref[ia]))), np.sqrt(np.abs(np.diag(lm_ref[ib])))
        elif ka == LM:
            d = dofs(kb, ib, K, Kbg, Kba)
            want, da, db = xr.landmark_cross(terms, Sig, ia, d), np.sqrt(np.abs(np.diag(lm_ref[ia]))), dg[d]
        else:
            a, b = dofs(ka, ia, K, Kbg, Kba), dofs(kb, ib, K, Kbg, Kba)
            want, da, db = np.asarray(Sig)[np.ix_(a, b)], dg[a], dg[b]
        want, da, db = np.asarray(want, np.longdouble), np.asarray(da, np.float64), np.asarray(db, np.float64)
        out.append((want.T, db, da) if flip else (want, da, db))
    return out


def normalised(x, da, db):
    s = np.outer(da, db)
    return np.where(s > 0, np.abs(np.asarray(x, np.float64)) / np.where(s > 0, s, 1), 0.0)


def check_blocks(req, blocks, st, want, packed, lm, K, beta, m, fixed, Kbg, Kba):
    """Layout, exact copies of the pattern, exact transposes, constant dofs; returns (errors far, cross) and the largest
    normalised reference entry of the far and landmark blocks."""
    T = runtime.COV_TANGENT
    got_sig = cr.packed_to_dense(packed, K, beta, m)
    err_far, err_lm, biggest = 0.0, 0.0, 0.0
    seen = {}
    for q, ((ka, ia, kb, ib), (w, da, db)) in enumerate(zip(req, want)):
        ta, tb = T[int(ka)], T[int(kb)]
        blk = blocks[q]
        assert st[q] == 0, (q, req[q], st[q])
        assert np.all(blk[ta:, :] == 0) and np.all(blk[:, tb:] == 0), q
        b = blk[:ta, :tb]
        key = (int(ka), int(ia), int(kb), int(ib))
        if (key[2], key[3], key[0], key[1]) in seen:
            assert same_bits(b, seen[(key[2], key[3], key[0], key[1])].T), key
        seen[key] = b
        if ka != LM and kb != LM:
            a, c = dofs(ka, ia, K, Kbg, Kba), dofs(kb, ib, K, Kbg, Kba)
            assert np.all(b[fixed[a], :] == 0) and np.all(b[:, fixed[c]] == 0), key
            far = ka == KN and kb == KN and abs(int(ia) - int(ib)) > beta
            if not far:   # in the pattern: bit for bit
                assert same_bits(b, got_sig[np.ix_(a, c)]), key
                continue
            err_far = max(err_far, float(normalised(b - w, da, db).max()))
        elif ka == LM and kb == LM and ia == ib:
            assert same_bits(b, lm[ia]), key
            continue
        else:
            err_lm = max(err_lm, float(normalised(b - w, da, db).max()))
        biggest = max(biggest, float(normalised(w, da, db).max()))
    return err_far, err_lm, biggest


CASES = {"k4-cfg1": (4, 50), "k6-cfg1": (6, 50), "k4-K150": (4, 150), "k6-K150": (6, 150)}


@pytest.mark.parametrize("case", list(CASES))
def test_far_and_landmark_blocks(built, record_property, case):
    order, K = CASES[case]
    win = e2e_window(order, num_knots=K, num_landmarks=1000 if K == 50 else 1500, num_imu=2000 if K == 50 else 6000, seed=80 + order + K)
    Kbg, Kba, L = win.gyro_bias.shape[0], win.accel_bias.shape[0], win.landmarks.shape[0]
    m = 3 * (Kbg + Kba) + 2
    n = 6 * K + m
    ctx = runtime.Context(0)
    try:
        ctx.load_window(win)
        beta = ctx.bandwidth()
        req = requests(K, Kbg, Kba, L, beta, np.random.default_rng(K + order))
        buf, info, launches, packed, lm, blocks, st = compute(ctx, req)
        out, maps = ctx.outputs(), ctx.index_maps()
        # a second compute of the same build: bit for bit (the assembly's atomics ran once, in the build)
        info2 = ctx.compute_covariance()
        blocks2, st2 = ctx.covariance_blocks()
    finally:
        ctx.close()
    # selected inverse, landmark marginals, span read-back, far columns, requested blocks
    assert launches == 5, launches
    assert info2 == info and same_bits(blocks2, blocks) and np.array_equal(st2, st)
    fixed = sr.fixed_mask(K, Kbg, Kba, win.knot_const, win.bias_const, win.gravity_const)
    S_dev, *_ = sr.unpack_system(buf, K, beta, m)
    Sig = cr.dense_inverse_ld(S_dev, fixed)
    bound = sr.forward_bound(n, cr.kappa(S_dev, fixed))
    p = ar.problem(out, win, maps)
    lm_ref = cr.landmark_marginals(p, Sig)
    want = reference_blocks(req, p, Sig, lm_ref, K, Kbg, Kba)
    err_far, err_lm, biggest = check_blocks(req, blocks, st, want, packed, lm, K, beta, m, fixed, Kbg, Kba)
    for k, v in dict(n=n, beta=beta, requests=len(req), bound=bound, err_far=err_far, err_landmark=err_lm, largest_reference=biggest).items():
        record_property(k, v)
    print(f"{case}: beta {beta}, {len(req)} requests, far err {err_far:.3e}, landmark err {err_lm:.3e}, bound {bound:.3e}, largest {biggest:.3e}")
    assert err_far < bound, (err_far, bound)
    assert err_lm < 10 * bound, (err_lm, bound)
    assert biggest >= 1e3 * bound, (biggest, bound)


def test_status_snapshot_and_refusals(built):
    """Unobserved landmark (status 2), a bad index (-1, nothing launched), iterations, failed computes and a registration
    without a compute (the committed blocks stay)."""
    win = failure_window()
    keepv = win.v_lm != 5
    for key in ("v_stamp", "v_cam", "v_lm", "v_pixel"):
        setattr(win, key, np.ascontiguousarray(getattr(win, key)[keepv]))
    keepb = win.b_lm != 5
    for key in ("b_stamp", "b_cam", "b_lm", "b_bearing"):
        setattr(win, key, np.ascontiguousarray(getattr(win, key)[keepb]))
    K = win.knots.shape[0]
    req = np.array([(LM, 5, KN, 20), (LM, 5, LM, 5), (LM, 6, LM, 5), (LM, 6, KN, 25), (KN, 2, KN, 25)], np.int32)
    ctx = runtime.Context(0)
    try:
        ctx.set_deterministic(True)
        with pytest.raises(runtime.HB200Error, match="hb200 error -2"):
            ctx.covariance_blocks()                       # before any compute
        ctx.load_window(win)
        _, info, _, _, _, blocks, st = compute(ctx, req)
        assert info["unobserved_landmarks"] == 1
        assert list(st) == [2, 2, 2, 0, 0] and np.all(blocks[:3] == 0) and np.abs(blocks[3:, :3, :3]).max() > 0
        ctx.iterate(2)
        b, s = ctx.covariance_blocks()
        assert same_bits(b, blocks) and np.array_equal(s, st)
        # registering changes nothing until a compute; the committed count stays
        ctx.set_covariance_blocks(req[:2])
        b, _ = ctx.covariance_blocks()
        assert same_bits(b, blocks)
        # a bad index: -1, nothing launched, the previous blocks stay
        ctx.set_covariance_blocks([(KN, K, KN, 0)])
        ctx.build_covariance()
        l0 = ctx.launch_count
        with pytest.raises(runtime.HB200Error, match="hb200 error -1"):
            ctx.compute_covariance()
        assert ctx.launch_count == l0
        ctx.set_covariance_blocks(req)
        b, _ = ctx.covariance_blocks()
        assert same_bits(b, blocks)
        # failed computes (status 1: no gauge) keep the blocks and their count
        ctx.load_window(gauge_free_window())
        ctx.set_covariance_blocks(req[3:])
        ctx.build_covariance()
        assert ctx.compute_covariance()["status"] == 1
        b, s = ctx.covariance_blocks()
        assert same_bits(b, blocks) and np.array_equal(s, st)
        # a count other than the committed one
        assert ctx.lib.hb200_get_covariance_blocks(ctx.h, 2, runtime._d(np.zeros(72)), None) == -2
    finally:
        ctx.close()


def test_no_requests_unchanged(built):
    """Without a list: two launches, and (deterministic mode) registering then clearing a list leaves Sigma and the
    landmark blocks bit for bit as a context that never registered one."""
    win = e2e_window(4, num_knots=30, num_landmarks=300, num_imu=800, bearing=100, pose=10, seed=91)

    def run(register):
        ctx = runtime.Context(0)
        try:
            ctx.set_deterministic(True)
            ctx.load_window(win)
            if register:
                ctx.set_covariance_blocks([(KN, 0, KN, 20), (LM, 1, LM, 2)])
                ctx.build_covariance()
                ctx.compute_covariance()
                ctx.set_covariance_blocks([])
            ctx.build_covariance()
            l0 = ctx.launch_count
            info = ctx.compute_covariance()
            launches = ctx.launch_count - l0
            packed, lm, _ = ctx.covariance_packed()
            blocks, st = ctx.covariance_blocks()
        finally:
            ctx.close()
        return info, launches, packed, lm, blocks

    a, b = run(False), run(True)
    assert a[1] == 2 and b[1] == 2
    assert a[0] == b[0] and same_bits(a[2], b[2]) and same_bits(a[3], b[3])
    assert a[4].shape == (0, 6, 6) and b[4].shape == (0, 6, 6)


def test_deterministic_requests_repeat(built):
    """Deterministic assembly: two build + compute rounds give the same blocks bit for bit."""
    win = e2e_window(6, num_knots=30, num_landmarks=300, num_imu=800, bearing=100, pose=10, seed=92)
    ctx = runtime.Context(0)
    try:
        ctx.set_deterministic(True)
        ctx.load_window(win)
        req = requests(30, win.gyro_bias.shape[0], win.accel_bias.shape[0], 300, ctx.bandwidth(), np.random.default_rng(92), n_lm=20)
        first = compute(ctx, req)
        second = compute(ctx, req)
    finally:
        ctx.close()
    assert same_bits(first[5], second[5]) and np.array_equal(first[6], second[6])


def test_sharded_blocks(built, record_property):
    world = 2
    win = e2e_window(4, num_knots=30, num_landmarks=300, num_imu=800, bearing=150, pose=10, seed=93)
    K, Kbg, Kba, L = 30, win.gyro_bias.shape[0], win.accel_bias.shape[0], win.landmarks.shape[0]
    m = 3 * (Kbg + Kba) + 2
    n = 6 * K + m
    owner = np.random.default_rng(93).integers(0, world, L)
    shards, index = shard_by_owner(win, owner, world)   # every rank holds every landmark (not compact)
    ctxs, _, beta = open_ranks(shards)
    state = [(KN, 1, KN, 20), (KN, 25, KN, 3), (KN, 10, KN, 10 + beta + 1), (BG, 1, KN, 28), (GR, 0, KN, 15)]
    mine = [int(np.nonzero(owner == r)[0][0]) for r in range(world)]
    both = [int(l) for l in np.nonzero(owner == 0)[0][1:3]]
    lmreq = [(LM, mine[0], KN, 22), (LM, mine[1], KN, 12), (LM, both[0], LM, both[1]), (LM, mine[1], GR, 0)]   # (knots 0..3 constant)
    req = np.array(state + lmreq, np.int32)
    try:
        red = HostReducer(world)
        red.attach(ctxs)
        res = on_ranks(red, ctxs, lambda r, c: (c.set_covariance_blocks(req), c.build_covariance(), c.compute_covariance())[2])
        assert all(i["status"] == 0 for i in res), res
        got = [c.covariance_blocks() for c in ctxs]
        bufs = [read_system(c) for c in ctxs]
    finally:
        for c in ctxs:
            c.close()
    ns = len(state)
    for r in range(world):
        assert same_bits(got[r][0][:ns], got[0][0][:ns]) and np.all(got[r][1][:ns] == 0)
    # the reduced buffer is the same on every rank; Sigma of it in long double
    assert same_bits(bufs[0], bufs[1])
    S_dev, *_ = sr.unpack_system(bufs[0], K, beta, m)
    fixed = sr.fixed_mask(K, Kbg, Kba, win.knot_const, win.bias_const, win.gravity_const)
    Sig = cr.dense_inverse_ld(S_dev, fixed)
    bound = sr.forward_bound(n, cr.kappa(S_dev, fixed))
    dg = np.sqrt(np.abs(np.diagonal(Sig)).astype(np.float64))
    err = 0.0
    for q, (ka, ia, kb, ib) in enumerate(state):
        a, b = dofs(ka, ia, K, Kbg, Kba), dofs(kb, ib, K, Kbg, Kba)
        blk = got[0][0][q][:len(a), :len(b)]
        err = max(err, float(normalised(blk - np.asarray(Sig)[np.ix_(a, b)], dg[a], dg[b]).max()))
    record_property("err_state", err)
    assert err < bound, (err, bound)
    # landmark pairs: computed by the owner, status 1 on the other rank
    expect_owner = [0, 1, 0, 1]
    for q, r in enumerate(expect_owner):
        assert got[r][1][ns + q] == 0 and np.abs(got[r][0][ns + q]).max() > 0, (q, r)
        assert got[1 - r][1][ns + q] == 1 and np.all(got[1 - r][0][ns + q] == 0), (q, r)


@pytest.mark.parametrize("order", [4, 6])
def test_host_full_pattern(built, tmp_path, record_property, order):
    exe = os.path.join(ROOT, "hyperslam_b200", "lib", "cross_covariance_test")
    assert os.path.exists(exe), "cross_covariance_test not built (python -c 'import __graft_entry__ as g; g.build()')"
    import oracle_lib as ol
    from hyperslam_b200 import synthetic
    base = synthetic.make_window(order=order, num_knots=20, num_landmarks=60, num_imu=400, seed=synthetic.SEED_BASE + 2400 + order)
    win = synthetic.add_bearing_and_pose_factors(base, num_bearing=20, num_pose=8, seed=synthetic.SEED_BASE + 2450 + order)
    win.knot_const = np.zeros(20, np.uint8)
    win.knot_const[:order] = 1
    win.knot_const[cr.untouched_knots(win)] = 1
    win.bias_const, win.gravity_const = 0, 0
    src, dst = tmp_path / "window.txt", tmp_path / "out.txt"
    dump_window(win, src)
    res = subprocess.run([exe, str(src), str(dst)], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, res.stdout + res.stderr
    lines = open(dst).read().split("\n")
    head = lines[0].split()
    assert head[:6] == ["refused", "3", "3", "accepted", "3", "beta"], head   # off: refused; on: accepted
    beta = int(head[6])
    assert lines[1].split()[:3] == ["compute", "1", "0"]
    kinds = {"state": KN, "gyro": BG, "accel": BA, "gravity": GR, "landmark": LM}
    pairs, tans, ambs = [], [], []
    i = 2
    while lines[i].startswith("pair"):
        _, ka, ja, kb, jb = lines[i].split()
        pairs.append((kinds[ka], int(ja), kinds[kb], int(jb)))
        tans.append(np.array(lines[i + 1].split(), float))
        ambs.append(np.array(lines[i + 2].split(), float))
        i += 3
    assert lines[i].split() == ["failures", "0"] and len(pairs) == 12
    ctx = runtime.Context(0)
    try:
        ctx.load_window(win)
        assert ctx.bandwidth() == beta
        ctx.set_covariance_blocks(pairs)
        ctx.build_covariance()
        assert ctx.compute_covariance()["status"] == 0
        blocks, st = ctx.covariance_blocks()
    finally:
        ctx.close()
    assert np.all(st == 0)

    def conv(kind, j):
        if kind == KN:
            return np.diag([0.5, 0.5, 0.5, 1, 1, 1]), ol.manifold_plus_jacobian(ol.M_STATE, win.knots[j])
        if kind == BG:
            return np.eye(3), ol.manifold_plus_jacobian(ol.M_BIAS, win.gyro_bias[j])
        if kind == BA:
            return np.eye(3), ol.manifold_plus_jacobian(ol.M_BIAS, win.accel_bias[j])
        if kind == GR:
            return np.eye(2), ol.manifold_plus_jacobian(ol.M_SPHERE, win.gravity)
        return np.eye(3), ol.manifold_plus_jacobian(ol.M_EUCLIDEAN, win.landmarks[j])

    worst_t = worst_a = 0.0
    for q, (ka, ja, kb, jb) in enumerate(pairs):
        ta, tb = runtime.COV_TANGENT[ka], runtime.COV_TANGENT[kb]
        D = blocks[q][:ta, :tb]
        Ta, Pa = conv(ka, ja)
        Tb, Pb = conv(kb, jb)
        want_t = Ta @ D @ Tb.T
        if ka == KN and kb == KN:
            assert np.allclose(cr.ceres_tangent(D), want_t, rtol=0, atol=0)
            want_a = cr.ambient(D, Pa) if ja == jb else Pa @ want_t @ Pb.T
        else:
            want_a = Pa @ want_t @ Pb.T
        scale = max(np.abs(want_t).max(), 1e-300)
        worst_t = max(worst_t, float(np.abs(tans[q].reshape(want_t.shape) - want_t).max() / scale))
        worst_a = max(worst_a, float(np.abs(ambs[q].reshape(want_a.shape) - want_a).max() / max(np.abs(want_a).max(), 1e-300)))
    record_property("tangent_err", worst_t)
    record_property("ambient_err", worst_a)
    # two computes of the same window (two processes) differ only by the assembly's floating-point atomics
    assert worst_t < 1e-8 and worst_a < 1e-8, (worst_t, worst_a)
