"""The sharded LM iteration on one GPU (need an H100): N contexts on device 0, each holding a factor shard of the same
window, reduce their partial systems through the all-reduce callback (hb200_set_allreduce) with a reducer written here.

This reaches what only a sharded solve runs and a one-GPU run of the rest of the suite does not: partial systems built
from a landmark-owner shard, a band layout widened past the shard's own longest track (hb200_set_min_bandwidth),
scalars_kernel, accept_kernel without the fused scalars, and the reduction points of enqueue_reduce_system /
enqueue_reduce_scalars.  (The NCCL and peer-memory reductions need two GPUs: tests/test_gpu_multi.py.)

Per case:
* partial systems (contexts without the hook, all at the agreed half-width): every shard's raw packed buffer against
  tests/asmref.py within its componentwise bound, exact zeros outside the shard's own tracks included, and the rank-order
  float64 sum of the buffers against the long-double sum of the shard references;
* iterations through the hook: records and replicated state bit-identical across ranks; every landmark, read from its
  owner, against one context on the whole window and against the CPU oracle; landmarks a rank does not own unchanged;
* which kernels ran (profile_iteration names) against sysref.solver_plan and the switch the case targets.
Termination through the hook: function and parameter tolerance as on one context, a gradient tolerance refused, and the
reported gradient maximum norm restricted to the replicated blocks.
"""
import threading

import numpy as np
import pytest

import asmref as ar
import oracle_lib as ol
import sysref as sr
from hyperslam_b200 import runtime, synthetic
from test_gpu_assembly import SCHUR_GROUP_MIN, num_sms, read_system
from test_shardref import by_index

pytestmark = pytest.mark.gpu

RADIUS = 1e4
ITERS = 4
BARRIER_TIMEOUT = 60.0      # seconds a rank waits in the reducer for the others
SOLVER_KERNELS = {"band_solve_kernel", "band_solve_kernel<false>", "bcr_solve_kernel", "cholesky_kernel"}
HOOK_MARKS = {"allreduce_callback(system)", "scalars_kernel", "allreduce_callback(scalars)", "accept_kernel"}
# the tolerances of tests/test_gpu_multi.py's worker
COST_TOL, COST_NEW_TOL, STATE_TOL = 1e-7, 1e-6, 1e-6


def shard_by_owner(win, owner, world, i_cuts=None, compact=False):
    """Shards of `win` under an explicit landmark -> rank map: visual factors follow their landmark's owner, inertial and
    pose factors are split into contiguous index ranges (i_cuts: the world + 1 boundaries of the inertial ranges, default
    even).  compact: a shard holds only the landmarks its rank owns, re-indexed, instead of all of them.
    Returns (shards, index) with index[r] the window landmark of each landmark of shard r."""
    owner = np.asarray(owner)
    ranks = dict(pixel=owner[win.v_lm], bearing=owner[win.b_lm], pose=by_index(win.m_stamp.size, world),
                 inertial=by_index(win.i_stamp.size, world) if i_cuts is None else
                 np.searchsorted(i_cuts, np.arange(win.i_stamp.size), side="right") - 1)
    shards = ar.partition(win, ranks, world)
    L = win.landmarks.shape[0]
    index = [np.arange(L) for _ in range(world)]
    if compact:
        for r, s in enumerate(shards):
            index[r] = np.nonzero(owner == r)[0]
            local = np.full(L, -1, np.int32)
            local[index[r]] = np.arange(index[r].size)
            s.landmarks = np.ascontiguousarray(win.landmarks[index[r]])
            s.v_lm, s.b_lm = np.ascontiguousarray(local[s.v_lm]), np.ascontiguousarray(local[s.b_lm])
    return shards, index


class HostReducer:
    """The all-reduce behind every rank's hook, in this process.  Rank r's buffer is wrapped as a float64 tensor; each rank
    records an event on its own stream and meets the others at a barrier; rank 0 then sums the buffers in rank order on a
    private stream that has waited for every rank's event and copies the sum into every buffer; every rank's stream waits
    for the event recorded after those copies.  A failing rank aborts the barrier, so the others raise instead of waiting."""

    def __init__(self, n):
        import torch
        self.torch, self.n = torch, n
        self.dev = torch.device("cuda", 0)
        self.barrier = threading.Barrier(n, timeout=BARRIER_TIMEOUT)
        self.private = torch.cuda.Stream(self.dev)
        self.ready = [torch.cuda.Event() for _ in range(n)]
        self.done = torch.cuda.Event()
        self.bufs = [None] * n
        self.tensors = {}
        self.error = None

    def _wrap(self, ptr, count):
        if (ptr, count) not in self.tensors:
            class _Arr:
                __cuda_array_interface__ = dict(shape=(count,), typestr="<f8", data=(ptr, False), version=2)
            self.tensors[(ptr, count)] = self.torch.as_tensor(_Arr(), device=self.dev)
        return self.tensors[(ptr, count)]

    def hook(self, rank, stream):
        torch = self.torch
        ext = torch.cuda.ExternalStream(stream, device=self.dev)

        def allreduce(ptr, count, _stream):
            try:
                self.bufs[rank] = self._wrap(ptr, count)
                self.ready[rank].record(ext)
                self.barrier.wait()
                if rank == 0:
                    sizes = {b.numel() for b in self.bufs}
                    if len(sizes) != 1:
                        raise RuntimeError(f"the ranks reduce buffers of different sizes {sizes}")
                    with torch.cuda.stream(self.private):
                        for e in self.ready:
                            self.private.wait_event(e)
                        total = self.bufs[0].clone()
                        for b in self.bufs[1:]:
                            total += b
                        for b in self.bufs:
                            b.copy_(total)
                        self.done.record(self.private)
                self.barrier.wait()
                ext.wait_event(self.done)
                return 0
            except Exception as e:   # reported through the library's error code; the others must not wait
                self.error = self.error or e
                self.barrier.abort()
                return 1
        return allreduce

    def attach(self, ctxs):
        for r, c in enumerate(ctxs):
            c.set_allreduce(self.hook(r, c.stream))


def on_ranks(reducer, ctxs, fn):
    """fn(rank, ctx) for every rank, each in its own thread (ctypes releases the GIL around the library calls)."""
    out, err = [None] * len(ctxs), [None] * len(ctxs)

    def work(r):
        try:
            out[r] = fn(r, ctxs[r])
        except BaseException as e:
            err[r] = e
            reducer.barrier.abort()
    threads = [threading.Thread(target=work, args=(r,)) for r in range(len(ctxs))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    if any(e is not None for e in err):
        raise AssertionError(f"rank errors {err!r}; reducer {reducer.error!r}")
    return out


def open_ranks(shards, force_dense=False):
    """One context per shard (no CUDA graph, as with any callback hook), all at the largest half-width of any shard.
    Returns (contexts, each shard's own half-width, the agreed one)."""
    ctxs = []
    for s in shards:
        ctxs.append(runtime.Context(0, use_graph=False, force_dense=force_dense))
        ctxs[-1].load_window(s, radius=RADIUS)
    own = [c.bandwidth() for c in ctxs]
    for c in ctxs:
        c.set_min_bandwidth(max(own))
    assert all(c.bandwidth() == max(own) for c in ctxs)
    return ctxs, own, max(own)


def worst(res):
    return max(v for k, v in res.items() if k not in ("nonzero_outside", "finite"))


def check_record(rec, ref):
    assert abs(rec["cost"] - ref["cost"]) <= COST_TOL * ref["cost"], (rec, ref["cost"])
    assert abs(rec["cost_new"] - ref["cost_new"]) <= COST_NEW_TOL * abs(ref["cost_new"]), (rec, ref["cost_new"])
    assert rec["accepted"] == ref["accepted"] and rec["spd"] == 1, (rec, ref["accepted"])


def run_case(win, shards, index, owner, report, force_dense=False):
    """Partial systems, ITERS iterations through the hook and the kernel plan of one partition.  Returns what the case
    asserts on: each rank's own and the agreed half-width, the solver plan and the kernel names of every rank and of a
    single context on the whole window."""
    N, owner = len(shards), np.asarray(owner)
    K, m = win.knots.shape[0], 3 * (win.gyro_bias.shape[0] + win.accel_bias.shape[0]) + 2
    ctxs, own, beta = open_ranks(shards, force_dense)
    try:
        bufs, refs = [], []
        for r, (c, s) in enumerate(zip(ctxs, shards)):
            c.evaluate()
            c.build_system()
            bufs.append(read_system(c))
            refs.append(ar.assemble(ar.problem(c.outputs(), s, c.index_maps()), RADIUS))
            report(f"rank{r}_ratio", worst(ar.check(bufs[-1], refs[-1], beta)))
        res = ar.compare_summed_buffers(bufs, refs, beta)
        report("partial_sum_ratio", worst(res))
        assert res["finite"] and res["nonzero_outside"] == 0 and worst(res) <= 1.0, res
        sum_cost_bound = sum(r["cost_bound"] for r in refs) + (N - 1) * ar.U * sum(abs(float(r["cost"])) for r in refs)

        red = HostReducer(N)
        red.attach(ctxs)
        recs = on_ranks(red, ctxs, lambda r, c: c.iterate(ITERS))
        states = [c.state() for c in ctxs]
        names = on_ranks(red, ctxs, lambda r, c: {n for n, _ in c.profile_iteration(reps=1)})
    finally:
        for c in ctxs:
            c.close()

    single = runtime.Context(0, force_dense=force_dense)
    try:
        single.load_window(win, radius=RADIUS)
        single.evaluate()
        full = ar.assemble(ar.problem(single.outputs(), win, single.index_maps()), RADIUS)
        srecs = single.iterate(ITERS)
        sstate = single.state()
        snames = {n for n, _ in single.profile_iteration(reps=1)}
    finally:
        single.close()
    ow = ol.OracleWindow(win, radius=RADIUS)
    orecs = [ow.iterate(apply=True, outputs=False)["stats"] for _ in range(ITERS)]
    orecs = [dict(cost=s[0], cost_new=s[1], accepted=int(s[5])) for s in orecs]
    ostate = ow.state()

    keys = ("cost", "cost_new", "rho", "radius", "accepted", "spd")
    for r in range(1, N):
        assert [[x[k] for k in keys] for x in recs[r]] == [[x[k] for k in keys] for x in recs[0]], r
        for key in ("knots", "gyro_bias", "accel_bias", "gravity"):
            assert np.array_equal(states[r][key], states[0][key]), (r, key)
    for it in range(ITERS):
        check_record(recs[0][it], srecs[it])
        check_record(recs[0][it], orecs[it])
    cost_err = abs(recs[0][0]["cost"] - srecs[0]["cost"])
    report("cost_ratio", cost_err / (sum_cost_bound + float(full["cost_bound"])))
    assert cost_err <= sum_cost_bound + float(full["cost_bound"]), (recs[0][0]["cost"], srecs[0]["cost"])
    lms = np.full_like(win.landmarks, np.nan)
    for r in range(N):
        mine = owner[index[r]] == r
        lms[index[r][mine]] = states[r]["landmarks"][mine]
        assert np.array_equal(states[r]["landmarks"][~mine], shards[r].landmarks[~mine]), r
    for ref in (sstate, ostate):
        for key in ("knots", "gyro_bias", "accel_bias", "gravity"):
            assert np.abs(states[0][key] - ref[key]).max() <= STATE_TOL, key
        assert np.abs(lms - ref["landmarks"]).max() <= STATE_TOL
    report("landmark_max_diff_single", float(np.abs(lms - sstate["landmarks"]).max()))

    plan = sr.solver_plan(K, beta, m, num_sms(), force_dense)
    for r in range(N):
        assert HOOK_MARKS <= names[r], (r, names[r])
        assert names[r] & SOLVER_KERNELS == {plan["kernel"]}, (r, names[r] & SOLVER_KERNELS, plan)
    assert not (HOOK_MARKS - {"accept_kernel"}) & snames, snames      # one context: scalars fused into accept_kernel
    report("solver", plan["kernel"])
    report("own_beta", ",".join(map(str, own)))
    return dict(own_beta=own, beta=beta, plan=plan, names=names, single_names=snames)


# ---- cases -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [2, 3, 8])
def test_default_partition(built, record_property, world):
    """cfg1-shaped (order 4, stereo pixel + IMU factors) under Window.shard; the inertial ranges are cut inside runs of
    factors that share their knot and bias bases (51 knots: with 50 the middle of the window falls on a knot)."""
    win = synthetic.make_config(1, scale=0.25, num_knots=51, constant_knots=2)
    L, Ni = win.landmarks.shape[0], win.i_stamp.size
    bases = np.stack([synthetic.segment(win.knots[:, 7], win.order, win.i_stamp)[0],
                      synthetic.segment(win.gyro_bias[:, 3], win.bias_order, win.i_stamp)[0],
                      synthetic.segment(win.accel_bias[:, 3], win.bias_order, win.i_stamp)[0]], 1)
    cuts = [(Ni * r) // world for r in range(1, world)]
    assert all((bases[c - 1] == bases[c]).all() for c in cuts), cuts
    shards = [win.shard(r, world) for r in range(world)]
    out = run_case(win, shards, [np.arange(L)] * world, by_index(L, world), record_property)
    assert all("inertial_hessian_kernel" in n and "schur_kernel" in n for n in out["names"])


def test_bearing_and_pose_factors(built, record_property):
    """Order 6 with bearing and pose factors, landmark owners drawn at random over three ranks; every rank gets pixel,
    bearing, inertial and pose factors."""
    base = synthetic.make_window(order=6, num_knots=30, num_landmarks=150, num_imu=400, seed=synthetic.SEED_BASE + 900, constant_knots=2)
    win = synthetic.add_bearing_and_pose_factors(base, num_bearing=120, num_pose=12, seed=synthetic.SEED_BASE + 901)
    owner = np.random.default_rng(900).integers(0, 3, win.landmarks.shape[0])
    shards, index = shard_by_owner(win, owner, 3)
    assert all(s.v_stamp.size and s.b_stamp.size and s.i_stamp.size and s.m_stamp.size == 4 for s in shards)
    out = run_case(win, shards, index, owner, record_property)
    assert all("manifold_hessian_kernel" in n for n in out["names"])


def test_shards_with_empty_families(built, record_property):
    """Six ranks, five landmarks: rank 5 owns no landmark (no visual factor), rank 0 gets no inertial factor."""
    win = synthetic.make_window(order=4, num_knots=16, num_landmarks=5, num_imu=300, seed=synthetic.SEED_BASE + 910, constant_knots=2)
    Ni = win.i_stamp.size
    owner = np.arange(5)
    shards, index = shard_by_owner(win, owner, 6, i_cuts=[0] + [(Ni * r) // 5 for r in range(6)])
    assert shards[0].i_stamp.size == 0 and shards[0].v_stamp.size and shards[5].v_stamp.size == 0 and shards[5].i_stamp.size
    out = run_case(win, shards, index, owner, record_property)
    assert not {"inertial_hessian_kernel", "inertial_hessian_mma_kernel"} & out["names"][0]
    assert not {"schur_kernel", "schur_group_kernel"} & out["names"][5]


def long_track_window(num_tracks=4, span_knots=8):
    """A window with `num_tracks` extra landmarks, each seen by both cameras of the stereo pair at 2 span_knots + 1 stamps
    over span_knots knot intervals (the other landmarks span two or three)."""
    win = synthetic.make_window(order=4, num_knots=40, num_landmarks=200, num_imu=400, seed=synthetic.SEED_BASE + 920, constant_knots=2)
    dt = win.knots[1, 7] - win.knots[0, 7]
    st, cam, idx, lms = [win.v_stamp], [win.v_cam], [win.v_lm], [win.landmarks]
    L = win.landmarks.shape[0]
    for j in range(num_tracks):
        t = win.knots[4 + 8 * j, 7] + 0.3 * dt + np.linspace(0, span_knots * dt, 2 * span_knots + 1)
        R, p, *_ = synthetic.spline_eval(win.knots, win.order, t[span_knots:span_knots + 1])
        lms.append(p[0] + R[0] @ np.array([0.2 * j, 0.0, 5.0]))
        st += [t, t]
        cam += [np.zeros(t.size, np.int32), np.ones(t.size, np.int32)]
        idx += [np.full(2 * t.size, L + j, np.int32)]
    win.landmarks = np.ascontiguousarray(np.vstack([lms[0], np.stack(lms[1:])]))
    st, cam, idx = np.concatenate(st), np.concatenate(cam), np.concatenate(idx)
    px, p_s = synthetic.pixel_model(win.knots, win.order, win.cameras, win.landmarks, st, cam, idx)
    new = idx >= L
    assert (p_s[new, 2] > 0.5).all() and (px[new] > 0).all() and (px[new, 0] < synthetic.IMAGE_SIZE[0]).all() and (px[new, 1] < synthetic.IMAGE_SIZE[1]).all()
    px[new] += np.random.default_rng(920).normal(0, 0.5, px[new].shape)
    px[~new] = np.concatenate([win.v_pixel])
    o = np.argsort(st, kind="stable")
    win.v_stamp, win.v_cam, win.v_lm, win.v_pixel = (np.ascontiguousarray(a[o]) for a in (st, cam, idx, px))
    return win, L


def test_long_tracks_on_one_rank(built, record_property):
    """Rank 0 owns the long tracks: rank 1's own half-width is smaller, and set_min_bandwidth widens its packed layout."""
    win, L0 = long_track_window()
    owner = (np.arange(win.landmarks.shape[0]) < L0).astype(int)   # long tracks (index >= L0) -> rank 0
    shards, index = shard_by_owner(win, owner, 2)
    out = run_case(win, shards, index, owner, record_property)
    assert out["own_beta"][1] < out["own_beta"][0] == out["beta"], out["own_beta"]


def test_schur_kernels_differ_between_ranks(built, record_property):
    """12000 landmarks seen once by the stereo pair; each rank holds only the landmarks it owns: 9000 on rank 0
    (schur_group_kernel, >= 8192), 3000 on rank 1 (schur_kernel).  One context on the whole window takes the group kernel."""
    win = synthetic.make_window(order=4, num_knots=120, num_landmarks=12000, frames_per_landmark=1, num_imu=300, seed=synthetic.SEED_BASE + 930,
                                constant_knots=2)
    owner = (np.arange(12000) >= 9000).astype(int)
    shards, index = shard_by_owner(win, owner, 2, compact=True)
    assert shards[0].landmarks.shape[0] >= SCHUR_GROUP_MIN > shards[1].landmarks.shape[0]
    out = run_case(win, shards, index, owner, record_property)
    assert "schur_group_kernel" in out["names"][0] and "schur_kernel" not in out["names"][0]
    assert "schur_kernel" in out["names"][1] and "schur_group_kernel" not in out["names"][1]
    assert "schur_group_kernel" in out["single_names"]


@pytest.mark.parametrize("path", ["bcr", "dense"])
def test_other_solver_paths(built, record_property, path):
    """Two ranks on a 140-knot window (block cyclic reduction), and on a 30-knot window with the dense solver forced."""
    if path == "bcr":
        win = synthetic.make_window(order=4, num_knots=140, num_landmarks=300, num_imu=600, seed=synthetic.SEED_BASE + 940, constant_knots=2)
    else:
        win = synthetic.make_window(order=4, num_knots=30, num_landmarks=200, num_imu=400, seed=synthetic.SEED_BASE + 941, constant_knots=2)
    L = win.landmarks.shape[0]
    shards = [win.shard(r, 2) for r in range(2)]
    out = run_case(win, shards, [np.arange(L)] * 2, by_index(L, 2), record_property, force_dense=(path == "dense"))
    assert out["plan"]["path"] == path, out["plan"]


# ---- termination through the hook ------------------------------------------------------------------------------------
def termination_window():
    """The window tests/test_gpu_termination.py ends by each tolerance (order 4)."""
    return synthetic.make_window(order=4, num_knots=18, num_landmarks=120, num_imu=300, seed=synthetic.SEED_BASE + 3004, constant_knots=2)


TOLERANCES = {"function": (dict(function_tolerance=1e-3, parameter_tolerance=0.0), 1),
              "parameter": (dict(function_tolerance=0.0, parameter_tolerance=3e-2), 2)}


@pytest.mark.parametrize("name", list(TOLERANCES))
def test_termination_matches_one_context(built, name):
    tol, want = TOLERANCES[name]
    tol = dict(tol, gradient_tolerance=0.0, min_trust_region_radius=1e-32)
    win = termination_window()
    max_iter = 40
    single = runtime.Context(0)
    single.load_window(win, radius=RADIUS)
    single.set_termination(**tol)
    srecs = single.iterate(max_iter)
    ts = single.termination()
    single.close()
    assert ts["type"] == want and 0 < ts["iterations"] < max_iter, ts
    ctxs, _, _ = open_ranks([win.shard(r, 3) for r in range(3)])
    try:
        red = HostReducer(3)
        red.attach(ctxs)
        for c in ctxs:
            c.set_termination(**tol)
        recs = on_ranks(red, ctxs, lambda r, c: c.iterate(max_iter))
        terms = [c.termination() for c in ctxs]
    finally:
        for c in ctxs:
            c.close()
    for r in range(3):
        assert (terms[r]["type"], terms[r]["iterations"]) == (ts["type"], ts["iterations"]), (r, terms[r], ts)
        assert recs[r] == recs[0]
    for i in range(ts["iterations"]):
        check_record(recs[0][i], srecs[i])


def test_gradient_tolerance_is_refused_through_the_hook(built):
    """Whether the tolerance is set before or after the hook is attached, hb200_iterate and hb200_optimize refuse it;
    switched off, the same contexts iterate."""
    win = termination_window()
    ctxs, _, _ = open_ranks([win.shard(r, 2) for r in range(2)])
    try:
        ctxs[0].set_termination(gradient_tolerance=1e-10)
        red = HostReducer(2)
        red.attach(ctxs)
        ctxs[1].set_termination(gradient_tolerance=1e-10)
        for c in ctxs:
            with pytest.raises(runtime.HB200Error, match="gradient tolerance"):
                c.iterate(1)
            st = c.state()
            with pytest.raises(runtime.HB200Error, match="gradient tolerance"):
                c.optimize(1, st["knots"], st["gyro_bias"], st["accel_bias"], st["gravity"], st["landmarks"])
            c.set_termination(0.0, 0.0, 0.0, 0.0)
        recs = on_ranks(red, ctxs, lambda r, c: c.iterate(2))
        assert recs[0] == recs[1] and all(x["cost"] > 0 for x in recs[0])
    finally:
        for c in ctxs:
            c.close()


def quat_exp(th):
    t2 = float(th @ th)
    t = np.sqrt(t2)
    s, c = (0.5 - t2 / 48.0, 1.0 - t2 / 8.0) if t < 1e-7 else (np.sin(0.5 * t) / t, np.cos(0.5 * t))
    return np.array([s * th[0], s * th[1], s * th[2], c])


def quat_mul(a, b):
    return np.array([a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1], a[3] * b[1] - a[0] * b[2] + a[1] * b[3] + a[2] * b[0],
                     a[3] * b[2] + a[0] * b[1] - a[1] * b[0] + a[2] * b[3], a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2]])


def sphere_plus(x, d):
    nd = np.hypot(d[0], d[1])
    if nd == 0.0:
        return x.copy()
    sigma = x[0] * x[0] + x[1] * x[1]
    v, beta = np.array([x[0], x[1], 1.0]), 0.0
    if sigma <= 2.220446049250313e-16:
        beta = 2.0 if x[2] < 0.0 else 0.0
    else:
        mu = np.sqrt(x[2] * x[2] + sigma)
        vp = x[2] - mu if x[2] <= 0.0 else -sigma / (x[2] + mu)
        beta = 2.0 * vp * vp / (sigma + vp * vp)
        v[:2] /= vp
    y = np.array([np.sin(nd) / nd * d[0], np.sin(nd) / nd * d[1], np.cos(nd)])
    return np.sqrt(sigma + x[2] * x[2]) * (y - v * beta * (v @ y))


def replicated_gradient_max(g, win):
    """|x - Plus(x, -g)|_inf over the non-constant knots, bias knots and gravity (accept_kernel's v[10]): a knot's rotation
    moves by -4 g_theta (Ceres' local rotation coordinate is half of this library's), its position, the biases and the
    gravity tangent by -g."""
    K, Kbg, Kba = win.knots.shape[0], win.gyro_bias.shape[0], win.accel_bias.shape[0]
    fixed = sr.fixed_mask(K, Kbg, Kba, win.knot_const, win.bias_const, win.gravity_const)
    v = 0.0
    for j in range(K):
        if not fixed[6 * j]:
            q = win.knots[j, :4]
            v = max(v, np.abs(quat_mul(quat_exp(-4.0 * g[6 * j:6 * j + 3]), q) - q).max(), np.abs(g[6 * j + 3:6 * j + 6]).max())
    for o in range(6 * K, 6 * K + 3 * (Kbg + Kba), 3):
        if not fixed[o]:
            v = max(v, np.abs(g[o:o + 3]).max())
    o = 6 * K + 3 * (Kbg + Kba)
    if not fixed[o]:
        v = max(v, np.abs(sphere_plus(win.gravity, -g[o:o + 2]) - win.gravity).max())
    return v


def gradient_window():
    """Every knot constant, landmarks 0.3 m further off: the landmark gradient (about 1e3 on each of three ranks) dominates
    the biases' and gravity's (about 0.1)."""
    win = synthetic.make_window(order=4, num_knots=18, num_landmarks=120, num_imu=300, seed=synthetic.SEED_BASE + 950, constant_knots=18)
    win.landmarks = np.ascontiguousarray(win.landmarks + np.random.default_rng(950).normal(0, 0.3, win.landmarks.shape))
    return win


def test_gradient_norm_through_the_hook(built, record_property):
    """With the termination tests on (gradient tolerance 0), gradient_max_norm through the hook is the replicated-block part
    of one context's value: the reduced g restated in numpy, and no more than one context reports.  (A sum of the ranks'
    landmark maxima would exceed it here.)"""
    win = gradient_window()
    tol = dict(function_tolerance=0.0, gradient_tolerance=0.0, parameter_tolerance=0.0, min_trust_region_radius=1e-32)
    single = runtime.Context(0)
    single.load_window(win, radius=RADIUS)
    single.set_termination(**tol)
    single.iterate(1)
    g_single = single.termination()["gradient_max_norm"]
    single.close()
    world = 3
    ctxs, _, beta = open_ranks([win.shard(r, world) for r in range(world)])
    try:
        red = HostReducer(world)
        red.attach(ctxs)
        for c in ctxs:
            c.set_termination(**tol)
        on_ranks(red, ctxs, lambda r, c: c.iterate(1))
        g_hook = [c.termination()["gradient_max_norm"] for c in ctxs]
        buf = read_system(ctxs[0])   # the reduced system of that iteration
    finally:
        for c in ctxs:
            c.close()
    Lay = sr.layout(win.knots.shape[0], beta, 3 * (win.gyro_bias.shape[0] + win.accel_bias.shape[0]) + 2)
    restated = replicated_gradient_max(buf[Lay["og"]:Lay["og"] + Lay["n"]], win)
    record_property("gradient_max_norm_hook", g_hook[0])
    record_property("gradient_max_norm_single", g_single)
    record_property("gradient_max_norm_restated", restated)
    assert g_single > 2.0 * restated, (g_single, restated)   # the landmark part dominates
    assert all(g == g_hook[0] for g in g_hook), g_hook
    assert g_hook[0] <= g_single, (g_hook[0], g_single)
    # (the quaternion difference of a rotation entry is formed from unit-size values: a few ulps of 1 on top)
    assert abs(g_hook[0] - restated) <= 1e-12 * restated + 8 * sr.EPS, (g_hook[0], restated)
