"""Deterministic assembly (hb200_set_deterministic) on an H100: reruns are bit-identical.

* every assembly switch of test_gpu_assembly.py: two contexts and a second build in one of them give the same packed
  buffer bit for bit (int64 views), the buffer is within tests/asmref.py's componentwise bound with exact zeros where it
  has zeros, and the deterministic kernels are the ones that ran;
* LM iterations with termination on (graph and direct launches) and hb200_optimize: identical records and state;
* the device-side sliding window (stereo tracks, pose and inertial appends, slides dropping bias knots) in two contexts
  without re-synchronising their states;
* covariance build + compute twice with an iteration undone by restore in between; the covariance end-to-end checks of
  test_gpu_covariance.py (covref's selected inverse of the device's undamped system and of asmref's long-double one,
  landmark marginals, interpolated covariances) on deterministic contexts;
* the sharded LM loop through the all-reduce hook, run twice; two GPUs through peer memory, run twice (skipped below two
  devices);
* with the switch off the kernels are those of the default path, also after switching it on and off again.
"""
import ctypes as C
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import asmref as ar
import oracle_lib as ol
from hyperslam_b200 import runtime, synthetic
import test_gpu_covariance as tcov
from test_gpu_covariance import e2e_window
from test_gpu_assembly import (ASSEMBLY_KERNELS, EVAL_THREADS, IMU_MMA_MIN, SCHUR_GROUP_MIN, num_sms, plan, read_system, schur_window, subset,
                               valid_span, with_imu)
from test_gpu_sharded import HostReducer, on_ranks, open_ranks
from test_gpu_stereo_window import frame_loop_setup

pytestmark = pytest.mark.gpu

DET_NAMES = {"factor_eval_kernel": "factor_eval_det_kernel", "pixel_eval_kernel": "pixel_eval_det_kernel",
             "inertial_hessian_kernel": "inertial_hessian_det_kernel", "inertial_hessian_mma_kernel": "inertial_hessian_mma_det_kernel",
             "manifold_hessian_kernel": "manifold_hessian_det_kernel", "schur_kernel": "schur_det_kernel",
             "schur_group_kernel": "schur_group_det_kernel"}
DET_KERNELS = set(DET_NAMES.values()) | {"det_index_kernel", "det_reduce_kernel"}


def det_kernels(p):
    """The kernels of a deterministic iteration: the J^T J kernels swapped for their deterministic variants; the factor
    kernels of the trial-cost evaluation (no J^T J) stay."""
    trial = {k for k in p["kernels"] if k in ("factor_eval_kernel", "pixel_eval_kernel")}
    return {DET_NAMES.get(k, k) for k in p["kernels"]} | trial | {"det_index_kernel", "det_reduce_kernel"}


def same_bits(a, b):
    return a.shape == b.shape and np.array_equal(np.ascontiguousarray(a).view(np.int64), np.ascontiguousarray(b).view(np.int64))


def det_context(win, radius=1e4, **kw):
    ctx = runtime.Context(0, **kw)
    ctx.set_deterministic(True)
    assert ctx.deterministic()
    ctx.load_window(win, radius=radius)
    return ctx


def built_system(ctx):
    ctx.evaluate()
    ctx.build_system()
    return read_system(ctx)


def run_det_case(win, radius, report, expect=None):
    p = plan(win, num_sms())
    a = det_context(win, radius)
    b = det_context(win, radius)
    try:
        buf_a = built_system(a)
        buf_a2 = built_system(a)
        buf_b = built_system(b)
        prob = ar.problem(a.outputs(), win, a.index_maps())
        beta = a.bandwidth()
        ran = {name for name, _ in a.profile_iteration(reps=1)} & (ASSEMBLY_KERNELS | DET_KERNELS)
    finally:
        a.close()
        b.close()
    assert same_bits(buf_a, buf_b), "two contexts differ"
    assert same_bits(buf_a, buf_a2), "two builds differ"
    res = ar.compare(buf_a, ar.assemble(prob, radius), beta)
    for key, v in res.items():
        report(key, v)
    report("kernels", ",".join(sorted(ran)))
    bad = {k: v for k, v in res.items() if k not in ("nonzero_outside", "finite") and not v <= 1.0}
    assert res["finite"] and res["nonzero_outside"] == 0 and not bad, res
    assert ran == det_kernels(p), (ran, det_kernels(p))
    if expect:
        assert expect <= {DET_NAMES.get(k, k) for k in ran} | ran, (expect, ran)
    return p


# ---- 1. every assembly switch --------------------------------------------------------------------------------------
@pytest.mark.parametrize("order", [4, 6])
@pytest.mark.parametrize("side", ["merged", "separate"])
def test_merged_and_separate(built, record_property, order, side):
    win = synthetic.make_window(order=order, num_knots=40, num_landmarks=300, num_imu=0, seed=synthetic.SEED_BASE + 700 + order)
    npb = -(-win.v_stamp.size // EVAL_THREADS)
    ni = EVAL_THREADS * (4 * num_sms() - npb) + (1 if side == "separate" else 0)
    lo, hi = valid_span(win)
    win = with_imu(win, lo + (np.arange(ni) + 0.5) * (hi - lo) / ni, seed=order)
    p = run_det_case(win, 1e4, record_property)
    assert p["merged"] == (side == "merged")


@pytest.mark.parametrize("order", [4, 6])
@pytest.mark.parametrize("tail", [1, 63])
def test_visual_tails_bearing_pose(built, record_property, order, tail):
    base = synthetic.make_window(order=order, num_knots=24, num_landmarks=120, num_imu=500, seed=synthetic.SEED_BASE + 710 + order)
    win = synthetic.add_bearing_and_pose_factors(base, num_bearing=150, num_pose=12, seed=synthetic.SEED_BASE + 720 + order)
    nv = win.v_stamp.size + win.b_stamp.size
    win = subset(win, keep_v=np.arange(win.v_stamp.size) >= (nv - tail) % 64)
    assert (win.v_stamp.size + win.b_stamp.size) % 64 == tail
    run_det_case(win, 1e4, record_property, expect={"manifold_hessian_det_kernel"})


@pytest.mark.parametrize("order", [4, 6])
@pytest.mark.parametrize("ni", [IMU_MMA_MIN - 1, IMU_MMA_MIN])
def test_inertial_switch(built, record_property, order, ni):
    win = synthetic.make_window(order=order, num_knots=30, num_landmarks=60, num_imu=0, bias_dt=1.0, seed=synthetic.SEED_BASE + 730 + order)
    for b in (win.gyro_bias, win.accel_bias, win.truth["gyro_bias"], win.truth["accel_bias"]):
        b[:, 3] -= 0.05
    lo, hi = valid_span(win)
    u = np.sort(np.random.default_rng(730 + order).random(IMU_MMA_MIN) ** 3)
    win = with_imu(win, lo + u[:ni] * (hi - lo) * (1 - 1e-9), seed=order)
    want = "inertial_hessian_det_kernel" if ni < IMU_MMA_MIN else "inertial_hessian_mma_det_kernel"
    run_det_case(win, 1e4, record_property, expect={want})


@pytest.mark.parametrize("radius", [1e4, 1e16])
@pytest.mark.parametrize("L", [SCHUR_GROUP_MIN - 1, SCHUR_GROUP_MIN])
def test_schur_single_observation(built, record_property, L, radius):
    win = schur_window(4, SCHUR_GROUP_MIN, single=512)
    if L < SCHUR_GROUP_MIN:
        win = subset(win, keep_v=win.v_lm < L)
        win.landmarks = np.ascontiguousarray(win.landmarks[:L])
    want = "schur_group_det_kernel" if L >= SCHUR_GROUP_MIN else "schur_det_kernel"
    run_det_case(win, radius, record_property, expect={want})


def test_schur_group_smem_fallback(built, record_property):
    win = schur_window(4, SCHUR_GROUP_MIN, single=64, extra_long=True, seed=1, num_knots=86)
    win = subset(win, keep_v=~np.isin(win.v_lm, np.arange(100, 140)))
    p = run_det_case(win, 1e16, record_property, expect={"schur_det_kernel"})
    assert p["group_smem"] > 200 * 1024


# ---- 2. LM iterations and termination ----------------------------------------------------------------------------
def lm_windows():
    return {"cfg1": synthetic.make_config(1, constant_knots=2),
            "order6": synthetic.make_window(order=6, num_knots=30, num_landmarks=400, num_imu=3000, constant_knots=2, seed=synthetic.SEED_BASE + 760)}


def lm_run(win, use_graph, iters=8):
    ctx = det_context(win, use_graph=use_graph)
    try:
        ctx.set_termination()
        rec = ctx.iterate(iters)
        term = ctx.termination()
        return rec, term, ctx.state()
    finally:
        ctx.close()


@pytest.mark.parametrize("use_graph", [True, False])
@pytest.mark.parametrize("name", ["cfg1", "order6"])
def test_lm_records_and_state(built, name, use_graph):
    win = lm_windows()[name]
    (ra, ta, sa), (rb, tb, sb) = lm_run(win, use_graph), lm_run(win, use_graph)
    assert ra == rb and ta == tb
    assert len(ra) >= 2
    for key in sa:
        assert same_bits(sa[key], sb[key]), key


def test_optimize_host_buffers(built):
    win = lm_windows()["cfg1"]
    outs = []
    for _ in range(2):
        ctx = det_context(win)
        try:
            s = ctx.state()
            blocks = [s[k].copy() for k in ("knots", "gyro_bias", "accel_bias", "gravity", "landmarks")]
            rec = ctx.optimize(4, *blocks)
            outs.append((rec, blocks))
        finally:
            ctx.close()
    assert outs[0][0] == outs[1][0]
    for a, b in zip(outs[0][1], outs[1][1]):
        assert same_bits(a, b)


# ---- 3. sliding window ------------------------------------------------------------------------------------------
def test_stereo_frame_loop(built):
    order, K0, width, frames = 4, 14, 9, 20
    full, hw, prev_hi, tracks = frame_loop_setup(order, K0, frames, synthetic.SEED_BASE + 4300 + order)
    ctxs = [runtime.Context(0), runtime.Context(0)]
    for ctx in ctxs:
        ctx.set_deterministic(True)
        ctx.load_window(hw.window())
    cams = full.cameras
    try:
        for frame in range(frames):
            hw.append_knot()
            for ctx in ctxs:
                ctx.append_knots(1)
            _, hi = hw.valid_range()
            knots = ctxs[0].state()["knots"]
            for s in np.unique(tracks["stamp"][(tracks["stamp"] >= prev_hi) & (tracks["stamp"] < hi)]):
                t = tracks["stamp"] == s
                gids, px0, px1 = tracks["gid"][t], tracks["px0"][t], tracks["px1"][t]
                n = gids.size
                pos = {g: p for p, g in enumerate(hw.lm_ids)}
                given = np.array([pos.get(g, -1) for g in gids.tolist()], dtype=np.int32)
                new = given < 0
                want = given.copy()
                want[new] = len(hw.lm_ids) + np.arange(int(new.sum()))
                stamp, c0, c1 = np.full(n, s), np.zeros(n, np.int32), np.ones(n, np.int32)
                for ctx in ctxs:
                    out, _ = ctx.append_stereo_tracks(stamp, c0, c1, px0, px1, given)
                    assert np.array_equal(out, want), frame
                base = int(hw.base_of(np.array([s]))[0])
                b0, b1, lm_w = ol.ingest_stereo_frame(knots[base:base + order], s, cams[0], cams[1], px0, px1)
                hw.add_landmarks(gids[new].tolist(), lm_w[new])
                bst, bcam = np.repeat(stamp, 2), np.stack([c0, c1], 1).ravel()
                hw.add_lists(b=dict(stamp=bst, cam=bcam, gid=np.repeat(gids, 2), bearing=np.stack([b0, b1], 1).reshape(-1, 3)))
            ii = (full.i_stamp >= prev_hi) & (full.i_stamp < hi)
            mi = np.flatnonzero((full.m_stamp >= prev_hi) & (full.m_stamp < hi))[:1] if frame % 3 == 0 else np.zeros(0, np.int64)
            prev_hi = hi
            for ctx in ctxs:
                ctx.append_inertial_factors(full.i_stamp[ii], full.i_meas[ii])
                ctx.append_manifold_factors(full.m_stamp[mi], full.m_sensor[mi], full.m_pose[mi])
            hw.add_lists(i=dict(stamp=full.i_stamp[ii], meas=full.i_meas[ii]), m=dict(stamp=full.m_stamp[mi], sensor=full.m_sensor[mi], pose=full.m_pose[mi]))
            lower = hw.knots[len(hw.knots) - 1 - width, 7] + 1e-9
            stats = [ctx.slide(lower, drop_inertial=True, drop_manifold=True, drop_bias=True) for ctx in ctxs]
            assert stats[0] == stats[1], frame
            hw.slide(lower, drop_inertial=True, drop_manifold=True)
            recs = [ctx.iterate(2) for ctx in ctxs]
            assert recs[0] == recs[1], frame
            sa, sb = ctxs[0].state(), ctxs[1].state()
            for key in sa:
                assert same_bits(sa[key], sb[key]), (frame, key)
            hw.knots, hw.lm_xyz = sa["knots"].copy(), sa["landmarks"].copy()
    finally:
        for ctx in ctxs:
            ctx.close()


# ---- 4. covariance --------------------------------------------------------------------------------------------------
def covariance_outputs(ctx, stamps):
    ctx.build_covariance()
    info = ctx.compute_covariance()
    assert info["rc"] == 0, info
    packed, lm, _ = ctx.covariance_packed()
    cov, bad = ctx.interpolate_covariance(stamps)
    assert bad == 0
    return [packed, lm, cov]


def test_covariance_rebuild(built):
    win = e2e_window(4)
    lo, hi = valid_span(win)
    stamps = np.linspace(lo, hi, 17)[:-1]
    results = []
    for _ in range(2):
        ctx = det_context(win)
        try:
            ctx.iterate(3)
            first = covariance_outputs(ctx, stamps)
            ctx.snapshot()
            ctx.iterate(1)
            ctx.restore()
            second = covariance_outputs(ctx, stamps)
        finally:
            ctx.close()
        for a, b in zip(first, second):
            assert same_bits(a, b)
        results.append(first)
    for a, b in zip(*results):
        assert same_bits(a, b)


class _DetContext(runtime.Context):
    def __init__(self, *args, **kw):
        super().__init__(*args, **kw)
        self.set_deterministic(True)


@pytest.fixture
def det_contexts(monkeypatch):
    """Every context test_gpu_covariance.py's checks open assembles deterministically."""
    monkeypatch.setattr(tcov.runtime, "Context", _DetContext)


@pytest.mark.parametrize("order", [4, 6])
def test_covariance_covref(built, record_property, det_contexts, order):
    """The undamped deterministic build (mu = 0 in the Schur variants) against covref and asmref, and the interpolated
    covariance within covref's tolerance: the checks of test_e2e_cfg1_shaped on deterministic contexts."""
    res = tcov.check_e2e(e2e_window(order, seed=order), record_property)
    assert {"schur_det_kernel", "det_reduce_kernel"} <= res["kernels"] and "schur_kernel" not in res["kernels"], res["kernels"]
    tcov.test_e2e_cfg1_shaped(built, record_property, order)


def test_covariance_covref_group_path(built, record_property, det_contexts):
    """K = 500 with 8192 landmarks: the undamped build through schur_group_det_kernel, against covref."""
    win = e2e_window(4, num_knots=500, num_landmarks=8192, num_imu=4000, bearing=0, pose=40, seed=21, frames=3)
    res = tcov.check_e2e(win, record_property, asm=False)
    assert "schur_group_det_kernel" in res["kernels"] and "schur_group_kernel" not in res["kernels"], res["kernels"]


# ---- 5. sharded -------------------------------------------------------------------------------------------------------
def sharded_run(win, world, iters=4):
    shards = [win.shard(r, world) for r in range(world)]
    ctxs, _, _ = open_ranks(shards)
    try:
        for c in ctxs:
            c.set_deterministic(True)
        reducer = HostReducer(world)
        reducer.attach(ctxs)
        recs = on_ranks(reducer, ctxs, lambda r, c: c.iterate(iters))
        return recs, [c.state() for c in ctxs]
    finally:
        for c in ctxs:
            c.close()


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_hook_repeat(built, world):
    win = synthetic.make_config(1, scale=0.25, num_knots=51, constant_knots=2)
    (ra, sa), (rb, sb) = sharded_run(win, world), sharded_run(win, world)
    assert ra == rb
    for a, b in zip(sa, sb):
        for key in a:
            assert same_bits(a[key], b[key]), key
    for s in sa[1:]:   # replicated blocks agree across the ranks
        for key in ("knots", "gyro_bias", "accel_bias", "gravity"):
            assert same_bits(s[key], sa[0][key]), key


def test_two_gpu_peer_memory_repeat(built):
    """Two ranks on two GPUs, partial systems summed through peer memory in rank order: two runs give the same records
    and the same state bit for bit on every rank, and the replicated knots agree across the ranks."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    runs = []
    for _ in range(2):
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
               "--master-port", "29547", os.path.join(root, "tests", "det_multi_gpu_worker.py")]
        res = subprocess.run(cmd, capture_output=True, text=True, timeout=150)
        assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]
        out = json.loads([line for line in res.stdout.splitlines() if line.startswith("{")][-1])
        assert out["deterministic"] and out["comm"]["peer_reduce"] and out["comm"]["graph"], out["comm"]
        runs.append(out)
    assert runs[0]["records"] == runs[1]["records"]
    assert runs[0]["states"] == runs[1]["states"]


# ---- 6. default path untouched -------------------------------------------------------------------------------------
def test_switch_off_restores_default_kernels(built):
    win = synthetic.make_config(1, constant_knots=2)
    p = plan(win, num_sms())
    ctx = runtime.Context(0)
    try:
        ctx.load_window(win)
        names = lambda: {n for n, _ in ctx.profile_iteration(reps=1)} & (ASSEMBLY_KERNELS | DET_KERNELS)
        assert not ctx.deterministic()
        assert names() == p["kernels"]
        ctx.set_deterministic(True)
        assert names() == det_kernels(p)
        ctx.set_deterministic(False)
        assert names() == p["kernels"]
    finally:
        ctx.close()


def test_switch_return_codes(built):
    """A change drops a built system and a pending covariance build; setting the current value changes nothing."""
    win = synthetic.make_window(order=4, num_knots=16, num_landmarks=60, num_imu=200, seed=synthetic.SEED_BASE + 780)
    ctx = runtime.Context(0)
    lib, h = ctx.lib, ctx.h
    try:
        assert lib.hb200_set_deterministic(h, 1) == 0   # before hb200_bind
        ctx.load_window(win)
        ctx.evaluate()
        ctx.build_system()
        assert lib.hb200_set_deterministic(h, 1) == 0   # unchanged: the built system stays
        assert lib.hb200_solve(h) == 0
        assert lib.hb200_set_deterministic(h, 0) == 0
        assert lib.hb200_solve(h) == -2
        assert lib.hb200_get_system(h, None, None) == -2
        # (a compute that runs reports the window's own status: not positive definite or degenerate landmarks count as run)
        compute = lambda: lib.hb200_compute_covariance(h, C.byref(runtime.CovarianceInfo()))
        ran = (0, runtime.COV_NOT_POSITIVE_DEFINITE, runtime.COV_DEGENERATE_LANDMARKS)
        ctx.build_covariance()
        assert lib.hb200_set_deterministic(h, 1) == 0
        assert compute() == -2
        ctx.build_covariance()
        assert lib.hb200_set_deterministic(h, 1) == 0
        assert compute() in ran
        assert lib.hb200_get_deterministic(h, None) == -1
    finally:
        ctx.close()

