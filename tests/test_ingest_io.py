"""Ingest (pixels -> bearings, stereo triangulation) and trajectory output around the hot path
(SURVEY.md section 8f rank 4; reference abstract.cpp:186-264, main.cpp:56-83, evaluation/conversions.py).

The k*_stereo_ingest known answers (tests/golden/ingest/, 80 digits: bearings from mp.findroot on the distortion, the
midpoint p_0 and the world landmark from the stored double inputs) hold every output to |got - ref| <= C u scale,
u = 2^-53, C = 150 (the bound of test_gpu_spline_edges.py):
  * bearing: scale 1.  Ten Newton steps on the 2 x 2 distortion system, then a normalisation: a few ulps of a unit vector;
  * landmark: scale max(|lm|, |p_0|^2 / |t_01|).  The rays s b_0 and t_01 + u d_1 meet at a parallax angle of about
    |t_01| / |p_0|, so tilting either bearing by u (its rounding) slides the midpoint along the ray by about
    |p_0| u / (|t_01| / |p_0|) = |p_0|^2 / |t_01| u; moving p_0 into the world frame rounds at the size of |lm|.
    The Gram form of the midpoint (det = a c - b^2 = sin^2 of the parallax, and its numerators) loses another factor
    of about |p_0| / |t_01| to cancellation: worst ratios of 250 - 500 at 2 m, 1600 - 2200 at 10 m and 9e3 - 2.5e4 at
    100 m on these fixtures (device and oracle), against below 5 at every depth for the cross-product form.
Parallel rays (cameras 4 and 5: identity rotations, no distortion, principal points) have no midpoint: ingest returns a
non-finite landmark without counting it invalid, and append_stereo_tracks rejects the track (status 2).
"""
import dataclasses
import glob
import json
import os

import numpy as np
import pytest

import oracle_lib as ol
from hyperslam_b200 import synthetic, trajectory
from test_oracle import window_from_golden

U = 2.0 ** -53
C = 150.0
INGEST = sorted(glob.glob(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ingest", "*.json")))


def stereo_frame(win, stamp, n, rng, noise=0.0):
    """n landmarks seen by cameras 0 and 1 at `stamp`: pixels from the numpy forward model."""
    k = win.order
    truth = win.truth
    base = int(np.searchsorted(truth["knots"][:, 7], stamp, side="right") - 1 - (k - 1) // 2)
    lm_idx = rng.choice(win.landmarks.shape[0], size=n, replace=False)
    st = np.full(n, stamp)
    px0, ps0 = synthetic.pixel_model(truth["knots"], k, win.cameras, truth["landmarks"], st, np.zeros(n, dtype=int), lm_idx)
    px1, ps1 = synthetic.pixel_model(truth["knots"], k, win.cameras, truth["landmarks"], st, np.ones(n, dtype=int), lm_idx)
    ok = (ps0[:, 2] > 0.3) & (ps1[:, 2] > 0.3)
    return base, lm_idx[ok], px0[ok] + rng.normal(0, noise, px0[ok].shape), px1[ok] + rng.normal(0, noise, px1[ok].shape), ps0[ok], ps1[ok]


def make_truth_window(order):
    return synthetic.make_window(order=order, num_knots=16, num_landmarks=200, num_imu=0, seed=synthetic.SEED_BASE + 700 + order, perturb=False)


@pytest.mark.parametrize("order", [4, 6])
def test_oracle_ingest_is_exact_on_noise_free_tracks(order):
    """distort(undistort(pixel)) = pixel, bearings are the unit rays of the landmark in each sensor frame, and the
    midpoint triangulation returns the landmark itself when the rays intersect."""
    win = make_truth_window(order)
    rng = np.random.default_rng(5)
    stamp = 0.731
    base, lm, px0, px1, ps0, ps1 = stereo_frame(win, stamp, 60, rng)
    assert lm.size > 20
    B0, B1, L = ol.ingest_stereo_frame(win.knots[base:base + order], stamp, win.cameras[0], win.cameras[1], px0, px1)
    assert np.abs(B0 - ps0 / np.linalg.norm(ps0, axis=1, keepdims=True)).max() < 1e-12
    assert np.abs(B1 - ps1 / np.linalg.norm(ps1, axis=1, keepdims=True)).max() < 1e-12
    assert np.abs(np.linalg.norm(B0, axis=1) - 1).max() < 1e-15
    assert np.abs(L - win.truth["landmarks"][lm]).max() < 1e-9
    # re-projecting the bearing through the forward camera model gives the pixel back
    back = synthetic.project(win.cameras, np.zeros(lm.size, dtype=int), B0)
    assert np.abs(back - px0).max() < 1e-9


def load_tracks(path):
    """The fixture, its tracks as arrays, and the window it runs on: its spline-edge fixture's knots, biases, gravity and
    IMU / pose factors with the fixture's cameras, and no landmarks or visual factors (tracks arrive in stamp order)."""
    with open(path) as f:
        case = json.load(f)
    with open(os.path.join(os.path.dirname(os.path.dirname(path)), case["edges"] + ".json")) as f:
        edges = json.load(f)
    win = dataclasses.replace(window_from_golden(dict(edges, pixel=[], bearing=[])), cameras=np.array(case["cameras"]), landmarks=np.zeros((0, 3)))
    tr = case["tracks"]
    cols = dict(stamp=np.array([t["stamp"] for t in tr]), cam0=np.array([t["cam0"] for t in tr], np.int32),
                cam1=np.array([t["cam1"] for t in tr], np.int32), px0=np.array([t["px0"] for t in tr]), px1=np.array([t["px1"] for t in tr]),
                parallel=np.array([t["lm"] is None for t in tr]))
    return case, cols, win


def ingest_ratios(case, b0, b1, lm):
    """Worst |got - ref| / (u scale) of the bearings and, per depth decade of |p_0|, of the landmarks."""
    cams = np.array(case["cameras"])
    worst = {}
    for n, t in enumerate(case["tracks"]):
        worst["bearing"] = max(worst.get("bearing", 0.0), np.abs(b0[n] - t["b0"]).max() / U, np.abs(b1[n] - t["b1"]).max() / U)
        if t["lm"] is None:
            continue
        p0, ref = np.array(t["p0"]), np.array(t["lm"])
        baseline = np.linalg.norm(cams[t["cam1"], 4:7] - cams[t["cam0"], 4:7])
        scale = max(np.linalg.norm(ref), p0 @ p0 / baseline)
        key = "landmark_%gm" % 10.0 ** np.floor(np.log10(np.linalg.norm(p0)))
        worst[key] = max(worst.get(key, 0.0), np.abs(lm[n] - ref).max() / (U * scale))
    return worst


def check_ingest(worst, record_property, name):
    for key, v in worst.items():
        record_property(f"{name}:{key}", round(v, 3))
    bad = {key: v for key, v in worst.items() if not v <= C}
    assert not bad, f"{name}: worst |got - ref| / (u scale) above C = {C:g}: {bad}"


@pytest.mark.parametrize("path", INGEST, ids=[os.path.basename(p) for p in INGEST])
def test_oracle_ingest_against_golden(path, record_property):
    """CPU twin of the GPU test: oracle/ho_ingest.h under the same bound."""
    case, t, win = load_tracks(path)
    k, cams = win.order, win.cameras
    out = [np.zeros((t["stamp"].size, 3)) for _ in range(3)]
    for n, stamp in enumerate(t["stamp"]):
        j = int(np.searchsorted(win.knots[:, 7], stamp, side="right") - 1) - (k - 1) // 2
        res = ol.ingest_stereo_frame(win.knots[j:j + k], stamp, cams[t["cam0"][n]], cams[t["cam1"][n]], t["px0"][n:n + 1], t["px1"][n:n + 1])
        for o, r in zip(out, res):
            o[n] = r[0]
    assert not np.isfinite(out[2][t["parallel"]]).any() and np.isfinite(out[2][~t["parallel"]]).all()
    check_ingest(ingest_ratios(case, *out), record_property, os.path.basename(path))


def test_trajectory_format_and_tum_conversion(tmp_path):
    """One line per sample: stamp, qx, qy, qz, qw, px, py, pz in %.20e separated by ', ' (reference main.cpp:57-79);
    TUM conversion reorders to stamp, position, quaternion (evaluation/conversions.py:7)."""
    lower, upper = trajectory.state_range(np.arange(10) * 0.1, 4)
    assert (lower, upper) == (0.1, 0.7000000000000001) or (abs(lower - 0.1) < 1e-15 and abs(upper - 0.7) < 1e-12)
    stamps = trajectory.sample_range(0.1, 0.7, 100)
    assert stamps.size == 60 and abs(stamps[0] - 0.1) < 1e-15 and stamps[-1] < 0.7
    line = trajectory.format_line(1.5, np.array([0.0, 0.0, 0.6, 0.8, 1.0, -2.0, 3.25]))
    fields = line.split(", ")
    assert len(fields) == 8 and fields[0] == "1.50000000000000000000e+00" and fields[5] == "1.00000000000000000000e+00"
    src, dst = tmp_path / "estimation.hyper", tmp_path / "estimation.tum"
    rows = np.random.default_rng(1).normal(size=(5, 8))
    with open(src, "w") as f:
        for r in rows:
            f.write(trajectory.format_line(r[0], r[1:]) + "\n")
    trajectory.convert_hyper_to_tum_format(str(src), str(dst))
    tum = np.loadtxt(dst)
    assert tum.shape == (5, 8) and np.array_equal(tum, rows[:, [0, 5, 6, 7, 1, 2, 3, 4]])
    assert len(open(dst).readline().split(" ")) == 8


@pytest.mark.gpu
@pytest.mark.parametrize("order", [4, 6])
def test_gpu_ingest_matches_oracle(built, order):
    from hyperslam_b200 import runtime
    win = make_truth_window(order)
    rng = np.random.default_rng(9)
    ctx = runtime.Context(0)
    ctx.load_window(win)
    stamps, c0, c1, p0, p1, refs = [], [], [], [], [], []
    for stamp in (0.41, 0.655, 0.93):
        base, lm, px0, px1, _, _ = stereo_frame(win, stamp, 50, rng, noise=0.4)
        B0, B1, L = ol.ingest_stereo_frame(win.knots[base:base + order], stamp, win.cameras[0], win.cameras[1], px0, px1)
        stamps += [stamp] * lm.size; c0 += [0] * lm.size; c1 += [1] * lm.size
        p0.append(px0); p1.append(px1); refs.append((B0, B1, L))
    b0, b1, lm_w, bad = ctx.ingest_stereo(np.array(stamps), np.array(c0), np.array(c1), np.concatenate(p0), np.concatenate(p1))
    assert bad == 0
    assert np.abs(b0 - np.concatenate([r[0] for r in refs])).max() < 1e-12
    assert np.abs(b1 - np.concatenate([r[1] for r in refs])).max() < 1e-12
    ref_l = np.concatenate([r[2] for r in refs])
    assert np.abs(lm_w - ref_l).max() < 1e-9 * max(1.0, np.abs(ref_l).max())
    # invalid stamp / camera are reported, not silently processed
    _, _, _, bad = ctx.ingest_stereo(np.array([99.0, 0.5]), np.array([0, 7]), np.array([1, 1]), np.zeros((2, 2)), np.zeros((2, 2)))
    assert bad == 2
    ctx.close()


@pytest.mark.gpu
@pytest.mark.parametrize("path", INGEST, ids=[os.path.basename(p) for p in INGEST])
def test_gpu_ingest_against_golden(built, path, record_property):
    """hb200_ingest_stereo against the known answers; hb200_append_stereo_tracks writes the same landmarks and
    bearing factors bit for bit, and rejects the parallel track."""
    from hyperslam_b200 import runtime
    from test_gpu_stereo_window import error_code
    case, t, win = load_tracks(path)
    ctx, ref = runtime.Context(0), runtime.Context(0)
    ctx.load_window(win)
    ref.load_window(win)
    args = [t[key] for key in ("stamp", "cam0", "cam1", "px0", "px1")]
    b0, b1, lm, bad = ctx.ingest_stereo(*args)
    par = t["parallel"]
    assert bad == 0 and not np.isfinite(lm[par]).any() and np.isfinite(lm[~par]).all()
    worst = ingest_ratios(case, b0, b1, lm)

    counts = ctx.factor_counts().tolist()
    assert error_code(ctx.append_stereo_tracks, *[a[par] for a in args], -np.ones(int(par.sum()), np.int32)) == 2
    assert ctx.L == 0 and ctx.factor_counts().tolist() == counts
    ok = ~par
    n = int(ok.sum())
    out, n_new = ctx.append_stereo_tracks(*[a[ok] for a in args], -np.ones(n, np.int32))
    assert n_new == n and np.array_equal(out, np.arange(n))
    assert np.array_equal(ctx.state()["landmarks"], lm[ok])
    # the bearing factors it wrote: the same as appending ingest's bearings at positions 2i, 2i + 1
    ref.append_landmarks(lm[ok])
    ref.append_bearing_factors(np.repeat(t["stamp"][ok], 2), np.stack([t["cam0"][ok], t["cam1"][ok]], 1).ravel(), np.repeat(np.arange(n, dtype=np.int32), 2),
                               np.stack([b0[ok], b1[ok]], 1).reshape(-1, 3))
    assert ctx.factor_counts().tolist() == ref.factor_counts().tolist()
    outs = []
    for c in (ctx, ref):
        c.evaluate(jacobians=True)
        outs.append(c.outputs())
    for key in ("b_r", "b_Jp", "b_Jl"):
        assert np.array_equal(outs[0][key], outs[1][key]), key
    ctx.close()
    ref.close()
    check_ingest(worst, record_property, os.path.basename(path))


@pytest.mark.gpu
def test_gpu_estimation_dump_matches_oracle_interpolation(built, tmp_path):
    from hyperslam_b200 import runtime
    win = synthetic.make_window(order=4, num_knots=14, num_landmarks=30, num_imu=40, seed=synthetic.SEED_BASE + 720)
    ctx = runtime.Context(0)
    ctx.load_window(win)
    path = tmp_path / "estimation.hyper"
    n = trajectory.write_estimation(ctx, str(path), win.knots[:, 7], win.order, root=100.0)
    data = np.loadtxt(path, delimiter=",")
    lower, upper = trajectory.state_range(win.knots[:, 7], win.order)
    assert data.shape == (n, 8) and n == trajectory.sample_range(lower, upper).size
    left = (win.order - 1) // 2
    stamps = trajectory.sample_range(lower, upper)
    for i in range(0, n, max(1, n // 25)):
        t, row = stamps[i], data[i]
        assert abs(row[0] - (100.0 + t)) < 1e-12
        j = int(np.searchsorted(win.knots[:, 7], t, side="right") - 1) - left
        v, _, _, _ = ol.state_evaluate(win.knots[j:j + win.order], t, 0, False)
        if np.dot(v[:4], row[1:5]) < 0:
            v[:4] = -v[:4]          # q and -q are the same rotation
        assert np.abs(row[1:] - v).max() < 1e-12, (i, t, row[1:], v)
    ctx.close()
