"""Every factor pass the solver runs against the 80-digit known answers in tests/golden/, on windows of any size.

A golden factor's residual and Jacobians depend only on that factor and the state.  A window that keeps a fixture's
state (knots, biases, gravity, cameras, IMU block, landmarks, pose sensors) and holds counts[family][g] copies of its
golden factor g therefore has an exact known answer for every factor.  `replicate` builds such a window in a shuffled
user order (hb200_bind's stable sort by knot base does the grouping) and returns the golden index of every user-order
factor; `expand` maps the fixture's factor lists through it, so test_gpu_spline_edges.factor_ratios applies unchanged.

Shapes, per fixture:
  S0           the fixture as it is;
  S1           4 SMs - 1 evaluation CTAs (n_pix_blocks + n_imu_blocks): the merged factor_eval_kernel on many CTAs;
  S2-merged    exactly 4 SMs CTAs: still merged (test_gpu_assembly.test_merged_and_separate_eval);
  S2-separate  4 SMs + 1 CTAs: pixel_eval_kernel and inertial_eval_kernel as separate launches;
  S3           >= 40 000 visual and >= 16 384 inertial factors: separate launches.
The bearing_pose fixtures have no inertial factors, so their windows always take separate launches; they carry the
bearing and pose families.  RUNS sets the visual runs (factors of one knot base, consecutive in the bound list) so that
over each order's windows runs of 1, 63, 64, 65 and several hundred factors start at tile offsets 0 and 63, Nv = 1 and
63 (mod 64) occur, pixel and bearing factors share tiles (spline_edges), more than 64 pose factors run
manifold_eval_kernel on several CTAs, and the inertial J^T J splits its runs (imu_splits > 1).  `shape_facts` reads
the runs, tiles and counts from the bound index maps; imu_splits is not read back from the device but restated from
the host heuristic (`inertial_splits`) on the run count the index maps give, a guard on the shape design only.

Passes, on every shape: evaluate (hb200_evaluate with Jacobians), fused (hb200_build_system: its factor kernels
rewrite the residuals and Jacobians while they accumulate the pixel J^T J), the deterministic fused pass
(set_deterministic) and the cost-only sweep (hb200_cost).  build_system needs an evaluate first, so its outputs could
be the evaluate pass's left in place; `fused_pass` therefore also fills the buffers at an LM iteration's trial state,
restores the state and requires the iteration profile's assembly (the same enqueue_assembly) to leave build_system's
bits.  (The direct route, a trial evaluate before build_system, is refused: the trial sweep clears evaluated_J.)
Checks:

* rows: every residual and Jacobian row of every copy, inertial bias weights included, within C u scale(row) of its
  known answer (factor_ratios, C = 150);
* position independence: within one pass all copies of a golden factor are bit-identical.  The kernels make a factor's
  outputs a function of that factor's inputs alone: pixel_factor and inertial_factor read their knot-table rows from
  the CTA's staged tile or, for tiles spanning more than kTileRows rows, from global memory (the same doubles).  The
  fixtures' knot bases span at most 8 table rows against kTileRows = 16, so every tile here is staged: the global-memory
  branch is out of reach of the known answers and only its argument, not its output, is covered here.  The inertial backward-sweep stash is a per-thread slot, manifold_eval_kernel reads the table
  directly, and nothing crosses lanes but the cost partials and, in the fused passes, the J^T J after the factor's rows
  are stored.  So one copy's rows stand for all of them: factor_ratios runs on the first copy of each golden factor
  once the copies are known to be identical (test_oracle_replicated_windows checks that this equals factor_ratios
  over every copy);
* across passes: the instantiations may contract differently, so evaluate and fused are not held to bit identity; the
  largest difference in ulps (exact integer distance, `ulps`) and whether the bits are equal are recorded;
* cost: hb200_cost against  sum_f rho_f / 2  in mpmath from the golden residuals, rho = Huber on s = |r|^2 with
  huber_pixel / huber_bearing for visual factors, imu_loss_scale s for inertial factors, s for pose factors:
      |cost - ref| <= sum_f w_f |r_f|_1 C u scale_f  +  gamma_N sum_f rho_f / 2,   gamma_N = N u / (1 - N u).
  The first term is each factor's own: d(rho_f / 2) / dr_i = w_f r_i with w_f = rho'(s) <= 1 (Huber), imu_loss_scale
  or 1, and every residual entry is within C u scale_f, scale_f the largest residual-row scale factor_ratios uses for
  that factor.  The second is the rounding of the terms and their sum: E = 10 roundings to evaluate one term (the
  squares and their sum, the square root, and 2 delta sqrt(s) - delta^2, whose cancellation is at most a factor 2
  since sqrt(s) > delta, the loss scale), and a sum of n values in any order is within gamma_(n-1).  N = E plus the
  values and partial sums that reach the total: on the device 64 lanes per evaluation CTA (idle lanes add exact
  zeros), two warp sums and one partial per CTA, and scalars_kernel's 256 lane sums; in the oracle the factors and
  three OpenMP reductions' partials.  The deltas sit between the two neighbouring |r| of each visual family with the
  largest ratio, so every visual family has factors on both sides of delta^2;
* kernels: the evaluate pass's labels (profile_iteration(evaluate_only=True)) and the fused passes' (the iteration
  profile) equal `plan()`.  A label does not tell the Jacobian, fused and cost-only instantiations apart; the call
  that ran decides which one it was.  The profiles are taken after the outputs are read: a full profile runs an LM
  iteration and moves the state.

hb200_interpolate is checked the same way on the spline_edges stamps replicated past 64 SMs stamps.
"""
import os
import zlib

import numpy as np
import pytest

import oracle_lib as ol
from test_gpu_assembly import ASSEMBLY_KERNELS, EVAL_THREADS, IMU_MMA_MIN, num_sms, plan
from test_gpu_spline_edges import C, GOLDEN, U, check, factor_ratios, interpolate_ratios, load, oracle_interpolate
from test_oracle import window_from_golden

FAMILIES = ("pixel", "bearing", "pose", "inertial")
OUT_KEYS = {"pixel": ("v_r", "v_Jp", "v_Jl"), "bearing": ("b_r", "b_Jp", "b_Jl"), "pose": ("m_r", "m_Jp"),
            "inertial": ("i_r", "i_Jp", "i_wg", "i_wa", "i_Jg")}
WINDOW_KEYS = {"pixel": ("v_stamp", "v_cam", "v_lm", "v_pixel"), "bearing": ("b_stamp", "b_cam", "b_lm", "b_bearing"),
               "pose": ("m_stamp", "m_sensor", "m_pose"), "inertial": ("i_stamp", "i_meas")}
EVAL_KERNELS = {"factor_eval_kernel", "pixel_eval_kernel", "inertial_eval_kernel", "manifold_eval_kernel"}
SHAPES = ("S0", "S1", "S2-merged", "S2-separate", "S3")
SMS_H100 = 132                  # H100 SXM: the CPU twin's S1-sized windows
E_TERM = 10                     # roundings to evaluate one cost term
POSE_COPIES = {"S3": 255}       # pose factors of the replicated windows (otherwise 129: three manifold CTAs)
LONG_RUN = 256                  # a run this long counts as "several hundred"

# Visual runs of each replicated window, in ascending knot base (pixel and bearing bases together): a run's length, or
# None for the run that takes the rest; and Nv mod 64 (1 .. 64).
RUNS = {
    "k4_bearing_pose": {"S1": ([1, None], 1), "S2-merged": ([63, None], 63), "S2-separate": ([None, 65], 1), "S3": ([64, None], 63)},
    "k4_euroc": {"S1": ([1, 63, None], 1), "S2-merged": ([63, 1, None], 63), "S2-separate": ([64, 65, None], 63), "S3": ([None, 65, 64], 64)},
    "k4_generic_calibration": {"S1": ([63, 64, None], 63), "S2-merged": ([64, 63, None], 1), "S2-separate": ([63, 63, None], 1),
                               "S3": ([65, None, 65], 64)},
    "k4_spline_edges": {"S1": ([1, 64, 65, None], 1), "S2-merged": ([63, None, 64, 65], 63), "S2-separate": ([None, 63, 64, 2], 1),
                        "S3": ([None, 64, 63, 300], 1)},
    "k6_bearing_pose": {"S1": ([None], 1), "S2-merged": ([None], 63), "S2-separate": ([None], 1), "S3": ([None], 63)},
    "k6_euroc": {"S1": ([65, None], 1), "S2-merged": ([None, 65], 64), "S2-separate": ([None, 64], 63), "S3": ([None, 63], 62)},
    "k6_generic_calibration": {"S1": ([1, None], 1), "S2-merged": ([None, 1], 64), "S2-separate": ([63, None], 63), "S3": ([64, None], 1)},
    "k6_spline_edges": {"S1": ([63, 64, None], 1), "S2-merged": ([64, 63, None], 63), "S2-separate": ([65, 63, None], 1),
                        "S3": ([None, 65, 300], 44)},
}
FIXTURES = [p for p in GOLDEN if os.path.basename(p)[:-5] in RUNS]
SPLINE_EDGES = [p for p in FIXTURES if "spline_edges" in p]


def fixture_name(path):
    return os.path.basename(path)[:-5]


# ---- replicated windows ----------------------------------------------------------------------------------------
def huber_deltas(case):
    """huber_pixel / huber_bearing between the two neighbouring |r| of each visual family with the largest ratio."""
    out = {}
    for fam, key in (("pixel", "huber_pixel"), ("bearing", "huber_bearing")):
        n = np.sort([np.linalg.norm(p["r"]) for p in case.get(fam, [])])
        if n.size >= 2:
            i = int(np.argmax(n[1:] / n[:-1]))
            out[key] = float(np.sqrt(n[i] * n[i + 1]))
    return out


def replicate(case, counts=None, seed=None):
    """The fixture's window with counts[family][g] copies of golden factor g (None: the fixture's factors once each), in
    user order shuffled by `seed` (None: golden order), and the Huber deltas of huber_deltas.  Returns (window, golden
    index of every user-order factor by family)."""
    win = window_from_golden(case)
    for key, v in huber_deltas(case).items():
        setattr(win, key, v)
    rng = np.random.default_rng(seed)
    gidx = {}
    for fam in FAMILIES:
        n = len(case.get(fam, []))
        g = np.repeat(np.arange(n), np.ones(n, int) if counts is None else counts[fam])
        gidx[fam] = g if seed is None else rng.permutation(g)
        for key in WINDOW_KEYS[fam]:
            setattr(win, key, np.ascontiguousarray(getattr(win, key)[gidx[fam]]))
    return win, gidx


def expand(case, gidx):
    """The fixture's factor lists mapped through the golden index: one known answer per user-order factor."""
    out = dict(case)
    for fam in FAMILIES:
        if fam in case:
            out[fam] = [case[fam][g] for g in gidx[fam]]
    return out


def _split(n, parts):
    return np.array([n // parts + (i < n % parts) for i in range(parts)], int) if parts else np.zeros(0, int)


def visual_runs(case):
    """Golden visual factors grouped by knot base, ascending: [(base, [(family, g), ...])], pixel factors first."""
    by = {}
    for fam in ("pixel", "bearing"):
        for g, p in enumerate(case.get(fam, [])):
            by.setdefault(p["base"], []).append((fam, g))
    return sorted(by.items())


def eval_blocks(shape, sms):
    """n_pix_blocks + n_imu_blocks of a replicated shape (S3: no target)."""
    return {"S1": 4 * sms - 1, "S2-merged": 4 * sms, "S2-separate": 4 * sms + 1}.get(shape)


def shape_counts(name, case, shape, sms):
    """counts[family][g] of a replicated shape (None for S0)."""
    if shape == "S0":
        return None
    lengths, res = RUNS[name][shape]
    runs = visual_runs(case)
    assert len(lengths) == len(runs), (name, shape, len(runs))
    has_imu = bool(case["inertial"])
    if shape == "S3":
        nv, ni = 64 * 625 + res, (IMU_MMA_MIN + 27 if has_imu else 0)
    else:
        blocks = eval_blocks(shape, sms)
        npb = 2 * sms if has_imu else blocks
        nv = 64 * (npb - 1) + res
        ni = 64 * (blocks - npb - 1) + 37 if has_imu else 0
    fill = nv - sum(n for n in lengths if n is not None)
    counts = {fam: np.zeros(len(case.get(fam, [])), int) for fam in FAMILIES}
    for (_, members), n in zip(runs, lengths):
        for (fam, g), c in zip(members, _split(fill if n is None else n, len(members))):
            counts[fam][g] = c
    counts["inertial"] = _split(ni, len(case["inertial"]))
    counts["pose"] = _split(POSE_COPIES.get(shape, 129), len(case.get("pose", [])))
    for fam in FAMILIES:
        assert (counts[fam] >= 1).all(), (name, shape, fam, counts[fam])   # every golden factor has a copy
    return counts


def shape_window(path, shape, sms):
    case = load(path)
    name = fixture_name(path)
    counts = shape_counts(name, case, shape, sms)
    seed = None if counts is None else zlib.crc32(f"{name}-{shape}".encode())
    win, gidx = replicate(case, counts, seed)
    return case, win, gidx


def inertial_splits(ni, nruns, k, sms):
    """CTAs per inertial run of the J^T J kernel (hb200_api.cu: imu_splits / imu_splits_mma and inertial_splits)."""
    r = max(nruns, 1)
    if ni < IMU_MMA_MIN or k != 4:
        return max(1, min((2 * sms + r - 1) // r, max(1, ni // (8 * r))))
    return max(1, min((6 * sms + r - 1) // r, max(1, ni // (16 * r))))


def shape_facts(case, gidx, pixel_base, imu_maps, sms):
    """What the bound window holds, from the pixel and inertial index maps and the bearing factors' golden bases: the
    visual runs as (length, tile offset of their first factor), Nv mod 64, tiles holding pixel and bearing factors,
    manifold CTAs, evaluation CTAs, and the inertial J^T J's CTAs per run."""
    bb = np.array([case["bearing"][g]["base"] for g in gidx["bearing"]], np.int64)
    base = np.concatenate([np.asarray(pixel_base, np.int64), bb])
    kind = np.repeat([0, 1], [len(pixel_base), bb.size])
    o = np.argsort(base, kind="stable")      # the bound visual list: [pixel | bearing] stable-sorted by knot base
    base, kind = base[o], kind[o]
    nv = base.size
    starts = np.flatnonzero(np.r_[True, base[1:] != base[:-1]]) if nv else np.zeros(0, int)
    lengths = np.diff(np.r_[starts, nv])
    tile = np.arange(nv) // EVAL_THREADS
    ib, ig, ia = imu_maps
    ni, nm = len(ib), gidx["pose"].size
    nruns = len(set(zip(ib.tolist(), ig.tolist(), ia.tolist())))
    npb, nib = -(-nv // EVAL_THREADS), -(-ni // EVAL_THREADS)
    return dict(nv=nv, nv_mod=nv % 64, runs=sorted(set(zip(lengths.tolist(), (starts % EVAL_THREADS).tolist()))),
                mixed_tiles=int(np.intersect1d(tile[kind == 0], tile[kind == 1]).size), ni=ni, pose_ctas=-(-nm // EVAL_THREADS),
                eval_blocks=npb + nib, imu_splits=inertial_splits(ni, nruns, case["window"]["order"], sms) if ni else 0)


def golden_facts(case, gidx, sms):
    """shape_facts from the golden bases (what the index maps must show)."""
    ib = np.array([case["inertial"][g]["base"] for g in gidx["inertial"]], np.int64)
    bb = np.array([case["inertial"][g]["bias_base"] for g in gidx["inertial"]], np.int64)
    return shape_facts(case, gidx, [case["pixel"][g]["base"] for g in gidx["pixel"]], (ib, bb, bb), sms)


def run_category(length):
    return length if length in (1, 63, 64, 65) else ("several hundred" if length >= LONG_RUN else None)


REQUIRED_RUNS = {(n, o) for n in (1, 63, 64, 65, "several hundred") for o in (0, EVAL_THREADS - 1)}


# ---- the checker -----------------------------------------------------------------------------------------------
def copy_mismatches(gidx, out):
    """(output key, golden index) of every golden factor whose copies are not bit-identical."""
    bad = []
    for fam, keys in OUT_KEYS.items():
        g = gidx[fam]
        if not g.size:
            continue
        _, first = np.unique(g, return_index=True)
        for key in keys:
            bits = np.ascontiguousarray(out[key]).reshape(g.size, -1).view(np.int64)
            diff = (bits != bits[first[g]]).any(axis=1)
            bad += [(key, int(x)) for x in np.unique(g[diff])]
    return bad


def representatives(gidx, out):
    """The outputs of the first copy of every golden factor, in golden order."""
    rep = {}
    for fam, keys in OUT_KEYS.items():
        g = gidx[fam]
        if g.size:
            ids, first = np.unique(g, return_index=True)
            assert np.array_equal(ids, np.arange(ids.size)), f"{fam}: a golden factor has no copy"
            rep.update({key: out[key][first] for key in keys})
    return rep


def pass_ratios(case, gidx, out):
    """(copies that differ, factor_ratios of the pass).  With identical copies, the first copy's ratios are every copy's."""
    return copy_mismatches(gidx, out), factor_ratios(case, representatives(gidx, out))


def ulps(a, b):
    """Largest distance in units in the last place between two float64 arrays of one shape, in exact integer
    arithmetic: each double maps to its signed position on the number line (+0 and -0 both 0); a distance between two
    of one sign fits int64, one across zero is taken in Python integers."""
    def ordered(x):
        i = np.ascontiguousarray(x, np.float64).view(np.int64).ravel().copy()
        neg = i < 0
        i[neg] = np.iinfo(np.int64).min - i[neg]
        return i
    oa, ob = ordered(a), ordered(b)
    same = (oa < 0) == (ob < 0)
    worst = int(np.abs(oa[same] - ob[same]).max(initial=0))
    for x, y in zip(oa[~same].tolist(), ob[~same].tolist()):
        worst = max(worst, abs(x - y))
    return worst


def same_bits(a, b):
    return a.shape == b.shape and np.array_equal(np.ascontiguousarray(a).view(np.int64), np.ascontiguousarray(b).view(np.int64))


def residual_scale(fam, p):
    """The largest residual-row scale factor_ratios uses for golden factor p."""
    if fam == "pixel":
        J = np.hstack([np.array(p["Jp"]), np.array(p["Jl"])])
        return max(max(np.abs(J[i]).max(), abs(p["r"][i]), np.abs(p["pixel"]).max()) for i in range(2))
    if fam == "bearing":
        return max(np.abs(np.concatenate([p["Jp"], p["Jl"]])).max(), abs(p["r"][0]), 1.0)
    if fam == "pose":
        J = np.array(p["Jp"])
        return max(max(np.abs(J[i]).max(), abs(p["r"][i]), np.abs(p["pose"]).max()) for i in range(6))
    Jg = np.array(p["Jg"])
    rows = [np.concatenate([p["Jp"][i], p["wg"] if i < 3 else p["wa"], Jg[i]]) for i in range(6)]
    return max(max(np.abs(rows[i]).max(), abs(p["r"][i]), np.abs(p["meas"][:3] if i < 3 else p["meas"][3:]).max()) for i in range(6))


def cost_reference(case, win, gidx):
    """(sum_f rho_f / 2 over the copies in gidx, in mpmath from the golden residuals; the factors' own bound terms
    sum_f w_f |r_f|_1 C u scale_f)."""
    import mpmath as mp
    mp.mp.dps = 40
    total, own = mp.mpf(0), 0.0
    for fam in FAMILIES:
        if not gidx[fam].size:
            continue
        copies = np.bincount(gidx[fam], minlength=len(case[fam]))
        for g, p in enumerate(case[fam]):
            r = [mp.mpf(x) for x in p["r"]]
            s = sum(x * x for x in r)
            if fam in ("pixel", "bearing"):
                d = mp.mpf(win.huber_pixel if fam == "pixel" else win.huber_bearing)
                rho, w = (s, 1.0) if s <= d * d else (2 * d * mp.sqrt(s) - d * d, float(d / mp.sqrt(s)))
            elif fam == "inertial":
                rho, w = mp.mpf(win.imu_loss_scale) * s, win.imu_loss_scale
            else:
                rho, w = s, 1.0
            total += int(copies[g]) * rho / 2
            own += int(copies[g]) * w * float(sum(abs(x) for x in r)) * C * U * residual_scale(fam, p)
    return total, own


def gamma(n):
    return n * U / (1 - n * U)


def cost_ratio(cost, ref, own, n):
    """|cost - ref| over its bound own + gamma_(E + n) ref (n: values and partial sums that reach the total)."""
    import mpmath as mp
    bound = own + gamma(E_TERM + n) * float(ref)
    return float(abs(mp.mpf(cost) - ref)) / bound, bound


def device_cost_terms(win):
    """Values and partial sums of hb200_cost: 64 lanes, two warp sums and one partial per CTA, scalars_kernel's 256."""
    ctas = sum(-(-n // EVAL_THREADS) for n in (win.v_stamp.size + win.b_stamp.size, win.i_stamp.size, win.m_stamp.size))
    return (EVAL_THREADS + 3) * ctas + 256


def visual_delta_sides(case, win):
    """Visual families whose golden factors lie on both sides of delta^2."""
    both = set()
    for fam, d in (("pixel", win.huber_pixel), ("bearing", win.huber_bearing)):
        s = np.array([np.dot(p["r"], p["r"]) for p in case.get(fam, [])])
        if s.size and (s <= d * d).any() and (s > d * d).any():
            both.add(fam)
    return both


# ---- CPU twin --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("order", [4, 6])
def test_replicated_shapes_cover_the_tile_edges(order):
    """The replicated windows of one order, at H100 size, hold every case the device tests target."""
    sms = SMS_H100
    runs, nv_mod, mixed = set(), set(), 0
    for path in FIXTURES:
        case = load(path)
        if case["window"]["order"] != order:
            continue
        win, _ = replicate(case)
        assert visual_delta_sides(case, win) == {f for f in ("pixel", "bearing") if case.get(f)}, fixture_name(path)
        for shape in SHAPES[1:]:
            case, win, gidx = shape_window(path, shape, sms)
            f = golden_facts(case, gidx, sms)
            p = plan(win, sms)
            tag = (fixture_name(path), shape)
            runs |= {(run_category(n), o) for n, o in f["runs"]}
            nv_mod.add(f["nv_mod"])
            mixed += f["mixed_tiles"]
            if case.get("pose"):
                assert f["pose_ctas"] > 1, tag
            if case["inertial"]:
                assert f["imu_splits"] > 1, tag
                assert p["merged"] == (shape in ("S1", "S2-merged")), tag
            else:
                assert not p["merged"], tag
            if shape == "S3":
                assert f["nv"] >= 40000 and (f["ni"] >= 16384 or not case["inertial"]), tag
            else:
                assert f["eval_blocks"] == eval_blocks(shape, sms), (tag, f["eval_blocks"])
    assert REQUIRED_RUNS <= runs, REQUIRED_RUNS - runs
    assert {1, 63} <= nv_mod and mixed > 0, (nv_mod, mixed)


@pytest.mark.parametrize("path", FIXTURES, ids=[os.path.basename(p) for p in FIXTURES])
def test_oracle_replicated_windows(path, record_property):
    """The oracle on the S1-sized window (H100): index maps, copies, every row of every copy and the cost under the
    device's bounds; the first-copy ratios equal those over every copy."""
    case, win, gidx = shape_window(path, "S1", SMS_H100)
    name = fixture_name(path)
    ow = ol.OracleWindow(win)
    assert ow.bad == 0
    vb, ib, ig, ia = ow.index_maps()
    f = shape_facts(case, gidx, vb, (ib, ig, ia), SMS_H100)
    assert f == golden_facts(case, gidx, SMS_H100), f
    out = ow.evaluate()
    bad, worst = pass_ratios(case, gidx, out)
    assert not bad, bad[:10]
    assert factor_ratios(expand(case, gidx), out) == worst
    check(worst, record_property, name)
    ref, own = cost_reference(case, win, gidx)
    ratio, _ = cost_ratio(ow.cost(), ref, own, sum(g.size for g in gidx.values()) + 3 * ol.num_threads())
    record_property(f"{name}:cost_ratio", ratio)
    assert ratio <= 1.0, ratio
    if "interpolate" in case:
        gi = replicated_stamps(case, SMS_H100)
        big = dict(case, interpolate=[case["interpolate"][g] for g in gi])
        pose, vel, acc = oracle_interpolate(big)
        check(interpolate_ratios(big, pose, vel, acc), record_property, name)


def _step(x, n):
    """x moved up by n ulps."""
    for _ in range(n):
        x = np.nextafter(x, np.inf)
    return x


@pytest.mark.parametrize("x", [1.0, 0.37, 123.4, -2.5, 1e-3, 5e-324, 1.7e308, -1e300])
@pytest.mark.parametrize("n", [0, 1, 3, 600])
def test_ulps_counts_each_step(x, n):
    """ulps is the exact number of nextafter steps, at every magnitude and on both sides of zero."""
    a = np.array([x, -x, 0.5])
    b = np.array([_step(x, n), -_step(x, n), 0.5])
    assert ulps(a, b) == n
    assert ulps(b, a) == n
    assert same_bits(a, b) == (n == 0)


def test_ulps_across_zero():
    tiny = np.nextafter(0.0, 1.0)
    assert ulps(np.array([0.0]), np.array([-0.0])) == 0 and not same_bits(np.array([0.0]), np.array([-0.0]))
    assert ulps(np.array([tiny]), np.array([-tiny])) == 2
    assert ulps(np.array([-tiny]), np.array([_step(tiny, 4)])) == 6
    top = np.finfo(np.float64).max
    assert ulps(np.array([top]), np.array([-top])) == 2 * int(np.array(top).view(np.int64))


@pytest.mark.parametrize("path", FIXTURES, ids=[os.path.basename(p) for p in FIXTURES])
def test_checker_rejects_perturbations(path):
    """The checker fails on one copy moved by one ulp, on a golden-index map rotated by one, and on a cost off by twice
    its bound."""
    case = load(path)
    counts = {fam: np.full(len(case.get(fam, [])), 3) for fam in FAMILIES}
    win, gidx = replicate(case, counts, seed=5)
    out = ol.OracleWindow(win).evaluate()
    bad, worst = pass_ratios(case, gidx, out)
    assert not bad and max(worst.values()) <= C
    rng = np.random.default_rng(1)
    for fam, keys in OUT_KEYS.items():
        g = gidx[fam]
        if not g.size:
            continue
        _, first = np.unique(g, return_index=True)
        f = int(rng.choice(np.setdiff1d(np.arange(g.size), first)))   # a copy other than the first
        for key in keys:
            moved = {k: v.copy() for k, v in out.items()}
            row = moved[key][f].reshape(-1)
            e = int(rng.integers(row.size))
            row[e] = np.nextafter(row[e], np.inf)
            moved[key][f] = row.reshape(moved[key][f].shape)
            assert (key, int(g[f])) in pass_ratios(case, gidx, moved)[0], (fam, key)
        if len(case[fam]) > 1:
            rotated = dict(gidx, **{fam: np.roll(g, 1)})
            assert pass_ratios(case, rotated, out)[0], fam
            assert max(factor_ratios(expand(case, rotated), out).values()) > C, fam
    ref, own = cost_reference(case, win, gidx)
    n = sum(g.size for g in gidx.values()) + 3 * ol.num_threads()
    ratio, bound = cost_ratio(ol.OracleWindow(win).cost(), ref, own, n)
    assert ratio <= 1.0, ratio
    for off in (2 * bound, -2 * bound):
        assert cost_ratio(float(ref) + off, ref, own, n)[0] > 1.0, off


def replicated_stamps(case, sms):
    """Golden index of every stamp of a shuffled replication of the interpolate stamps past 64 SMs stamps."""
    n = len(case["interpolate"])
    copies = -(-(64 * sms + 1) // n)
    return np.random.default_rng(11).permutation(np.repeat(np.arange(n), copies))


# ---- GPU -------------------------------------------------------------------------------------------------------
def _names(profile):
    return {name for name, _ in profile}


def fused_pass(ctx, failures, tag):
    """build_system's outputs, after checking that its factor kernels write them: the buffers are filled at a moved
    state (an LM iteration's trial state), the state is restored, and the iteration profile -- whose assembly is
    build_system's -- must leave the same bits build_system left.  build_system cannot be checked that way directly:
    it refuses to run after a trial evaluate, which clears evaluated_J.  Every factor must differ between the two
    states in every output but the inertial bias weights, which depend on the stamps alone.  Returns (outputs, kernels
    the profile ran)."""
    ctx.evaluate(jacobians=True)
    ctx.build_system()
    out = ctx.outputs()
    ctx.snapshot()
    ctx.iterate(1)                           # builds the trial state x + delta, accepted or not
    ctx.evaluate(jacobians=True, trial=True)
    moved = ctx.outputs()
    ctx.restore()
    ran = _names(ctx.profile_iteration(reps=1))
    again = ctx.outputs()
    for key in out:
        if key not in ("i_wg", "i_wa") and out[key].size and (moved[key] == out[key]).reshape(len(out[key]), -1).all(axis=1).any():
            failures.append(f"{tag}: the trial state leaves factors of {key} in place")
        if not same_bits(again[key], out[key]):
            failures.append(f"{tag}: the iteration's fused pass left {key} other than build_system did")
    return out, ran


@pytest.mark.gpu
@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("path", FIXTURES, ids=[os.path.basename(p) for p in FIXTURES])
def test_gpu_factor_passes(built, path, shape, record_property):
    from hyperslam_b200 import runtime
    from test_gpu_deterministic import DET_KERNELS, det_kernels
    sms = num_sms()
    case, win, gidx = shape_window(path, shape, sms)
    name = f"{fixture_name(path)}:{shape}"
    p = plan(win, sms)
    outs, kernels, failures = {}, {}, []
    ctx = runtime.Context(0)
    try:
        ctx.load_window(win)
        cost = ctx.cost()
        ctx.evaluate(jacobians=True)
        outs["evaluate"] = ctx.outputs()
        maps = ctx.index_maps()
        kernels["evaluate"] = _names(ctx.profile_iteration(reps=1, evaluate_only=True)) & (EVAL_KERNELS | DET_KERNELS)
        outs["fused"], ran = fused_pass(ctx, failures, "fused")
        kernels["fused"] = ran & (ASSEMBLY_KERNELS | DET_KERNELS)
    finally:
        ctx.close()
    ctx = runtime.Context(0)
    try:
        ctx.set_deterministic(True)
        ctx.load_window(win)
        outs["deterministic"], ran = fused_pass(ctx, failures, "deterministic")
        kernels["deterministic"] = ran & (ASSEMBLY_KERNELS | DET_KERNELS)
    finally:
        ctx.close()

    want = golden_facts(case, gidx, sms)
    got = shape_facts(case, gidx, maps[0], maps[1:], sms)
    for key in ("nv_mod", "pose_ctas", "imu_splits", "mixed_tiles", "eval_blocks"):
        record_property(f"{name}:{key}", got[key])
    record_property(f"{name}:runs", str(got["runs"]))
    if got != want:
        failures.append(f"bound index maps {got} != golden bases {want}")
    for pas, out in outs.items():
        bad, worst = pass_ratios(case, gidx, out)
        if bad:
            failures.append(f"{pas}: copies differ: {bad[:10]}")
        try:
            check(worst, record_property, f"{name}:{pas}")
        except AssertionError as e:
            failures.append(str(e))
    record_property(f"{name}:evaluate_fused_ulps", max(ulps(outs["evaluate"][k], outs["fused"][k]) for k in outs["evaluate"]))
    record_property(f"{name}:evaluate_fused_same_bits", all(same_bits(outs["evaluate"][k], outs["fused"][k]) for k in outs["evaluate"]))
    ref, own = cost_reference(case, win, gidx)
    ratio, _ = cost_ratio(cost, ref, own, device_cost_terms(win))
    record_property(f"{name}:cost_ratio", ratio)
    if not ratio <= 1.0:
        failures.append(f"cost {cost!r} vs {float(ref)!r}: {ratio:.3g} of its bound")
    expect = {"evaluate": p["kernels"] & EVAL_KERNELS, "fused": p["kernels"], "deterministic": det_kernels(p)}
    for pas, ran in kernels.items():
        record_property(f"{name}:kernels:{pas}", ",".join(sorted(ran)))
        if ran != expect[pas]:
            failures.append(f"{pas}: kernels {sorted(ran)} != plan {sorted(expect[pas])}")
    if shape != "S0":
        merged = bool(case["inertial"]) and shape in ("S1", "S2-merged")
        if p["merged"] != merged:
            failures.append(f"merged {p['merged']} != {merged}")
    assert not failures, "\n".join(failures)


@pytest.mark.gpu
@pytest.mark.parametrize("path", SPLINE_EDGES, ids=[os.path.basename(p) for p in SPLINE_EDGES])
def test_gpu_interpolate_many_stamps(built, path, record_property):
    """hb200_interpolate at the spline_edges stamps, shuffled and replicated past 64 SMs stamps: every copy of a stamp
    bit-identical, every row within interpolate_ratios' bound."""
    from hyperslam_b200 import runtime
    case = load(path)
    win, _ = replicate(case)
    gi = replicated_stamps(case, num_sms())
    stamps = np.array([a["stamp"] for a in case["interpolate"]])[gi]
    ctx = runtime.Context(0)
    try:
        ctx.load_window(win)
        pose, vel, acc, bad = ctx.interpolate(stamps)
    finally:
        ctx.close()
    assert bad == 0
    assert stamps.size > 64 * num_sms()
    _, first = np.unique(gi, return_index=True)
    for key, a in (("pose", pose), ("vel", vel), ("acc", acc)):
        bits = a.view(np.int64)
        differ = np.unique(gi[(bits != bits[first[gi]]).any(axis=1)])
        assert not differ.size, f"{key}: copies of stamps {differ.tolist()} differ"
    check(interpolate_ratios(dict(case, interpolate=[case["interpolate"][g] for g in gi]), pose, vel, acc), record_property,
          fixture_name(path))
