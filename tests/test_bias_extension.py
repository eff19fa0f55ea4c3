"""The bias-spline extension rule of hb200_append_bias_knots, restated on the host and checked against the oracle's bind.

To each bias spline the call appends the fewest knots that put a stamp inside the spline's valid span -- the span the
bind accepts (segment_base: the stamp's segment j must give kb control points, base = j - (kb-1)/2 >= 0 and
base + kb - 1 <= K - 1).  New knots follow hb200_append_knots: the new knots and the current last one take the value of
the second to last, and new stamp i is fma(i + 1, dt, last stamp) with dt the spline's last separation (one rounding,
as the device computes it).  The restatement below is what tests/test_gpu_bias_window.py checks the device against;
here it is checked against the oracle's segment_base, read through the gyro and accel base maps of an oracle window.
"""
import dataclasses
import math
from fractions import Fraction

import numpy as np

import oracle_lib as ol
from hyperslam_b200 import synthetic

MAX_APPEND = 1024   # HB200_BIAS_APPEND_MAX


def fma(a, b, c):
    """a * b + c rounded once (Python's int / int division rounds correctly)."""
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def extend(bias, count):
    """A bias spline [K][4] after appending `count` knots by the extrapolation rule."""
    out = np.array(bias, dtype=np.float64)
    if count == 0:
        return out
    s = out[:, 3]
    dt = s[-1] - s[-2]
    new = np.repeat(out[-2:-1], count, axis=0)
    new[:, 3] = [fma(float(i + 1), dt, s[-1]) for i in range(count)]
    out[-1, :3] = out[-2, :3]
    return np.vstack([out, new])


def valid(stamps, t, kb=4):
    """The valid span [s[left], s[K - right]) of a spline of order kb (left = (kb-1)/2 control points before the segment)."""
    left = (kb - 1) // 2
    right = kb - 1 - left
    return len(stamps) >= kb and stamps[left] <= t < stamps[len(stamps) - right]


def append_count(bias, t, kb=4):
    """Fewest knots that make t valid; None for a stamp before the span (the call never prepends) or past MAX_APPEND."""
    s = bias[:, 3]
    if not math.isfinite(t) or t < s[(kb - 1) // 2]:
        return None
    for most in (64, MAX_APPEND):   # new stamps depend on the original spline only: extend once, test every prefix
        full = extend(bias, most)[:, 3]
        for n in range(most + 1):
            if valid(full[:len(s) + n], t, kb):
                return n
    return None


def bias_base(stamps, t, kb=4):
    """Bias base of stamps t on a spline with the given knot stamps (segment_base for stamps inside the span)."""
    j = np.searchsorted(stamps, t, side="right") - 1
    return j - (kb - 1) // 2


def spline(rng, t0, sep, K=4):
    b = np.zeros((K, 4))
    b[:, :3] = rng.uniform(-0.05, 0.05, (K, 3))
    b[:, 3] = t0 + (np.arange(K) - 1) * sep
    return b


def oracle_bases(template, gyro, accel, stamps):
    win = dataclasses.replace(template, gyro_bias=gyro, accel_bias=accel, i_stamp=np.ascontiguousarray(stamps, dtype=np.float64),
                              i_meas=np.zeros((len(stamps), 6)))
    _, ib, ig, ia = ol.OracleWindow(win).index_maps()
    assert np.all(ib >= 0)   # the pose spline covers every stamp used here
    return ig, ia


def test_fewest_knots_agree_with_the_oracle_bind():
    template = synthetic.make_window(order=4, num_knots=600, num_landmarks=0, num_imu=0, seed=synthetic.SEED_BASE + 5100)
    rng = np.random.default_rng(5100)
    # gyro and accel with different separations (and an irrational-looking one, so that fma and a two-rounding
    # restatement differ for some new stamps)
    gyro, accel = spline(rng, 1.0, 0.7), spline(rng, 0.95, 1.1 / 3.0)   # valid spans start at 1.0 and 0.95
    stamps, kinds = [], []
    for b in (gyro, accel):
        s = b[:, 3]
        sep = s[-1] - s[-2]
        for n in range(8):
            end = extend(b, n)[len(b) + n - 2, 3]        # t_end of the spline with n knots appended
            stamps += [np.nextafter(end, -np.inf), end]  # last valid stamp (one ulp below t_end), t_end
        stamps += [s[-1] + j * sep for j in (1, 2, 3, 5, 8, 13)]   # several separations past
        stamps += [s[1], s[1] + 0.5 * sep]                        # inside: nothing appended
    stamps += list(rng.uniform(1.0, 1.0 + 20 * 0.7, 60))
    stamps = np.array(sorted(t for t in stamps if t >= 1.0))
    for t in stamps:
        ng, na = append_count(gyro, t), append_count(accel, t)
        assert ng is not None and na is not None, t
        ig, ia = oracle_bases(template, extend(gyro, ng), extend(accel, na), [t])
        assert ig[0] >= 0 and ia[0] >= 0, (t, ng, na)
        assert ig[0] == bias_base(extend(gyro, ng)[:, 3], t) and ia[0] == bias_base(extend(accel, na)[:, 3], t), t
        if ng:
            g1, _ = oracle_bases(template, extend(gyro, ng - 1), extend(accel, na), [t])
            assert g1[0] < 0, (t, ng)
        if na:
            _, a1 = oracle_bases(template, extend(gyro, ng), extend(accel, na - 1), [t])
            assert a1[0] < 0, (t, na)
        kinds.append((ng > 0, na > 0))
    assert (False, False) in kinds and (True, True) in kinds
    # the gyro and accel counts differ for some stamps: the splines are extended independently
    assert any(append_count(gyro, t) != append_count(accel, t) for t in stamps)


def test_extrapolation_values_and_rejections():
    rng = np.random.default_rng(5101)
    b = spline(rng, 2.0, 1.1 / 3.0, K=6)
    e = extend(b, 5)
    assert np.array_equal(e[:5], b[:5]) and np.array_equal(e[5, :3], b[4, :3]) and e[5, 3] == b[5, 3]
    assert np.all(e[6:, :3] == b[4, :3])
    dt = b[5, 3] - b[4, 3]
    assert all(e[6 + i, 3] == fma(float(i + 1), dt, b[5, 3]) for i in range(5))
    assert np.all(np.diff(e[:, 3]) > 0)
    # before the span, non-finite, and too far for one call
    assert append_count(b, np.nextafter(b[1, 3], -np.inf)) is None and append_count(b, b[1, 3]) == 0
    assert append_count(b, float("nan")) is None and append_count(b, float("inf")) is None
    assert append_count(b, b[-1, 3] + (MAX_APPEND - 1.5) * dt) == MAX_APPEND
    assert append_count(b, b[-1, 3] + (MAX_APPEND + 1) * dt) is None
