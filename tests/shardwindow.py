"""Restatement of the agreement that a sharded window's collective sliding-window calls run (hb200_window.cuh:
window_vote_kernel, window_agree_kernel): every rank's payload of doubles, its sum over the ranks, and what every rank
reads from the sum.  Plain numpy, written from the rules in include/hyperb200.h's SHARDING CONTRACT, not from the kernels.

Payload: [header 9 | header squared 9 | status 2 | smallest kept knot base K | gyro bias base Kbg | accel bias base Kba |
beta K]; the header (1, K, Kbg, Kba, call kind, slide flags, ub, ubg, uba) and its squares must sum to nranks times each
rank's own (both together: every rank holds the same header), the status slots count the ranks whose own checks failed
(bad index, else arrival order), and the votes are one-hot."""
import numpy as np

HEADER, STATUS = 9, 2
HEAD = 2 * HEADER + STATUS   # votes start here
NO_VOTE = 0x7fffffff


def payload(K, Kbg, Kba, header, status=(0, 0), knot_min=None, bias_min=(None, None), beta=None):
    """One rank's payload.  None (or NO_VOTE): no vote -- the rank holds no factor of that family."""
    p = np.zeros(HEAD + 2 * K + Kbg + Kba)
    h = np.asarray(header, dtype=float)
    p[:HEADER], p[HEADER:2 * HEADER] = h, h * h
    p[2 * HEADER] = 1.0 if status[0] else 0.0
    p[2 * HEADER + 1] = 1.0 if not status[0] and status[1] else 0.0
    votes = p[HEAD:]
    for off, n, v in ((0, K, knot_min), (K, Kbg, bias_min[0]), (K + Kbg, Kba, bias_min[1]), (K + Kbg + Kba, K, beta)):
        if v is not None and v != NO_VOTE and n > 0:
            votes[off + min(max(int(v), 0), n - 1)] = 1.0
    return p


def agree(total, K, Kbg, Kba, header):
    """What every rank reads from the summed payload (its own header to compare against)."""
    votes = total[HEAD:]
    h = np.asarray(header, dtype=float)

    def first(a):
        nz = np.flatnonzero(a)
        return int(nz[0]) if nz.size else NO_VOTE
    beta = np.flatnonzero(votes[K + Kbg + Kba:])
    return dict(status=2 if total[2 * HEADER] > 0 else (3 if total[2 * HEADER + 1] > 0 else 0),
                mismatch=bool(np.any(total[:HEADER] != total[0] * h) or np.any(total[HEADER:2 * HEADER] != total[0] * h * h)),
                beta=int(beta[-1]) if beta.size else 0, knot_min=first(votes[:K]), gyro_min=first(votes[K:K + Kbg]),
                accel_min=first(votes[K + Kbg:K + Kbg + Kba]))


def summed(payloads):
    """The rank-order float64 sum every channel (NCCL, peer memory, the hook) computes."""
    total = np.zeros_like(payloads[0])
    for p in payloads:
        total = total + p
    return total


def knot_shift(begin, knot_min, K, k):
    return max(0, min(min(begin, knot_min), K - k))


def bias_shift(stamps, lower, bias_min, kb):
    ub = int(np.searchsorted(stamps, lower, side="right"))
    return max(0, min(min(max(0, ub - 1 - (kb - 1) // 2), bias_min), len(stamps) - kb))


def own_beta(k, bases_by_landmark):
    """A rank's own band half-width vote: the longest landmark track in control points, at least k - 1 (None: no
    visual factor, no vote)."""
    if not bases_by_landmark:
        return None
    return max(k - 1, max(max(b) - min(b) + k - 1 for b in bases_by_landmark.values()))
