"""The captured LM iteration with the peer-memory reduction: one graph per arena half.

A one-rank NCCL communicator with the peer arena runs the two-graph path on one GPU.  The oracle is a context of the same
kind with use_graph off, which launches every iteration directly and so can never replay a stale graph.  Both contexts run
one call sequence in deterministic mode: iterations alternate with the setters that change what a captured iteration was
recorded with, and an odd number of iterations has run before each setter, so that arena half B runs first after it.
After every block of iterations the records, the cost and the state are bit-identical.

A change drops the graphs of both halves at once: one iteration, a change and three more iterations capture three graphs
(half A, then half B and half A again), counted from the HB200_GRAPH_DEBUG lines on stderr.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

from hyperslam_b200 import runtime, synthetic

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def window():
    return synthetic.make_config(1, constant_knots=2)


def peer_context(win, use_graph):
    """A deterministic context on a one-rank communicator with the peer arena; skips where NCCL cannot be loaded."""
    ctx = runtime.Context(0, use_graph=use_graph)
    try:
        uid = ctx.comm_unique_id()
    except runtime.HB200Error as e:
        ctx.close()
        if "libnccl" in str(e):
            pytest.skip(f"NCCL cannot be loaded: {e}")
        raise
    ctx.set_deterministic(True)
    ctx.load_window(win)
    ctx.comm_init_rank(1, 0, uid)
    ctx.peer_connect(1, 0, [ctx.peer_handle()])
    return ctx


def set_bearing_loss(ctx, huber):
    ctx._check(ctx.lib.hb200_set_bearing_loss(ctx.h, C.c_double(huber)))


def set_deterministic_off_on(ctx):
    ctx.set_deterministic(False)
    ctx.set_deterministic(True)


W_INERTIAL = np.diag([2.0, 2.0, 2.0, 0.5, 0.5, 0.5]) + 0.05 * np.triu(np.ones((6, 6)), 1)

# the setters between the blocks of iterations; each one drops the captured iterations
SETTERS = [
    ("set_options", lambda x, w: x.set_options(2 * w.huber_pixel, w.imu_loss_scale, 1e4)),
    ("set_bearing_loss", lambda x, w: set_bearing_loss(x, 2 * w.huber_bearing)),
    ("set_termination", lambda x, w: x.set_termination(1e-30, 1e-30, 1e-30, 1e-300)),
    ("set_weights", lambda x, w: x.set_weights(runtime.INERTIAL, W_INERTIAL)),
    ("set_deterministic off and on", lambda x, w: set_deterministic_off_on(x)),
]


def same_bits(a, b):
    a, b = np.ascontiguousarray(a, dtype=np.float64), np.ascontiguousarray(b, dtype=np.float64)
    return a.shape == b.shape and np.array_equal(a.view(np.int64), b.view(np.int64))


def test_two_halves_match_direct_launches(built):
    win = window()
    g = peer_context(win, use_graph=True)
    d = peer_context(win, use_graph=False)
    try:
        def step(name, iterations):
            rg, rd = g.iterate(iterations), d.iterate(iterations)
            assert same_bits([list(r.values()) for r in rg], [list(r.values()) for r in rd]), (name, rg, rd)
            assert same_bits(g.cost(), d.cost()), name
            sg, sd = g.state(), d.state()
            for key in sg:
                assert same_bits(sg[key], sd[key]), (name, key)

        step("start", 3)   # halves A, B, A: half B runs first after the next setter
        info = g.comm_info()
        assert info["peer_reduce"] and info["graph"], info
        assert d.comm_info()["peer_reduce"] and not d.comm_info()["graph"]
        for name, setter in SETTERS:
            setter(g, win)
            setter(d, win)
            step(name, 4)   # B, A, B, A: both fresh captures run and are replayed
    finally:
        g.close()
        d.close()


CAPTURE_SCRIPT = """
import sys
sys.path[:0] = [{root!r}, {tests!r}]
import test_gpu_iteration_graphs as t
ctx = t.peer_context(t.window(), use_graph=True)
ctx.iterate(1)
ctx.set_termination(1e-30, 1e-30, 1e-30, 1e-300)
ctx.iterate(3)
ctx.close()
"""


def test_a_change_drops_both_halves(built):
    peer_context(window(), use_graph=True).close()   # (skips where NCCL cannot be loaded)
    script = CAPTURE_SCRIPT.format(root=ROOT, tests=os.path.join(ROOT, "tests"))
    res = subprocess.run([sys.executable, "-c", script], cwd=ROOT, env=dict(os.environ, HB200_GRAPH_DEBUG="1"), capture_output=True,
                         text=True, timeout=300)
    assert res.returncode == 0, res.stderr[-4000:]
    captures = [line for line in res.stderr.splitlines() if line.startswith("[hb200] iteration graph")]
    assert len(captures) == 3, res.stderr[-4000:]
    assert [" (arena half B)" in line for line in captures] == [False, True, False], captures
