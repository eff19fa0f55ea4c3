import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from hyperslam_b200 import runtime, synthetic
win = synthetic.make_config(1, constant_knots=2)
for graph in (True, False):
    ctx = runtime.Context(0, use_graph=graph); ctx.load_window(win)
    st = torch.cuda.ExternalStream(ctx.stream_handle()) if hasattr(ctx, "stream_handle") else None
    ctx.snapshot()
    for name, fn in (("evaluate(J)", lambda: ctx.evaluate(True)), ("iterate(1)", lambda: ctx.iterate(1))):
        for _ in range(20): fn()
        ctx.synchronize()
        t0 = time.perf_counter()
        n = 300
        for _ in range(n):
            fn()
        ctx.synchronize()
        print(f"graph={graph} fork={'off' if os.environ.get('HB200_NO_FORK') else 'on'} {name}: {(time.perf_counter()-t0)/n*1e6:.1f} us/call (host wall, back-to-back)")
