"""Phase timeline of bcr_solve_kernel (CTA 0, globaltimer ns) for a large config: HB200_CFG=2|3|4."""
import ctypes as C
import os
import sys

os.environ["HB200_BAND_TIMING"] = "1"
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from hyperslam_b200 import runtime, synthetic

cfg = int(os.environ.get("HB200_CFG", "3"))
win = synthetic.make_config(cfg, scale=float(os.environ.get("HB200_SCALE", "0.05")), constant_knots=2)
ctx = runtime.Context(0)
ctx.load_window(win)
ctx.iterate(2)
ctx.synchronize()
buf = (C.c_longlong * 144)()
ctx.lib.hb200_debug_band_timing(ctx.h, buf)
n = buf[0]
t = [buf[1 + i] for i in range(n)]
print("cfg", cfg, "K", win.knots.shape[0], "beta", ctx.bandwidth(), "stamps", n)
labels = ["gather"]
print("total us", (t[-1] - t[0]) / 1e3)
print("level-0 phase 1 of CTA 0 (us): stage, chol, forward, stores, gram(warp 0), gram barrier, corner share + loop end:",
      [round((t[i + 1] - t[i]) / 1e3, 2) for i in range(2, 9)])
t = t[:3] + t[9:]
d = [round((b - a) / 1e3, 1) for a, b in zip(t[:-1], t[1:])]
print("work / barrier-wait pairs (us):", list(zip(d[0::2], d[1::2])))
print("sum work", round(sum(d[0::2]), 1), "sum barrier", round(sum(d[1::2]), 1))
for name, ms in ctx.profile_iteration(reps=3):
    if "solve" in name:
        print(name, ms * 1e3, "us")
