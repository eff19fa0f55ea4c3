import os, sys, ctypes as C
os.environ["HB200_BAND_TIMING"]="1"
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from hyperslam_b200 import runtime, synthetic
win = synthetic.make_config(int(os.environ.get("HB200_CFG", "1")), constant_knots=2)
ctx = runtime.Context(0); ctx.load_window(win)
ctx.iterate(1)
cyc = (C.c_longlong*72)()
ctx.lib.hb200_debug_band_timing(ctx.h, cyc)
names=["potf2 prologue","two-sided factorisation","merge + separator columns","block inverses + deferred corner update","corner Cholesky","corner back substitution","outward back substitution","arrow pre-pass + row transform"]
tot=sum(cyc[0:8])
for n,c in zip(names,cyc): print(f"{n:40s} {c:9d} cycles {c/1.965e3:8.1f} us {100*c/max(tot,1):5.1f}%")


print("chain 0, steps 4..11: cycles relative to the update warp's release (B of the previous step)")
print("step  panel_end  A_release  upd_end | la_release  la_end | next_release")
for i in range(8):
    r = cyc[8+8*i:8+8*i+6]
    nxt = cyc[8+8*(i+1)] if i < 7 else 0
    b = r[0]
    print(f"{i+4:4d} {r[1]-b:9d} {r[2]-b:9d} {r[3]-b:8d} | {r[4]-b:9d} {r[5]-b:8d} | {(nxt-b) if nxt else 0:9d}")

print("TOTAL cycles", tot, "us", tot/1.965e3)
print(f"before the first tick: staging (damping, mask) {cyc[14]} cycles {cyc[14]/1.965e3:.1f} us, gather {cyc[15]} cycles {cyc[15]/1.965e3:.1f} us; kernel entry -> exit {cyc[22]} cycles {cyc[22]/1.965e3:.1f} us")

print("gather split (thread 0): chain-0 band", cyc[23], "chain-1 band", cyc[30], "chain-0 arrow", cyc[31], "chain-1 arrow", cyc[38], "corner + barrier", cyc[39])
