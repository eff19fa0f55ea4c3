import os, sys, ctypes as C
os.environ["HB200_BAND_TIMING"]="1"
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
from hyperslam_b200 import runtime, synthetic
win = synthetic.make_config(int(os.environ.get("HB200_CFG", "1")), constant_knots=2)
ctx = runtime.Context(0); ctx.load_window(win)
ctx.iterate(1)
hz = torch.cuda.get_device_properties(0).clock_rate * 1e3   # SM clock of this device (clock_rate is in kHz)
print(f"{torch.cuda.get_device_name(0)}: SM clock {hz / 1e9:.3f} GHz")
us = lambda c: c / (hz / 1e6)
buf = (C.c_longlong*144)()
ctx.lib.hb200_debug_band_timing(ctx.h, buf)
# the resident solver runs chain r on CTA r of a 2-CTA cluster; each CTA records its own phases (72 values each)
names = {0: ["potf2 prologue", "two-sided factorisation (chain 0)", "wait for CTA 1 (barrier 1), merge + separator columns",
             "own corner update + panel-row transform", "wait for CTA 1 (barrier 2), its corner partial, corner Cholesky",
             "corner back subst., arrow pre-pass, rhs transform, separator back subst., stores to CTA 1", "outward back substitution", "-"],
         1: ["potf2 prologue", "two-sided factorisation (chain 1)", "separator copy to CTA 0 (barrier 1)",
             "own corner partial + panel-row transform", "wait for CTA 0 (barrier 2)", "wait for CTA 0 (corner and separator solutions)",
             "outward back substitution", "arrow pre-pass + rhs transform"]}
for r in (0, 1):
    cyc = buf[72 * r:72 * (r + 1)]
    if r > 0 and cyc[22] == 0:
        break   # single-CTA kernel (chunked workspace)
    print(f"==== CTA {r}" + (f" (SPD flag of the solve: {cyc[70]})" if r == 0 else ""))
    tot=sum(cyc[0:8])
    for n,c in zip(names[r],cyc): print(f"{n:72s} {c:9d} cycles {us(c):8.1f} us {100*c/max(tot,1):5.1f}%")
    print(f"chain {r}, steps 4..11: cycles relative to the update warp's release (B of the previous step)")
    print("step  panel_end  A_release  upd_end | la_release  la_end | next_release")
    for i in range(8):
        s = cyc[8+8*i:8+8*i+6]
        nxt = cyc[8+8*(i+1)] if i < 7 else 0
        b = s[0]
        print(f"{i+4:4d} {s[1]-b:9d} {s[2]-b:9d} {s[3]-b:8d} | {s[4]-b:9d} {s[5]-b:8d} | {(nxt-b) if nxt else 0:9d}")
    print("TOTAL cycles", tot, "us", us(tot))
    print(f"before the first tick: staging (damping, mask) {cyc[14]} cycles {us(cyc[14]):.1f} us, gather {cyc[15]} cycles {us(cyc[15]):.1f} us; kernel entry -> exit {cyc[22]} cycles {us(cyc[22]):.1f} us")
    print("gather split (thread 0): chain-0 band", cyc[23], "chain-1 band", cyc[30], "chain-0 arrow", cyc[31], "chain-1 arrow", cyc[38], "corner + barrier", cyc[39])
