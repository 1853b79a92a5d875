"""Rates of the FP64 pipe next to the integer path (sb_calibrate what = 1..4)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import snarkjs_b200
c = snarkjs_b200.getCurveFromName("bn128")
f = lambda w: c.lib.sb_calibrate(c.handle, w)
sm, clk = 132, 1.98e9   # H100 SXM: SMs, maximum SM clock
mod, dfma, lp, lp_mixed = f(1), f(2), f(3), f(4)
print(f"modmul (IMAD path)        {mod:.3e}/s  = {mod / sm / clk:.3f} per clk per SM")
print(f"DFMA (8 chains/thread)    {dfma:.3e}/s  = {dfma / sm / clk:.1f} per clk per SM")
print(f"52-bit limb products      {lp:.3e}/s  = {lp / sm / clk:.2f} per clk per SM  -> /55 = {lp / 55:.3e} modmul-equivalents/s")
print(f"limb products on half the warps while the other half runs IMAD modmuls: {lp_mixed:.3e}/s (alone at half the warps would be ~{lp / 2:.3e})")
