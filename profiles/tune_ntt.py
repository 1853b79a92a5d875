"""Primitive-level timings on one GPU (BASELINE.json configs #2 and #3): BN254 G1/G2 MSM at 2^20 and Fr NTT/iNTT at
2^20..2^24, device-resident (CUDA events inside the library) and through the host-buffer C ABI calls."""
import ctypes, json, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import snarkjs_b200
from snarkjs_b200 import synth
from snarkjs_b200.curve import _ptr
c = snarkjs_b200.getCurveFromName("bn128")
lib, h = c.lib, c.handle
out = {}
rng = np.random.default_rng(3)
n = 1 << 20
sc = rng.integers(0, 256, size=n * 32, dtype=np.uint8); sc.reshape(n, 32)[:, 31] &= 0x1f
for grp in ():
    G = c.G1 if grp == 1 else c.G2
    bases = synth.gen_points(c, grp, 7, n)
    # plain call, host buffers both ways (the drop-in multiExpAffine)
    for _ in range(2): G.multiExpAffine(bases, sc)
    t = time.perf_counter(); reps = 5
    for _ in range(reps): G.multiExpAffine(bases, sc)
    dt_host = (time.perf_counter() - t) / reps
    dev_plain = c.last_ms(2)
    hb = G.registerBases(bases)
    for _ in range(2): G.multiExpRegistered(hb, sc)
    t = time.perf_counter()
    for _ in range(reps): G.multiExpRegistered(hb, sc)
    dt_reg = (time.perf_counter() - t) / reps
    dev_reg = c.last_ms(2)
    out[f"msm_g{grp}_2^20"] = {"multiExpAffine_host_buffers_ms": dt_host * 1e3, "device_ms_plain_windows": dev_plain,
                               "registered_bases_host_scalars_ms": dt_reg * 1e3, "device_ms_table_mode": dev_reg,
                               "Mop_per_s_table_mode_device": n / dev_reg / 1e3, "Mop_per_s_plain_device": n / dev_plain / 1e3}
for tile in (12, 11, 10):
  lib.sb_set_tuning(7, tile)
  for L in (20, 24):
      m = 1 << L
      x = rng.integers(0, 256, size=m * 32, dtype=np.uint8); x.reshape(m, 32)[:, 31] &= 0x1f
      a = lib.sb_dev_alloc(h, m * 32); b = lib.sb_dev_alloc(h, m * 32)
      lib.sb_dev_upload(h, a, _ptr(x), m * 32)
      res = ctypes.c_void_p()
      for inv in (0, 1):
          for _ in range(3): lib.sb_ntt_fr_dev(h, a, b, m, inv, ctypes.byref(res))
          ms = c.last_ms(0)
          muls = m * L / 2 + (m if inv else 0)
          out[f"tile{tile}_ntt_2^{L}_{'inv' if inv else 'fwd'}"] = {"device_ms": ms, "GB_per_s_algorithmic(1r+1w)": 2 * 32 * m / ms / 1e6,
                                                       "G_butterfly_modmul_per_s": muls / ms / 1e6}
      t = time.perf_counter(); y = c.Fr.fft(x); dt = time.perf_counter() - t
      out[f"tile{tile}_ntt_2^{L}_fwd"]["host_buffers_ms"] = dt * 1e3
      lib.sb_dev_free(h, a); lib.sb_dev_free(h, b)
print(json.dumps(out, indent=1))
