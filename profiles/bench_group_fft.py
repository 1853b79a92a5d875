#!/usr/bin/env python
"""Device time of the group iFFT (G1/G2.ifft, csrc/gfft.cuh) per (curve, group, log2 n), and what it implies for
`powersoftau prepare phase2`.  Prints one JSON line:
  * per case: device ms of the transform kernels (sb_last_ms 2: twiddles, load, stages, inverse scale, store), the
    scalar-multiplication count (n/2)(log2 n - 1) + n, the base-field (Fq) multiplies they take by the operation counts
    below, and the implied Fq-multiply rate;
  * projected prepare-phase2 time at powers 20 and 24: the sum over its blocks (section 12: 2^0..2^(power+1) G1 points,
    13: 2^0..2^power G2, 14 and 15: 2^0..2^power G1) of scalar multiplications times the measured time per scalar
    multiplication at the nearest measured size (blocks below 2^16 use the 2^16 rate, above 2^20 the 2^20 rate);
  * the card name and power limit, read in the same run;
  * the CPU oracle's time for the same iFFT at 2^12 on BN254 G1: the C++/OpenMP restatement in tests/host/group_fft_oracle.cpp
    (built on oracle/), not snarkjs' Node+WASM path.
Usage: python profiles/bench_group_fft.py [--logs 16,18,20] [--pairs bn128:1,bn128:2,bls12381:1,bls12381:2]"""
import argparse
import ctypes
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# Fq multiplies (squarings counted as multiplies) of the XYZZ formulas in ec.cuh: dbl 6M + 3S, add 12M + 2S; an Fp2
# multiply is 3 Fq multiplies (Karatsuba) and an Fp2 squaring 2.  gfft_mul: table 1 dbl + 6 add, then 252 doublings
# and ~60 additions (64 signed 4-bit digits, 15 in 16 of them non-zero for uniform scalars).
FQ_MULS = {1: {"dbl": 9, "add": 14}, 2: {"dbl": 6 * 3 + 3 * 2, "add": 12 * 3 + 2 * 2}}


def smul_count(L):
    n = 1 << L
    return (n // 2) * max(L - 1, 0) + n


def fq_muls(grp, L):
    c = FQ_MULS[grp]
    per_smul = 253 * c["dbl"] + 66 * c["add"]
    n = 1 << L
    return smul_count(L) * per_smul + (n // 2) * L * 2 * c["add"]   # + the two additions of every butterfly


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=60).stdout.strip().splitlines()
        name, plim = [x.strip() for x in out[0].split(",")]
        return {"gpu": name, "power_limit": plim}
    except Exception as e:   # the numbers still print; the card is then unknown
        return {"gpu": f"unknown ({e})", "power_limit": "unknown"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--logs", default="16,18,20")
    ap.add_argument("--pairs", default="bn128:1,bn128:2,bls12381:1,bls12381:2")
    ap.add_argument("--no-cpu", action="store_true")
    a = ap.parse_args()
    import snarkjs_b200
    logs = [int(x) for x in a.logs.split(",")]
    res = {"metric": "group_ifft_device_ms", **card(), "cases": [], "projected_prepare_phase2_s": {}}
    per_smul = {}
    for pair in a.pairs.split(","):
        name, grp = pair.split(":")
        grp = int(grp)
        c = snarkjs_b200.getCurveFromName(name)
        G = c.G1 if grp == 1 else c.G2
        nmax = 1 << max(logs)
        x = np.empty(nmax * 2 * G.n8, np.uint8)
        c.check(c.lib.sb_gen_points(c.handle, grp, 1, nmax, x.ctypes.data_as(ctypes.c_void_p)))
        G.ifft(x[:1024 * 2 * G.n8])                       # warm-up: module load, twiddle tables
        for L in logs:
            G.ifft(x[:(1 << L) * 2 * G.n8])
            ms = c.last_ms(2)
            ops = fq_muls(grp, L)
            res["cases"].append({"curve": name, "group": grp, "log2n": L, "device_ms": round(ms, 3),
                                 "total_ms": round(c.last_ms(0), 3), "scalar_muls": smul_count(L), "fq_muls": ops,
                                 "fq_muls_per_s": ops / (ms * 1e-3)})
            per_smul[(name, grp, L)] = ms * 1e-3 / smul_count(L)
        c.terminate()

    def rate(name, grp, p):
        ms = [L for L in logs if (name, grp, L) in per_smul]
        L = min(ms, key=lambda L: abs(L - p)) if ms else None
        return per_smul.get((name, grp, L))

    for name in sorted({k[0] for k in per_smul}):
        for power in (20, 24):
            t, ok = 0.0, True
            for grp, top in ((1, power + 1), (2, power), (1, power), (1, power)):
                for p in range(top + 1):
                    r = rate(name, grp, p)
                    if r is None:
                        ok = False
                        break
                    t += smul_count(p) * r
            if ok:
                res["projected_prepare_phase2_s"][f"{name}_power{power}"] = round(t, 1)
    if not a.no_cpu:
        from oracle import oracle as O
        from tests import gfft_oracle as GO
        xs = O.gen_points(O.BN254, 1, 1, 1 << 12)
        t0 = time.perf_counter()
        GO.group_fft(O.BN254, 1, xs, inverse=True)
        res["cpu_oracle_cxx_restatement"] = {"case": "bn128 G1 ifft 2^12", "ms": round((time.perf_counter() - t0) * 1e3, 1),
                                             "threads": int(O.lib().or_num_threads())}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
