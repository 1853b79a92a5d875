"""Batch throughput over N GPUs: one sb_*_prove_batch_multi call of N x K proofs on N contexts, one per device, for
N in {1, 2, 4, 8} up to the devices present.  Workloads: Groth16 BN254 on the synthetic chain keys at 2^16 (K = 64) and
2^20 (K = 16), PLONK BLS12-381 and fflonk BN254 on the synthetic chain keys at 2^16 (K = 64).

Every (workload, N) is warmed up with one call and timed as the best of --reps calls; the rate is N x K over
sb_last_ms(ctxs[0], 0), the host wall clock of the whole call, and every rank's own batch time (sb_last_ms(ctxs[i], 0)) is
reported beside it, which shows imbalance between ranks.  "ideal" is N x the N = 1 rate.  At the largest N the timed proofs
are checked against one context's sb_*_prove_batch of the same inputs.  One JSON line per point, with the card's name, power
limit and max SM clock read in the same run:
  {"workload", "N", "count", "ms", "proofs_per_s", "ideal_proofs_per_s", "scaling", "rank_ms", "checked", "gpu",
   "power_limit_w", "max_sm_mhz"}
Usage: python profiles/bench_batch_multi.py [--workloads groth16-bn-16,groth16-bn-20,plonk-bls-16,fflonk-bn-16] [--N 1,2,4,8] [--reps 3]"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from snarkjs_b200 import fflonk, getCurveFromName, groth16, plonk, synth  # noqa: E402

# name: (protocol, curve, log2 of the domain, proofs per GPU)
WORKLOADS = {"groth16-bn-16": ("groth16", "bn128", 16, 64), "groth16-bn-20": ("groth16", "bn128", 20, 16),
             "plonk-bls-16": ("plonk", "bls12381", 16, 64), "fflonk-bn-16": ("fflonk", "bn128", 16, 64)}
MODULES = {"groth16": groth16, "plonk": plonk, "fflonk": fflonk}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl, sm = [x.strip() for x in out.split(",")]
        return name, float(pl.split()[0]), float(sm.split()[0])
    except Exception as e:   # the numbers stay meaningless without the card: say so in the line
        return f"unknown ({e})", None, None


def inputs(proto, curve, L, count):
    """(zkey, witnesses, randomness) of count proofs"""
    if proto == "groth16":
        zkey = synth.synth_groth16_zkey(curve, L)
        base = synth.chain_witness(curve.r, L)
        # distinct witnesses without count Python chain evaluations: the same digit distribution, other values
        ws = [base] + [synth.witness_like(base, seed=i) for i in range(1, count)]
        return zkey, ws, [(groth16.random_fr(curve), groth16.random_fr(curve)) for _ in range(count)]
    zkey, wit = (synth.synth_plonk_zkey if proto == "plonk" else synth.synth_fflonk_zkey)(curve, L)
    w = np.asarray(wit).reshape(-1).view(np.uint8)
    nb = 11 if proto == "plonk" else 9
    return zkey, [w] * count, [b"".join(groth16.random_fr(curve) for _ in range(nb)) for _ in range(count)]


def main():
    import torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--N", default="1,2,4,8")
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    nd = torch.cuda.device_count()
    if nd < 1:
        raise SystemExit("no CUDA device")
    name, pl, sm = card()
    Ns = [n for n in (int(x) for x in a.N.split(",")) if n <= nd]
    for wl in a.workloads.split(","):
        proto, cname, L, per = WORKLOADS[wl]
        M = MODULES[proto]
        curves = [getCurveFromName(cname, d) for d in range(max(Ns))]
        zkey, ws, rand = inputs(proto, curves[0], L, per * max(Ns))
        rate1 = None
        try:
            for n in Ns:
                count = n * per
                rk = M.ReplicatedProvingKey(zkey, curves[:n])
                try:
                    rk.prove_batch_raw(ws[:count], rand[:count])                            # warm-up
                    best, best_ranks, got = None, None, None
                    for _ in range(a.reps):
                        got = rk.prove_batch_raw(ws[:count], rand[:count])
                        ms = curves[0].last_ms(0)
                        if best is None or ms < best:
                            best, best_ranks = ms, [curves[i].last_ms(0) for i in range(1, n)]
                finally:
                    rk.release()
                checked = None
                if n == max(Ns):
                    pk = M.ProvingKey(zkey, curves[0])
                    try:
                        checked = pk.prove_batch_raw(ws[:count], rand[:count]) == got
                    finally:
                        pk.release()
                    assert checked, (wl, n)
                rate = count / (best / 1e3)
                rate1 = rate1 or (rate if n == 1 else None)
                ideal = n * rate1 if rate1 else None
                print(json.dumps({"workload": wl, "N": n, "count": count, "ms": round(best, 2), "proofs_per_s": round(rate, 2),
                                  "ideal_proofs_per_s": round(ideal, 2) if ideal else None,
                                  "scaling": round(rate / ideal, 3) if ideal else None,
                                  "rank_ms": [None] + [round(t, 2) for t in best_ranks], "checked": checked,
                                  "gpu": name, "power_limit_w": pl, "max_sm_mhz": sm}), flush=True)
        finally:
            for c in curves:
                c.terminate()


if __name__ == "__main__":
    main()
