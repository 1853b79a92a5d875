"""Groth16 throughput: K sequential sb_groth16_prove calls against one sb_groth16_prove_batch call of K proofs, on the
synthetic chain keys (synth.synth_groth16_zkey) at L in {10, 12, 14, 16, 18, 20} on BN254 and {12, 16} on BLS12-381,
K in {8, 32, 128}.  The library splits a batch into sub-batches that fit in device memory, so every point runs.

Every shape is warmed up (one sequential proof and one batch of K) before it is timed, and the faster of --reps timed
repetitions is reported; every batch proof is checked against its sequential proof.  One JSON line per point, with the card's name and power limit read in the same run:
  {"curve", "L", "K", "seq_ms", "batch_ms", "seq_proofs_per_s", "batch_proofs_per_s", "speedup", "gpu", "power_limit_w"}
Usage: python profiles/bench_groth16_batch.py [--curves bn128,bls12381] [--L 10,12] [--K 8,32] [--reps 2]"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from snarkjs_b200 import getCurveFromName, groth16, synth  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, pl = [x.strip() for x in out.split(",")]
        return name, float(pl.split()[0])
    except Exception as e:   # the numbers stay meaningless without the card: say so in the line
        return f"unknown ({e})", None


def witnesses(curve, L, K):
    base = synth.chain_witness(curve.r, L)
    # distinct witnesses without K Python chain evaluations: the same digit distribution, other values
    return [base] + [synth.witness_like(base, seed=i) for i in range(1, K)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--curves", default="bn128,bls12381")
    ap.add_argument("--L", default="")
    ap.add_argument("--K", default="8,32,128")
    ap.add_argument("--reps", type=int, default=2)
    a = ap.parse_args()
    name, pl = card()
    Ls = {"bn128": [10, 12, 14, 16, 18, 20], "bls12381": [12, 16]}
    for cname in a.curves.split(","):
        curve = getCurveFromName(cname)
        for L in ([int(x) for x in a.L.split(",")] if a.L else Ls[cname]):
            zkey = synth.synth_groth16_zkey(curve, L)
            pk = groth16.ProvingKey(zkey, curve=curve)
            try:
                for K in [int(x) for x in a.K.split(",")]:
                    ws = witnesses(curve, L, K)
                    rs = [(groth16.random_fr(curve), groth16.random_fr(curve)) for _ in range(K)]
                    wcat = np.concatenate(ws)
                    # warm-up of both shapes, and the check
                    seq = [pk.prove_raw(w, r, s) for w, (r, s) in zip(ws, rs)]
                    got = pk.prove_batch_raw(wcat, rs)
                    assert got == seq, (cname, L, K, [i for i in range(K) if got[i] != seq[i]])
                    t_seq, t_bat = [], []
                    for _ in range(a.reps):
                        t0 = time.perf_counter()
                        for w, (r, s) in zip(ws, rs):
                            pk.prove_raw(w, r, s)
                        t_seq.append(time.perf_counter() - t0)
                        t0 = time.perf_counter()
                        pk.prove_batch_raw(wcat, rs)
                        t_bat.append(time.perf_counter() - t0)
                    ts, tb = min(t_seq), min(t_bat)
                    print(json.dumps({"curve": cname, "L": L, "K": K, "seq_ms": round(ts * 1e3, 3), "batch_ms": round(tb * 1e3, 3),
                                      "seq_proofs_per_s": round(K / ts, 2), "batch_proofs_per_s": round(K / tb, 2),
                                      "speedup": round(ts / tb, 3), "gpu": name, "power_limit_w": pl}), flush=True)
            finally:
                pk.release()
        curve.terminate()


if __name__ == "__main__":
    main()
