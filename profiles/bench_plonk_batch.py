"""PLONK throughput: K sequential sb_plonk_prove calls against one sb_plonk_prove_batch call of K proofs, on the synthetic
chain keys (synth.synth_plonk_zkey) at log2 n in {10, 12, 14, 16, 18} on BN254 and BLS12-381, K in {8, 32, 128}.  The
library splits a batch into sub-batches that fit in device memory, so every point runs.

A few distinct chain witnesses (the chain re-run from other x_0, which the same key accepts) are cycled with distinct
blinders; building them stays outside the timed window.  Every shape is warmed up (K sequential proofs and one batch of K)
before it is timed, the faster of --reps timed repetitions is reported, and every batch proof is checked against its
sequential proof.  One JSON line per point, with the card's name and power limit read in the same run:
  {"curve", "log_n", "K", "seq_ms", "batch_ms", "seq_proofs_per_s", "batch_proofs_per_s", "speedup", "gpu", "power_limit_w"}
Usage: python profiles/bench_plonk_batch.py [--curves bn128,bls12381] [--log-n 10,12] [--K 8,32] [--reps 2]"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from snarkjs_b200 import getCurveFromName, plonk, synth  # noqa: E402
from profiles.bench_groth16_batch import card  # noqa: E402

DISTINCT = 4


def chain_witnesses(base: np.ndarray, r: int, count: int):
    """base = [1, x_m, x_0, ..., x_{m-1}] (32-byte LE); the chain x_{i+1} = x_i^2 + c re-run from other x_0."""
    w = [int.from_bytes(base[32 * i:32 * (i + 1)].tobytes(), "little") for i in range(base.size // 32)]
    m = len(w) - 2
    cst = (w[3] - w[2] * w[2]) % r
    out = [base]
    for t in range(1, count):
        x = [(w[2] + 1000 * t + 1) % r]
        for _ in range(m):
            x.append((x[-1] * x[-1] + cst) % r)
        out.append(np.frombuffer(b"".join(v.to_bytes(32, "little") for v in [1, x[m]] + x[:m]), np.uint8))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--curves", default="bn128,bls12381")
    ap.add_argument("--log-n", default="10,12,14,16,18")
    ap.add_argument("--K", default="8,32,128")
    ap.add_argument("--reps", type=int, default=2)
    a = ap.parse_args()
    name, pl = card()
    for cname in a.curves.split(","):
        curve = getCurveFromName(cname)
        for log_n in [int(x) for x in a.log_n.split(",")]:
            zkey, base = synth.synth_plonk_zkey(curve, log_n)
            pk = plonk.ProvingKey(zkey, curve=curve)
            distinct = chain_witnesses(base, curve.r, DISTINCT)
            try:
                for K in [int(x) for x in a.K.split(",")]:
                    ws = [distinct[i % DISTINCT] for i in range(K)]
                    bls = [b"".join(plonk.random_fr(curve) for _ in range(11)) for _ in range(K)]
                    # warm-up of both shapes, and the check
                    seq = [pk.prove_raw(w, b) for w, b in zip(ws, bls)]
                    got = pk.prove_batch_raw(ws, bls)
                    assert got == seq, (cname, log_n, K, [i for i in range(K) if got[i] != seq[i]])
                    t_seq, t_bat = [], []
                    for _ in range(a.reps):
                        t0 = time.perf_counter()
                        for w, b in zip(ws, bls):
                            pk.prove_raw(w, b)
                        t_seq.append(time.perf_counter() - t0)
                        t0 = time.perf_counter()
                        pk.prove_batch_raw(ws, bls)
                        t_bat.append(time.perf_counter() - t0)
                    ts, tb = min(t_seq), min(t_bat)
                    print(json.dumps({"curve": cname, "log_n": log_n, "K": K, "seq_ms": round(ts * 1e3, 3), "batch_ms": round(tb * 1e3, 3),
                                      "seq_proofs_per_s": round(K / ts, 2), "batch_proofs_per_s": round(K / tb, 2),
                                      "speedup": round(ts / tb, 3), "gpu": name, "power_limit_w": pl}), flush=True)
            finally:
                pk.release()
        curve.terminate()


if __name__ == "__main__":
    main()
