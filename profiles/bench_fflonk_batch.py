"""fflonk throughput: K sequential sb_fflonk_prove calls against one sb_fflonk_prove_batch call of K proofs, on the
synthetic chain keys (synth.synth_fflonk_zkey, BN254) at log2 n in {10, 12, 14, 16, 18}, K in {8, 32, 128}.  The library
splits a batch into sub-batches that fit in device memory, so every point runs.

A few distinct chain witnesses (the chain re-run from other x_0, which the same key accepts) are cycled with distinct
blinders; building them stays outside the timed window.  Every shape is warmed up (K sequential proofs and one batch of K)
before it is timed, the faster of --reps timed repetitions is reported, and every batch proof is checked against its
sequential proof.  One JSON line per point, with the card's name and power limit read in the same run:
  {"log_n", "K", "seq_ms", "batch_ms", "seq_proofs_per_s", "batch_proofs_per_s", "speedup", "gpu", "power_limit_w"}
Usage: python profiles/bench_fflonk_batch.py [--log-n 10,12] [--K 8,32] [--reps 2]"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from snarkjs_b200 import fflonk, getCurveFromName, synth  # noqa: E402
from profiles.bench_groth16_batch import card  # noqa: E402
from profiles.bench_plonk_batch import chain_witnesses  # noqa: E402

DISTINCT = 4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-n", default="10,12,14,16,18")
    ap.add_argument("--K", default="8,32,128")
    ap.add_argument("--reps", type=int, default=2)
    a = ap.parse_args()
    name, pl = card()
    curve = getCurveFromName("bn128")
    for log_n in [int(x) for x in a.log_n.split(",")]:
        zkey, base = synth.synth_fflonk_zkey(curve, log_n)
        pk = fflonk.ProvingKey(zkey, curve=curve)
        distinct = chain_witnesses(base, curve.r, DISTINCT)
        try:
            for K in [int(x) for x in a.K.split(",")]:
                ws = [distinct[i % DISTINCT] for i in range(K)]
                bls = [b"".join(fflonk.random_fr(curve) for _ in range(9)) for _ in range(K)]
                # warm-up of both shapes, and the check
                seq = [pk.prove_raw(w, b) for w, b in zip(ws, bls)]
                got = pk.prove_batch_raw(ws, bls)
                assert got == seq, (log_n, K, [i for i in range(K) if got[i] != seq[i]])
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
                print(json.dumps({"log_n": log_n, "K": K, "seq_ms": round(ts * 1e3, 3), "batch_ms": round(tb * 1e3, 3),
                                  "seq_proofs_per_s": round(K / ts, 2), "batch_proofs_per_s": round(K / tb, 2),
                                  "speedup": round(ts / tb, 3), "gpu": name, "power_limit_w": pl}), flush=True)
        finally:
            pk.release()
    curve.terminate()


if __name__ == "__main__":
    main()
