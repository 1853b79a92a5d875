"""One proof on several contexts: sb_plonk_prove / sb_fflonk_prove against sb_plonk_prove_multi / sb_fflonk_prove_multi on
the synthetic chain keys (synth.synth_plonk_zkey / synth_fflonk_zkey) at log2 n in {16, 18, 20}: PLONK on BLS12-381 and
fflonk on BN254, for each shard count of --shards over the --devices list (repeats allowed: several contexts on one device
measure the cost of the fan-out on that card, not a speedup).

Every shape is warmed up before it is timed; --reps proofs are timed one by one and the fastest is reported, with the per-round
host wall clock sb_last_ms(1..5) of that proof.  Every timed proof must equal the single-context proof.  One JSON line per
point, with the card's name and power limit read in the same run:
  {"proto", "curve", "log_n", "shards", "devices", "single_proofs_per_s", "multi_proofs_per_s", "single_rounds_ms",
   "multi_rounds_ms", "gpu", "power_limit_w"}
Usage: python profiles/bench_plonk_multi.py [--devices 0,0,0,0] [--shards 1,2,4] [--log-n 16,18,20] [--protos plonk,fflonk] [--reps 5]"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from snarkjs_b200 import fflonk, getCurveFromName, plonk, synth  # noqa: E402
from profiles.bench_groth16_batch import card  # noqa: E402

SETUPS = {"plonk": (plonk, "bls12381", synth.synth_plonk_zkey, 11), "fflonk": (fflonk, "bn128", synth.synth_fflonk_zkey, 9)}


def timed(prove, curve, reps, want):
    """(fastest seconds, its sb_last_ms(1..5)) over reps proofs, each checked against want"""
    best, rounds = None, None
    for _ in range(reps):
        t0 = time.perf_counter()
        got = prove()
        dt = time.perf_counter() - t0
        assert got == want, "proof differs from the single-context proof"
        if best is None or dt < best:
            best, rounds = dt, [round(curve.last_ms(i), 3) for i in range(1, 6)]
    return best, rounds


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--devices", default="0,0,0,0", help="device of each context; the first is rank 0")
    ap.add_argument("--shards", default="1,2,4")
    ap.add_argument("--log-n", default="16,18,20")
    ap.add_argument("--protos", default="plonk,fflonk")
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    devices = [int(x) for x in a.devices.split(",")]
    shard_counts = [int(x) for x in a.shards.split(",")]
    assert max(shard_counts) <= len(devices), "more shards than contexts in --devices"
    name, pl = card()
    for proto in a.protos.split(","):
        mod, cname, make, nbl = SETUPS[proto]
        curves = [getCurveFromName(cname, d) for d in devices]
        try:
            for log_n in [int(x) for x in a.log_n.split(",")]:
                zkey, wit = make(curves[0], log_n)
                bl = b"".join(mod.random_fr(curves[0]) for _ in range(nbl))
                pk = mod.ProvingKey(zkey, curves[0])
                try:
                    want = pk.prove_raw(wit, bl)
                    t_single, r_single = timed(lambda: pk.prove_raw(wit, bl), curves[0], a.reps, want)
                    for s in shard_counts:
                        sk = mod.ShardedProvingKey(zkey, curves[:s])
                        try:
                            sk.prove_raw(wit, bl)                                   # warm-up
                            t_multi, r_multi = timed(lambda: sk.prove_raw(wit, bl), curves[0], a.reps, want)
                        finally:
                            sk.release()
                        print(json.dumps({"proto": proto, "curve": cname, "log_n": log_n, "shards": s, "devices": devices[:s],
                                          "single_proofs_per_s": round(1 / t_single, 2), "multi_proofs_per_s": round(1 / t_multi, 2),
                                          "single_rounds_ms": r_single, "multi_rounds_ms": r_multi, "gpu": name, "power_limit_w": pl}),
                              flush=True)
                finally:
                    pk.release()
                del zkey
        finally:
            for c in curves:
                c.terminate()


if __name__ == "__main__":
    main()
