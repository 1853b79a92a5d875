"""PLONK (BN254, BLS12-381) and fflonk (BN254) verifications per second through sb_plonk_verify_batch /
sb_fflonk_verify_batch, for counts 1, 2^10, 2^14, 2^17 and 1 or 16 public inputs.  The time is sb_last_ms(0): CUDA events
around the whole call (upload of the key, publics and proofs, the line precomputation, the transcript and scalar kernel,
the scalar multiplications, the pairing kernel, status download).

The proofs are real: a pool of 64 from prove_batch on a synthetic structured key (oracle.plonk.chain_gates with 64 gates,
plonk_setup_synth / fflonk_setup_synth), repeated to the count.  Each shape is run once untimed first, then the best of
--reps calls is kept.  The card's name and power limit are printed in the same run.  No CPU arm is timed here.

    python profiles/bench_plonk_verify.py [--out results.json] [--reps 3]"""
import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import fflonk as OF  # noqa: E402
from oracle import oracle as O  # noqa: E402
from oracle import plonk as OP  # noqa: E402
from profiles.bench_groth16_verify import card  # noqa: E402

COUNTS = (1, 1 << 10, 1 << 14, 1 << 17)
N_PUBLIC = (1, 16)
CASES = (("plonk", O.BN254, "bn128"), ("plonk", O.BLS12_381, "bls12381"), ("fflonk", O.BN254, "bn128"))


def pool(proto, cid, c, n_public, size=64):
    """vk bytes, power, pool publics (plain LE), pool proofs (as the prover writes them): every proof verifies."""
    import snarkjs_b200
    m = snarkjs_b200.plonk if proto == "plonk" else snarkjs_b200.fflonk
    ci = O.CURVES[cid]
    gates, adds, n_vars, n_pub, wit = OP.chain_gates(64, r=ci.r, n_pub=n_public)
    if proto == "plonk":
        zkey = OP.plonk_setup_synth(gates, adds, n_vars, n_pub, tau=0x7E57 + n_public, curve=cid)
    else:
        zkey = OF.fflonk_setup_synth(gates, adds, n_vars, n_pub, tau=0x7E57 + n_public)
    vk = m.verification_key(zkey)
    pk = m.ProvingKey(zkey, c)
    try:
        items = m.prove_batch(pk, [OP.wtns_bytes(wit, ci.r)] * size)
    finally:
        pk.release()
    pubs = [b"".join(int(s).to_bytes(32, "little") for s in pub) for _p, pub in items]
    prfs = [m.proof_bytes(p, ci.n8q, ci.q, ci.r) for p, _pub in items]
    return m.vk_bytes(vk), int(vk["power"]), pubs, prfs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the rows as JSON to this file")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--counts", default=",".join(str(c) for c in COUNTS))
    args = ap.parse_args()
    import snarkjs_b200
    name, pl = card()
    print(f"card: {name}, power limit / max SM clock: {pl}", flush=True)
    rows = []
    for proto, cid, cname in CASES:
        c = snarkjs_b200.getCurveFromName(cname)
        fn = c.lib.sb_plonk_verify_batch if proto == "plonk" else c.lib.sb_fflonk_verify_batch
        for npub in N_PUBLIC:
            vk, power, pubs, prfs = pool(proto, cid, c, npub)
            for count in (int(x) for x in args.counts.split(",")):
                pub = b"".join(pubs[i % len(pubs)] for i in range(count))
                prf = b"".join(prfs[i % len(prfs)] for i in range(count))
                st = (ctypes.c_int32 * count)()
                ms = []
                for rep in range(args.reps + 1):       # rep 0 warms the shape up
                    c.check(fn(c.handle, vk, len(vk), npub, power, pub, prf, count, st))
                    if rep:
                        ms.append(c.last_ms(0))
                assert not any(st), "a proof did not verify"
                best = min(ms)
                row = {"protocol": proto, "curve": cname, "n_public": npub, "count": count, "ms": best, "ms_all": ms,
                       "verifications_per_s": count / (best / 1e3)}
                rows.append(row)
                print(json.dumps(row), flush=True)
        c.terminate()
    res = {"card": name, "power_limit_max_sm_clock": pl, "rows": rows}
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
