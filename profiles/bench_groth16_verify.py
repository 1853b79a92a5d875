"""Groth16 verifications per second through sb_groth16_verify_batch, on both curves, for counts 1, 2^10, 2^14, 2^17 and
1 or 16 public inputs.  The time is sb_last_ms(0): CUDA events around the whole call (upload of the key, publics and
proofs, line precomputation, e(alpha1, beta2), the scalar multiplications, the pairing kernel, status download).

The proofs are forged from known scalars (tests/test_gpu_groth16_verify.py): a pool of 64 valid proofs, repeated to the
count; every proof costs the same, whatever its bytes.  Each shape is run once untimed first.  The card's name and power
limit are printed in the same run.  No CPU arm is timed here.

    python profiles/bench_groth16_verify.py [--out results.json] [--reps 3]"""
import argparse
import ctypes
import json
import os
import random
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import oracle as O  # noqa: E402

COUNTS = (1, 1 << 10, 1 << 14, 1 << 17)
N_PUBLIC = (1, 16)


def g_bytes(cid, group, k):
    ci = O.CURVES[cid]
    gen = ci.g1_affine_bytes(ci.g1) if group == 1 else ci.g2_affine_bytes(ci.g2)
    return O.g_to_affine(cid, group, O.g_times(cid, group, O.g_from_affine(cid, group, gen), (k % ci.r).to_bytes(32, "little")))


def forged(cid, n_public, pool=64, seed=1):
    """vk bytes, pool publics (plain LE), pool proofs: every proof verifies."""
    rng = random.Random(seed)
    r = O.CURVES[cid].r
    a, b, g, d = (rng.randrange(1, r) for _ in range(4))
    k = [rng.randrange(1, r) for _ in range(n_public + 1)]
    vk = g_bytes(cid, 1, a) + g_bytes(cid, 2, b) + g_bytes(cid, 2, g) + g_bytes(cid, 2, d) + b"".join(g_bytes(cid, 1, x) for x in k)
    pubs, prfs = [], []
    for _ in range(pool):
        s = [rng.randrange(r) for _ in range(n_public)]
        x, y = rng.randrange(1, r), rng.randrange(1, r)
        cp = (k[0] + sum(si * ki for si, ki in zip(s, k[1:]))) % r
        z = (x * y - a * b - cp * g) * pow(d, -1, r) % r
        pubs.append(b"".join(v.to_bytes(32, "little") for v in s))
        prfs.append(g_bytes(cid, 1, x) + g_bytes(cid, 2, y) + g_bytes(cid, 1, z))
    return vk, pubs, prfs


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=60).stdout.strip()
    except Exception as e:          # the number still stands with the card's name; say what was not read
        pl = f"not read ({e})"
    return name, pl


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
    for cid, cname in ((O.BN254, "bn128"), (O.BLS12_381, "bls12381")):
        c = snarkjs_b200.getCurveFromName(cname)
        for npub in N_PUBLIC:
            vk, pubs, prfs = forged(cid, npub)
            for count in (int(x) for x in args.counts.split(",")):
                pub = b"".join(pubs[i % len(pubs)] for i in range(count))
                prf = b"".join(prfs[i % len(prfs)] for i in range(count))
                st = (ctypes.c_int32 * count)()
                ms = []
                for rep in range(args.reps + 1):       # rep 0 warms the shape up
                    c.check(c.lib.sb_groth16_verify_batch(c.handle, vk, len(vk), npub, pub, prf, count, st))
                    if rep:
                        ms.append(c.last_ms(0))
                assert not any(st), "a forged proof did not verify"
                best = min(ms)
                row = {"curve": cname, "n_public": npub, "count": count, "ms": best, "ms_all": ms,
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
