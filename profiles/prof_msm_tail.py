"""Where the MSM tail's time goes, per group.

1. The bench key (Groth16, BN254, domain 2^LOGN, synth_groth16_zkey seed 1) proved with every stream serialised
   (sb_set_tuning(2, 1)): the kernel-class breakdown of sb_last_stat 8..15, with head folding and bucket reduction split
   into G1 and G2 MSMs (16 / 17).  Median of REPS proofs.
2. One registered 2^LOGN MSM per (curve, group): device time of the call (CUDA events inside the library: sort,
   accumulation, tail, window-sum copy and host combine) and its fold / reduce share.  Median of REPS calls.
Prints one JSON object, with the GPU's name and power limit."""
import json, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import snarkjs_b200
from snarkjs_b200 import groth16, synth
from snarkjs_b200.curve import _ptr

L = int(os.environ.get("LOGN", "20"))
REPS = int(os.environ.get("REPS", "5"))
NAMES = ["digits_sort", "accumulate_g1", "accumulate_g2", "fold", "bucket_reduce", "qap_rows", "ntt_passes", "join_abc"]


def gpu():
    o = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True)
    return o.stdout.strip()


def med(xs):
    return sorted(xs)[len(xs) // 2]


def proof_breakdown():
    c = snarkjs_b200.getCurveFromName("bn128")
    lib, h = c.lib, c.handle
    pk = groth16.ProvingKey(synth.synth_groth16_zkey(c, L, seed=1), curve=c)
    w = synth.chain_witness(c.r, L)
    r = (5 * (1 << 256) % c.r).to_bytes(32, "little")
    s = (7 * (1 << 256) % c.r).to_bytes(32, "little")
    proof = np.empty(256, np.uint8)
    lib.sb_set_tuning(2, 1)
    runs = []
    for i in range(REPS + 2):
        c.check(lib.sb_groth16_prove(h, pk.handle, _ptr(w), w.size // 32, r, s, _ptr(proof)))
        if i < 2:
            continue
        st = {nm: lib.sb_last_stat(h, 8 + k) for k, nm in enumerate(NAMES)}
        st["fold_g2"], st["bucket_reduce_g2"] = lib.sb_last_stat(h, 16), lib.sb_last_stat(h, 17)
        st["fold_g1"], st["bucket_reduce_g1"] = st["fold"] - st["fold_g2"], st["bucket_reduce"] - st["bucket_reduce_g2"]
        st["tail"] = st["fold"] + st["bucket_reduce"]
        st["serialised_device_total"] = c.last_ms(0)
        runs.append(st)
    lib.sb_set_tuning(2, 0)
    pk.release()
    c.terminate()
    return {k: med([x[k] for x in runs]) for k in runs[0]}


def registered_msms():
    out = {}
    rng = np.random.default_rng(3)
    n = 1 << L
    sc = rng.integers(0, 256, size=n * 32, dtype=np.uint8)
    sc.reshape(n, 32)[:, 31] &= 0x1f                          # 253-bit scalars: below r on both curves
    for name in ("bn128", "bls12381"):
        c = snarkjs_b200.getCurveFromName(name)
        lib, h = c.lib, c.handle
        for grp in (1, 2):
            G = c.G1 if grp == 1 else c.G2
            hb = G.registerBases(synth.gen_points(c, grp, 7, n))
            ms, fold, red = [], [], []
            for i in range(REPS + 2):
                G.multiExpRegistered(hb, sc)
                if i >= 2:
                    ms.append(c.last_ms(2)); fold.append(lib.sb_last_stat(h, 11)); red.append(lib.sb_last_stat(h, 12))
            out[f"{name}_g{grp}"] = {"msm_ms": med(ms), "fold_ms": med(fold), "bucket_reduce_ms": med(red)}
        c.terminate()
    return out


if __name__ == "__main__":
    res = {"gpu": gpu(), "log_n": L, "reps": REPS, "groth16_serialised_ms": proof_breakdown(), "registered_msm_ms": registered_msms()}
    print(json.dumps(res, indent=1))
