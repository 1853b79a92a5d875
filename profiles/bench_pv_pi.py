"""The two forms of PI(xi) for the PLONK / fflonk verifiers, timed against each other on the GPU
(profiles/pv_pi_variants.cu): one thread per proof with one inversion for all its public inputs (the form
csrc/verify_plonk.cuh uses), against one thread and one inversion per (proof, public input) plus a per-proof sum.  Both
give the same PI and L_1 on the same inputs (checked before anything is printed).  The binary is compiled for sm_90a into a
temporary directory.  The card's name and power limit are printed in the same run.

    python profiles/bench_pv_pi.py [--count 131072] [--n-public 1,16] [--reps 5] [--out results.json]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from profiles.bench_groth16_verify import card  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--count", type=int, default=1 << 17)
    ap.add_argument("--n-public", default="1,16")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        exe = os.path.join(tmp, "pv_pi_variants")
        subprocess.check_call(["/usr/local/cuda/bin/nvcc", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                               "-o", exe, os.path.join(ROOT, "profiles", "pv_pi_variants.cu")])
        name, pl = card()
        print(f"card: {name}, power limit / max SM clock: {pl}", flush=True)
        rows = []
        for npub in (int(x) for x in args.n_public.split(",")):
            out = subprocess.run([exe, str(args.count), str(npub), str(args.reps)], check=True, capture_output=True, text=True).stdout
            for line in out.splitlines():
                rows.append(json.loads(line))
                print(line, flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"card": name, "power_limit_max_sm_clock": pl, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
