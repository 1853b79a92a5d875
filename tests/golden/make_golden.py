#!/usr/bin/env python
"""Extracts reference-produced golden vectors from the reference's committed fixtures
(test/** of a snarkjs checkout) into small .npz files under tests/golden/.  Needs the checkout, no GPU:
    SNARKJS_DIR=<snarkjs checkout> python tests/golden/make_golden.py

What is extracted (all bytes below were written by the reference's own Fr.fft /
G.multiExpAffine / G.ifft — SURVEY.md fact 6 / Appendix B):
  ntt_goldens.npz    [coef n | evals 4n] blocks from PLONK / fflonk zkeys: NTT_4n(coef||0) == evals
  msm_g1_goldens.npz PLONK header commitments == MSM(PTau[0:n], fromMontgomery(coef)); fflonk C0
  ptau_goldens.npz   ptau section 2/3 prefixes + selected Lagrange points of section 12/13:
                     L_{k,j} = sum_i (w_k^{-ij} / 2^k) * tau^i G   (G1 and G2 known answers)
  groth16_case.npz   test/groth16/witness.wtns + a Groth16 zkey produced by the ORACLE's restatement of
                     `zkey new` (src/zkey_new.js) from test/groth16/circuit.r1cs and powersOfTau15_final.ptau
                     (the reference ships no Groth16 zkey, SURVEY.md fact 5) — derived data, not reference bytes.
No reference source code is copied; only binary fixture data.
"""
import os
import struct
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
from oracle import oracle as O  # noqa: E402

REF = os.path.join(os.environ.get("SNARKJS_DIR", "snarkjs"), "test")


def u8(b):
    return np.frombuffer(bytes(b), dtype=np.uint8)


def ntt_goldens():
    out = {}
    # (file, [(section, byte offset in FEs, label)])
    for tag, path, blocks in [
        ("plonk8", f"{REF}/plonk_circuit/circuit.zkey", [(7, 0, "QM"), (8, 0, "QL"), (12, 0, "S1"), (12, 5, "S2"), (13, 0, "L0")]),
        ("fflonk256", f"{REF}/fflonk/circuit.zkey", [(7, 0, "QL"), (12, 0, "S1")]),
        ("plonk2048", f"{REF}/circuit2/circuit.zkey", [(7, 0, "QM"), (12, 10, "S3")]),
    ]:
        data, secs = O.read_binfile(path, "zkey", 2)
        zk = O.read_zkey_header(data, secs)
        n = zk["domainSize"]
        for sid, off_n, label in blocks:
            sec = O.section(data, secs, sid)
            o = off_n * n * 32
            out[f"{tag}_{label}_coef"] = u8(sec[o:o + 32 * n])
            out[f"{tag}_{label}_evals"] = u8(sec[o + 32 * n:o + 160 * n])
    np.savez(os.path.join(HERE, "ntt_goldens.npz"), **out)
    print("ntt_goldens:", {k: v.size for k, v in out.items()})


def msm_g1_goldens():
    out = {}
    for tag, path in [("plonk8", f"{REF}/plonk_circuit/circuit.zkey"), ("plonk2048", f"{REF}/circuit2/circuit.zkey")]:
        data, secs = O.read_binfile(path, "zkey", 2)
        zk = O.read_zkey_header(data, secs)
        n = zk["domainSize"]
        out[f"{tag}_ptau"] = u8(O.section(data, secs, 14)[:64 * n])
        picks = [("Qm", 7, 0), ("Ql", 8, 0), ("Qr", 9, 0), ("Qo", 10, 0), ("Qc", 11, 0), ("S1", 12, 0), ("S2", 12, 5), ("S3", 12, 10)]
        if tag == "plonk2048":
            picks = [picks[0], picks[5], picks[7]]   # keep the file small: 3 full-width 2048-term MSMs
        for name, sid, off_n in picks:
            sec = O.section(data, secs, sid)
            out[f"{tag}_{name}_coef_mont"] = u8(sec[off_n * n * 32:(off_n + 1) * n * 32])
            out[f"{tag}_{name}_commit"] = u8(zk[name])
    data, secs = O.read_binfile(f"{REF}/fflonk/circuit.zkey", "zkey", 2)
    zk = O.read_zkey_header(data, secs)
    n = zk["domainSize"]
    out["fflonk256_ptau"] = u8(O.section(data, secs, 16)[:64 * 8 * n])
    out["fflonk256_C0_coef_mont"] = u8(O.section(data, secs, 17)[:32 * 8 * n])
    out["fflonk256_C0_commit"] = u8(zk["C0"])
    np.savez(os.path.join(HERE, "msm_g1_goldens.npz"), **out)
    print("msm_g1_goldens:", {k: v.size for k, v in out.items()})


def ptau_goldens():
    data, secs = O.read_binfile(f"{REF}/plonk_circuit/powersOfTau15_final.ptau", "ptau", 1)
    out = {}
    out["tauG1"] = u8(O.section(data, secs, 2)[:64 * 4096])
    out["tauG2"] = u8(O.section(data, secs, 3)[:128 * 1024])
    s12, s13 = O.section(data, secs, 12), O.section(data, secs, 13)
    picks1 = [(0, 0), (1, 1), (2, 3), (4, 5), (7, 100), (10, 0), (10, 777), (12, 1), (12, 4095)]
    picks2 = [(0, 0), (2, 1), (3, 7), (5, 17), (8, 200), (10, 1023)]
    out["g1_picks"] = np.array(picks1, dtype=np.int64)
    out["g2_picks"] = np.array(picks2, dtype=np.int64)
    out["g1_expected"] = np.concatenate([u8(s12[((1 << k) - 1 + j) * 64:((1 << k) + j) * 64]) for k, j in picks1])
    out["g2_expected"] = np.concatenate([u8(s13[((1 << k) - 1 + j) * 128:((1 << k) + j) * 128]) for k, j in picks2])
    np.savez(os.path.join(HERE, "ptau_goldens.npz"), **out)
    print("ptau_goldens:", {k: v.size for k, v in out.items()})


def groth16_case():
    zkey = O.zkey_new(f"{REF}/groth16/circuit.r1cs", f"{REF}/plonk_circuit/powersOfTau15_final.ptau")
    wt = open(f"{REF}/groth16/witness.wtns", "rb").read()
    np.savez(os.path.join(HERE, "groth16_case.npz"), zkey=u8(zkey), wtns=u8(wt))
    print("groth16_case: zkey", len(zkey), "wtns", len(wt))


def plonk_case():
    """The reference's PLONK fixture as data: proving key, witness, verification key, public signals and the stored
    proof.json (kept although it is stale: see oracle/plonk.py header)."""
    d = f"{REF}/plonk_circuit"
    out = {name: u8(open(f"{d}/{fn}", "rb").read()) for name, fn in
           [("zkey", "circuit.zkey"), ("wtns", "witness.wtns"), ("vk_json", "verification_key.json"),
            ("public_json", "public.json"), ("proof_json", "proof.json")]}
    np.savez(os.path.join(HERE, "plonk_case.npz"), **out)
    print("plonk_case:", {k: v.size for k, v in out.items()})


def plonk_setup_cases():
    """Inputs of `plonk setup` for the two PLONK keys the reference ships (test/plonk_circuit: domain 8; test/circuit2: domain
    2048, 1001 additions, 4 public signals), with the sha256 of the zkey the reference produced from them: the r1cs, the
    witness, and the slices of the prepared ptau that src/plonk_setup.js reads (section 2 first n + 6 points, section 3 first
    two points, section 12 Lagrange points of the domain)."""
    import hashlib
    ptau = f"{REF}/plonk_circuit/powersOfTau15_final.ptau"
    pdata, psecs = O.read_binfile(ptau, "ptau", 1)
    out = {"ptau_header": u8(bytes(O.section(pdata, psecs, 1)))}
    for tag, d in (("c8", f"{REF}/plonk_circuit"), ("c2048", f"{REF}/circuit2")):
        zkey = open(f"{d}/circuit.zkey", "rb").read()
        zdata, zsecs = O.read_binfile(zkey, "zkey", 2)
        n = O.read_zkey_header(zdata, zsecs)["domainSize"]
        out[f"{tag}_r1cs"] = u8(open(f"{d}/circuit.r1cs", "rb").read())
        out[f"{tag}_wtns"] = u8(open(f"{d}/witness.wtns", "rb").read())
        out[f"{tag}_zkey_sha256"] = u8(hashlib.sha256(zkey).digest())
        out[f"{tag}_n"] = np.array([n], dtype=np.uint32)
        out[f"{tag}_ptau2"] = u8(bytes(O.section(pdata, psecs, 2)[:(n + 6) * 64]))
        out[f"{tag}_ptau12"] = u8(bytes(O.section(pdata, psecs, 12)[(n - 1) * 64:(2 * n - 1) * 64]))
    out["ptau3"] = u8(bytes(O.section(pdata, psecs, 3)[:256]))
    # fflonk setup (test/fflonk, domain 256): r1cs + the first 9n + 18 points of ptau section 2
    out["ff256_r1cs"] = u8(open(f"{REF}/fflonk/circuit.r1cs", "rb").read())
    out["ff256_ptau2"] = u8(bytes(O.section(pdata, psecs, 2)[:(9 * 256 + 18) * 64]))
    np.savez_compressed(os.path.join(HERE, "plonk_setup_cases.npz"), **out)
    print("plonk_setup_cases:", {k: v.size for k, v in out.items()})


def fflonk_case():
    """The reference's fflonk fixture as data (test/fflonk): proving key, witness, verification key, public signals."""
    d = f"{REF}/fflonk"
    out = {name: u8(open(f"{d}/{fn}", "rb").read()) for name, fn in
           [("zkey", "circuit.zkey"), ("wtns", "witness.wtns"), ("vk_json", "circuit_vk.json"), ("public_json", "public.json")]}
    np.savez_compressed(os.path.join(HERE, "fflonk_case.npz"), **out)
    print("fflonk_case:", {k: v.size for k, v in out.items()})


if __name__ == "__main__":
    which = sys.argv[1:] or ["ntt", "msm", "ptau", "groth16", "plonk", "fflonk", "plonk_setup"]
    if "ntt" in which:
        ntt_goldens()
    if "msm" in which:
        msm_g1_goldens()
    if "ptau" in which:
        ptau_goldens()
    if "groth16" in which:
        groth16_case()
    if "plonk" in which:
        plonk_case()
    if "fflonk" in which:
        fflonk_case()
    if "plonk_setup" in which:
        plonk_setup_cases()
