#!/usr/bin/env python
"""Extracts tests/golden/ptau_prepare_goldens.npz from the reference's prepared powers-of-tau fixture
(test/plonk_circuit/powersOfTau15_final.ptau of a snarkjs checkout).  Needs the checkout, no GPU:
    SNARKJS_DIR=<snarkjs checkout> python tests/golden/make_ptau_prepare_golden.py

What is extracted (binary fixture data only, no reference source):
  header, section6, section7   sections 1, 6 and 7 of the file
  alphaTauG1, betaTauG1        the first 1024 points of sections 4 and 5
  s{12,13,14,15}_sha256        the sha256 of every power-k block of the Lagrange sections that `powersoftau prepare phase2`
                               wrote (G.lagrangeEvaluations of the 2^k-point prefixes of sections 2-5; block k starts at
                               point 2^k - 1): k <= 12 for section 12, k <= 10 for sections 13-15
With the tauG1[0:4096] / tauG2[0:1024] prefixes of ptau_goldens.npz this recomputes each of those blocks and assembles a
power-10 ptau (sections 1-7) cut from the fixture."""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import oracle as O  # noqa: E402

REF = os.path.join(os.environ.get("SNARKJS_DIR", "snarkjs"), "test")


def u8(b):
    return np.frombuffer(bytes(b), dtype=np.uint8)


def main():
    data, secs = O.read_binfile(f"{REF}/plonk_circuit/powersOfTau15_final.ptau", "ptau", 1)
    out = {"header": u8(O.section(data, secs, 1)), "section6": u8(O.section(data, secs, 6)),
           "section7": u8(O.section(data, secs, 7)),
           "alphaTauG1": u8(O.section(data, secs, 4)[:64 * 1024]), "betaTauG1": u8(O.section(data, secs, 5)[:64 * 1024])}
    for sid, sg, kmax in ((12, 64, 12), (13, 128, 10), (14, 64, 10), (15, 64, 10)):
        sec = O.section(data, secs, sid)
        out[f"s{sid}_sha256"] = np.concatenate([u8(hashlib.sha256(sec[((1 << k) - 1) * sg:((2 << k) - 1) * sg]).digest())
                                                for k in range(kmax + 1)])
    np.savez(os.path.join(HERE, "ptau_prepare_goldens.npz"), **out)
    print("ptau_prepare_goldens:", {k: v.size for k, v in out.items()})


if __name__ == "__main__":
    main()
