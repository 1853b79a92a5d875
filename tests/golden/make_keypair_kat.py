"""Extracts the reference's only hard-coded known-answer vectors (test/keypar_test.js:20-119: three (g1_s, g1_sx, g2_spx)
triples of a powers-of-tau public key and the challenge they were made for) into tests/golden/keypair_kat.json.
Needs a snarkjs checkout (SNARKJS_DIR=<checkout> python tests/golden/make_keypair_kat.py); the tests only read the JSON."""
import json
import os
import re

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(os.environ.get("SNARKJS_DIR", "snarkjs"), "test", "keypar_test.js")


def main():
    t = open(SRC).read()
    chal = "".join(re.findall(r'"([0-9a-f]{32})"\s*\+?', t.split("hex2ByteArray(")[1].split(");")[0]))
    assert len(chal) == 128
    out = {"source": "iden3/snarkjs test/keypar_test.js:20-119", "challenge_hex": chal, "cases": []}
    for pers, name in enumerate(["tau", "alpha", "beta"]):
        def nums(var):
            body = t.split(f"const {name}_{var} = ")[1].split(");")[0]
            return [int(x, 16) for x in re.findall(r'Scalar\.e\("0x([0-9a-f]+)"\)', body)]
        s, sx, spx = nums("g1_s"), nums("g1_sx"), nums("g2_spx")
        assert len(s) == 2 and len(sx) == 2 and len(spx) == 4
        out["cases"].append({"name": name, "personalization": pers, "g1_s": [hex(v) for v in s], "g1_sx": [hex(v) for v in sx],
                             "g2_spx": [[hex(spx[0]), hex(spx[1])], [hex(spx[2]), hex(spx[3])]]})
    json.dump(out, open(os.path.join(HERE, "keypair_kat.json"), "w"), indent=1)
    print("wrote keypair_kat.json:", len(out["cases"]), "cases")


if __name__ == "__main__":
    main()
