"""CPU checks of the fflonk restatement in oracle/fflonk.py (its pins are listed in that file's header)."""
import copy
import json

import pytest

from oracle import fflonk
from oracle import oracle as orc

from tests import r1cs_shapes as S

BLINDERS = [0x4000 + 1299709 * i for i in range(9)]


@pytest.fixture(scope="module")
def ref_case(golden):
    return {k: bytes(v) for k, v in golden("fflonk_case.npz").items()}


def test_vk_from_reference_zkey_matches_reference_vk(ref_case):
    assert fflonk.fflonk_vk(ref_case["zkey"]) == json.loads(ref_case["vk_json"])


def test_prove_reference_zkey_verifies_with_reference_vk(ref_case):
    vk = json.loads(ref_case["vk_json"])
    proof, public = fflonk.fflonk_prove(ref_case["zkey"], ref_case["wtns"], BLINDERS)
    assert public == json.loads(ref_case["public_json"])
    assert list(proof["polynomials"]) == ["C1", "C2", "W1", "W2"]
    assert list(proof["evaluations"]) == list(fflonk.EVAL_NAMES) + ["inv"]
    assert fflonk.fflonk_verify(vk, public, proof)
    for key in ("C1", "C2", "W1", "W2"):
        bad = copy.deepcopy(proof)
        bad["polynomials"][key] = proof["polynomials"]["C1" if key != "C1" else "C2"]
        assert not fflonk.fflonk_verify(vk, public, bad), key
    for key in ("ql", "s3", "a", "zw", "t2w"):
        bad = copy.deepcopy(proof)
        bad["evaluations"][key] = str((int(proof["evaluations"][key]) + 1) % orc.P_BN_R)
        assert not fflonk.fflonk_verify(vk, public, bad), key
    assert not fflonk.fflonk_verify(vk, [str(int(public[0]) ^ 1)], proof)
    assert not fflonk.fflonk_verify(vk, [str(int(public[0]) + orc.P_BN_R)], proof)       # aliased public input
    # `inv` is the inverse of the product the on-chain verifier would otherwise have to invert (:1182-1245): not used
    # by the JS verifier, but it must be a field element and differ between proofs with different challenges
    p2, _ = fflonk.fflonk_prove(ref_case["zkey"], ref_case["wtns"], [b + 1 for b in BLINDERS])
    assert fflonk.fflonk_verify(vk, public, p2) and p2["evaluations"]["inv"] != proof["evaluations"]["inv"]


def test_wrong_witness_is_rejected(ref_case):
    _, w = orc.read_wtns(ref_case["wtns"])
    wit = [int.from_bytes(w[i:i + 32], "little") for i in range(0, len(w), 32)]
    wit[3] = (wit[3] + 1) % orc.P_BN_R
    from oracle.plonk import wtns_bytes
    with pytest.raises(ValueError):
        fflonk.fflonk_prove(ref_case["zkey"], wtns_bytes(wit), BLINDERS)


@pytest.mark.parametrize("n_gates,n_pub", [(13, 1), (120, 3)])
def test_synthetic_setup_prove_verify(n_gates, n_pub):
    from oracle import plonk
    gates, adds, n_vars, n_pub, wit = plonk.chain_gates(n_gates, n_pub=n_pub)
    zkey = fflonk.fflonk_setup_synth(gates, adds, n_vars, n_pub, tau=0xC0FFEE12345)
    proof, public = fflonk.fflonk_prove(zkey, plonk.wtns_bytes(wit), BLINDERS)
    vk = fflonk.fflonk_vk(zkey)
    assert len(public) == n_pub and fflonk.fflonk_verify(vk, public, proof)
    assert not fflonk.fflonk_verify(vk, [str(int(public[0]) ^ 1)] + public[1:], proof)


def test_fflonk_setup_reproduces_reference_zkey_byte_for_byte(golden, ref_case):
    """oracle.fflonk.fflonk_setup (r1cs -> gates and additions through r1cs_constraint_processor.js, selectors, sigmas with the
    two blinding rows, Lagrange, PTau, C0, header) gives exactly test/fflonk/circuit.zkey (593 092 bytes, 100 additions)."""
    g = golden("plonk_setup_cases.npz")
    ptau = orc.write_binfile("ptau", 1, [(1, bytes(g["ptau_header"])), (2, bytes(g["ff256_ptau2"])), (3, bytes(g["ptau3"])), (12, b"")])
    assert fflonk.fflonk_setup(bytes(g["ff256_r1cs"]), ptau) == ref_case["zkey"]


# ----------------------------------------------------------------------------- keys from tests/r1cs_shapes.py circuits
SHAPES_STRUCTURED = [label for label, c in S.PLONK_CASES.items()
                     if c[3] and c[1] == orc.BN254 and label not in S.FFLONK_ERRORS]


@pytest.mark.parametrize("label", SHAPES_STRUCTURED)
def test_shape_keys_prove_and_verify(label):
    """fflonk_setup over a ptau with known tau, for circuits shaped like circom output, including nPublic = 0 (fflonk
    reads the whole Lagrange section, fflonk_prove.js, so it proves such keys)."""
    circ = S.case(label)
    zkey = S.fflonk_zkey(label)
    proof, public = fflonk.fflonk_prove(zkey, circ.wtns(), BLINDERS)
    assert public == [str(x) for x in circ.public()]
    vk = fflonk.fflonk_vk(zkey)
    assert fflonk.fflonk_verify(vk, public, proof), label
    bad = copy.deepcopy(proof)
    bad["evaluations"]["qc"] = str((int(proof["evaluations"]["qc"]) + 1) % orc.P_BN_R)
    assert not fflonk.fflonk_verify(vk, public, bad), label


@pytest.mark.parametrize("k,extra,n_gates,domain", [(8, -2, 254, 256), (8, -1, 255, 512), (8, 0, 256, 512), (8, 1, 257, 512),
                                                    (12, 0, 4096, 8192), (12, 1, 4097, 8192)])
def test_gates_cases_land_on_their_domain(k, extra, n_gates, domain):
    """fflonk keeps the last two rows for blinding: 2^k - 2 gates fill the domain, 2^k - 1 double it."""
    zk = fflonk.read_fflonk_zkey(S.fflonk_zkey(f"gates{k}{extra:+d}"))
    assert (zk["nConstraints"], zk["domainSize"], zk["nAdditions"], zk["nPublic"]) == (n_gates, domain, 0, 2)


def test_repeated_signal_gives_a_key_that_does_not_divide():
    """r1cs_constraint_processor.js keys a linear combination by signal as plonk_setup.js does: a repeated signal keeps
    only its last entry, and the key no longer encodes the circuit."""
    assert S.FFLONK_ERRORS["coeffs"] == "Polynomial is not divisible"
    with pytest.raises(ValueError, match="^Polynomial is not divisible$"):
        fflonk.fflonk_prove(S.fflonk_zkey("coeffs"), S.case("coeffs").wtns(), BLINDERS)
