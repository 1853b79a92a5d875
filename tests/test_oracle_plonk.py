"""CPU checks of the PLONK restatement in oracle/plonk.py (what pins it is listed in that file's header)."""
import json

import pytest

from oracle import oracle as orc
from oracle import plonk

from tests import r1cs_shapes as S

BLINDERS = [0x1000 + 977 * i for i in range(11)]


def test_keccak256_known_answers():
    assert plonk.keccak256(b"").hex() == "c5d2460186f7233c927e7db2dcc703c0e500b653ca82273b7bfad8045d85a470"
    assert plonk.keccak256(b"abc").hex() == "4e03657aea45a94fc7d47ba826c8d667c0d1e6e33a64a036ec44f58fa12d6c45"
    # two-block message (rate is 136 bytes)
    assert len(plonk.keccak256(b"a" * 200)) == 32 and plonk.keccak256(b"a" * 200) != plonk.keccak256(b"a" * 199)


@pytest.fixture(scope="module")
def ref_case(golden):
    g = golden("plonk_case.npz")
    return {k: bytes(v) for k, v in g.items()}


def test_vk_from_reference_zkey_matches_reference_vk(ref_case):
    vk_ref = json.loads(ref_case["vk_json"])
    vk = plonk.plonk_vk(ref_case["zkey"])
    assert vk == vk_ref


def test_prove_reference_zkey_verifies_with_reference_vk(ref_case):
    vk_ref = json.loads(ref_case["vk_json"])
    proof, public = plonk.plonk_prove(ref_case["zkey"], ref_case["wtns"], BLINDERS)
    assert public == json.loads(ref_case["public_json"])            # ["7776", "1"]
    assert plonk.plonk_verify(vk_ref, public, proof)
    assert list(proof.keys()) == list(json.loads(ref_case["proof_json"]).keys())   # same JSON shape as the reference
    # every field matters
    for key in ("A", "Z", "T2", "Wxiw"):
        bad = dict(proof)
        bad[key] = proof["B"]
        assert not plonk.plonk_verify(vk_ref, public, bad), key
    for key in ("eval_a", "eval_s2", "eval_zw"):
        bad = dict(proof)
        bad[key] = str((int(proof[key]) + 1) % orc.P_BN_R)
        assert not plonk.plonk_verify(vk_ref, public, bad), key
    assert not plonk.plonk_verify(vk_ref, ["7777", "1"], proof)
    assert not plonk.plonk_verify(vk_ref, [str(7776 + orc.P_BN_R), "1"], proof)     # aliased public input
    # zero blinders are legal too (b = 0 leaves the polynomials unblinded)
    p0, pub0 = plonk.plonk_prove(ref_case["zkey"], ref_case["wtns"], [0] * 11)
    assert plonk.plonk_verify(vk_ref, pub0, p0)
    assert p0 != proof


def test_stored_reference_proof_is_stale(ref_case):
    """Documents why proof.json is not a pin (oracle/plonk.py header): the current verifier rejects it."""
    assert not plonk.plonk_verify(json.loads(ref_case["vk_json"]), json.loads(ref_case["public_json"]),
                                  json.loads(ref_case["proof_json"]))


@pytest.mark.parametrize("n_gates", [13, 120])
def test_synthetic_setup_prove_verify(n_gates):
    gates, adds, n_vars, n_pub, wit = plonk.chain_gates(n_gates)
    zkey = plonk.plonk_setup_synth(gates, adds, n_vars, n_pub, tau=0x1234567890ABCDEF1234567)
    proof, public = plonk.plonk_prove(zkey, plonk.wtns_bytes(wit), BLINDERS)
    vk = plonk.plonk_vk(zkey)
    assert plonk.plonk_verify(vk, public, proof)
    assert not plonk.plonk_verify(vk, [str(int(public[0]) ^ 1)], proof)
    # a wrong witness breaks the copy constraints (plonk_prove.js:436-438) or the divisibility of T
    wit2 = list(wit)
    wit2[3] = (wit2[3] + 1) % orc.P_BN_R
    with pytest.raises(ValueError):
        plonk.plonk_prove(zkey, plonk.wtns_bytes(wit2), BLINDERS)


def test_bls12381_pairing_is_bilinear():
    from oracle import pairing_bls as pb
    ci = orc.CURVES[orc.BLS12_381]
    g2 = orc.g_from_affine(ci.id, 2, ci.g2_affine_bytes(ci.g2))
    a, b = 0x1234567, 0x89ABCDE
    bq = ci.g2_from_affine_bytes(bytes(orc.g_to_affine(ci.id, 2, orc.g_times(ci.id, 2, g2, b.to_bytes(32, "little"))))[:4 * ci.n8q])
    ap = pb.g1_mul(ci.g1, a)
    assert pb.g1_valid(ap)
    assert pb.pairing_product_is_one([(ap, bq), (pb.g1_neg(pb.g1_mul(ci.g1, a * b % ci.r)), ci.g2)])
    assert not pb.pairing_product_is_one([(ap, bq), (pb.g1_neg(pb.g1_mul(ci.g1, (a * b + 1) % ci.r)), ci.g2)])


def test_plonk_on_bls12381_verifies():
    ci = orc.CURVES[orc.BLS12_381]
    gates, adds, n_vars, n_pub, wit = plonk.chain_gates(60, r=ci.r, n_pub=2)
    zkey = plonk.plonk_setup_synth(gates, adds, n_vars, n_pub, tau=99991, curve=orc.BLS12_381)
    proof, public = plonk.plonk_prove(zkey, plonk.wtns_bytes(wit, ci.r), BLINDERS)
    vk = plonk.plonk_vk(zkey)
    assert vk["curve"] == "bls12381" and plonk.plonk_verify(vk, public, proof)
    bad = dict(proof)
    bad["eval_c"] = str((int(proof["eval_c"]) + 1) % ci.r)
    assert not plonk.plonk_verify(vk, public, bad)
    assert not plonk.plonk_verify(vk, [public[1], public[0]], proof)


@pytest.mark.parametrize("tag", ["c8", "c2048"])
def test_plonk_setup_reproduces_reference_zkeys_byte_for_byte(golden, reference_plonk_key, tag):
    """oracle.plonk.plonk_setup (r1cs -> gates, additions, selectors, sigma, Lagrange, commitments, header) gives exactly the
    zkey files the reference ships: test/plonk_circuit/circuit.zkey (14 748 bytes) and test/circuit2/circuit.zkey (4 160 728
    bytes: domain 2048, 1001 additions, 4 public signals).  This pins the key layout and everything plonk_setup_synth shares."""
    g = golden("plonk_setup_cases.npz")
    zkey, wtns = reference_plonk_key(g, tag)
    if tag == "c8":
        assert zkey == bytes(golden("plonk_case.npz")["zkey"])
    # and the prover / verifier work on it (real circom circuit with additions for c2048)
    proof, public = plonk.plonk_prove(zkey, wtns, BLINDERS)
    assert plonk.plonk_verify(plonk.plonk_vk(zkey), public, proof)
    bad = dict(proof)
    bad["eval_s1"] = str((int(proof["eval_s1"]) + 1) % orc.P_BN_R)
    assert not plonk.plonk_verify(plonk.plonk_vk(zkey), public, bad)


# ----------------------------------------------------------------------------- keys from tests/r1cs_shapes.py circuits
SHAPES_STRUCTURED = [label for label, c in S.PLONK_CASES.items() if c[3] and label not in S.PLONK_ERRORS]


@pytest.mark.parametrize("label", SHAPES_STRUCTURED)
def test_shape_keys_prove_and_verify(label):
    """plonk_setup over a ptau with known tau, for circuits shaped like circom output: the proof verifies, and its public
    signals are the circuit's."""
    circ = S.case(label)
    zkey = S.plonk_zkey(label)
    proof, public = plonk.plonk_prove(zkey, circ.wtns(), BLINDERS)
    assert public == [str(x) for x in circ.public()]
    vk = plonk.plonk_vk(zkey)
    assert plonk.plonk_verify(vk, public, proof), label
    bad = dict(proof)
    bad["eval_b"] = str((int(proof["eval_b"]) + 1) % circ.r)
    assert not plonk.plonk_verify(vk, public, bad), label


@pytest.mark.parametrize("k,extra,n_gates,domain", [(8, 0, 256, 256), (8, 1, 257, 512), (8, -2, 254, 256), (8, -1, 255, 256),
                                                    (12, 0, 4096, 4096), (12, 1, 4097, 8192)])
def test_gates_cases_land_on_their_domain(k, extra, n_gates, domain):
    zk = plonk.read_plonk_zkey(S.plonk_zkey(f"gates{k}{extra:+d}"))
    assert (zk["nConstraints"], zk["domainSize"], zk["nAdditions"], zk["nPublic"]) == (n_gates, domain, 0, 2)


def test_repeated_signal_gives_a_key_that_does_not_divide():
    """plonk_setup keys a linear combination by signal, so a signal twice in one keeps only its last entry (plonk_setup.js:
    147-149): the gates no longer encode the constraint, and T is not divisible by Z_H, as in the reference."""
    assert S.PLONK_ERRORS["coeffs"] == "Polynomial is not divisible"
    with pytest.raises(ValueError, match="^Polynomial is not divisible$"):
        plonk.plonk_prove(S.plonk_zkey("coeffs"), S.case("coeffs").wtns(), BLINDERS)


@pytest.mark.parametrize("label", ["public0", "tiny1"])
def test_key_without_public_signals_is_refused_with_the_reference_text(label):
    """With nPublic = 0 the reference reads no Lagrange polynomial (plonk_prove.js:503-509), and round 3's first read of
    L1 throws (:613-617, evaluations.js:39-44)."""
    circ = S.case(label)
    zkey = S.plonk_zkey(label)
    assert plonk.read_plonk_zkey(zkey)["nPublic"] == 0
    with pytest.raises(ValueError, match=r"^Evaluations\.getEvaluation\(\) out of bounds$"):
        plonk.plonk_prove(zkey, circ.wtns(), BLINDERS)
