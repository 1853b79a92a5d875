"""CPU: the circuits of tests/r1cs_shapes.py through the oracle.  build_abc (the QAP rows A.w, B.w, A.w * B.w) equals a
per-row sum in Python integers for every shape, with section 4 in constraint order and shuffled; proofs from the
structured keys verify and reject a changed public signal; the reference's own circuit2 and c8 circuits, set up for
Groth16, do the same.  tests/test_gpu_groth16_shapes.py then holds the GPU prover to these oracle results."""
import numpy as np
import pytest

from oracle import oracle as O

from tests import r1cs_shapes as S


def _ints(curve, buf):
    r = O.CURVES[curve].r
    rinv = pow(1 << 256, -1, r)
    b = bytes(buf)
    return [int.from_bytes(b[i:i + 32], "little") * rinv % r for i in range(0, len(b), 32)]


def _coeffs(zkey):
    data, secs = O.read_binfile(zkey, "zkey", 2)
    return bytes(O.section(data, secs, 4))


@pytest.mark.parametrize("label", list(S.CASES))
def test_build_abc_equals_python_rows(label):
    circ = S.case(label)
    want = S.expected_abc(circ)
    w = circ.witness_array()
    zkey = S.case_zkey(label) if S.CASES[label][3] else None
    sec4 = _coeffs(zkey) if zkey else S.section4(circ)
    if zkey:
        assert sec4 == S.section4(circ), "zkey_new wrote another section 4 than the helper"
    shuffled = _coeffs(S.shuffle(O.write_binfile("zkey", 1, [(4, sec4)]), seed=3))
    assert shuffled != sec4 and sorted(shuffled[4:][i:i + 44] for i in range(0, len(sec4) - 4, 44)) == \
        sorted(sec4[4:][i:i + 44] for i in range(0, len(sec4) - 4, 44))
    for body in (sec4, shuffled):
        got = O.build_abc(circ.curve, body, w, circ.domain)
        assert [_ints(circ.curve, x) for x in got] == list(want), label


def test_shapes_have_their_advertised_geometry():
    """The properties the GPU tests rely on: the fit cases fill or just overflow a domain, tiny has the requested
    nVars, ratio puts nVars and the domain on different sides of 2^12, a wide row has 2^14 terms."""
    fit, dbl = S.case("fit_exact"), S.case("fit_double")
    assert len(fit.cons) + fit.n_public + 1 == fit.domain == 256
    assert len(dbl.cons) + dbl.n_public + 1 == 257 and dbl.domain == 512
    for label, (shape, _c, params, _s) in S.CASES.items():
        if shape == "tiny":
            assert S.case(label).n_vars == params["n_vars"]
        if shape == "public":
            assert S.case(label).n_public == params["n_public"]
    assert S.case("tiny2").n_vars == S.case("tiny2").n_public + 1 and S.case("tiny4").n_vars == S.case("tiny4").n_public + 1
    T = 1 << 12
    for pre in ("", "bls_"):
        v, r, b = S.case(pre + "ratio_vars"), S.case(pre + "ratio_rows"), S.case(pre + "ratio_both")
        assert v.n_vars >= T > v.domain and r.domain >= T > r.n_vars
        assert b.n_vars >= T and b.domain >= T and b.n_vars.bit_length() != b.domain.bit_length()
    assert max(len(c[0]) for c in S.case("wide").cons) >= 1 << 14 and max(len(c[1]) for c in S.case("wide").cons) >= 1 << 14
    assert max(len(c[0]) for c in S.case("bits").cons) == 254 and max(len(c[0]) for c in S.case("bls_bits").cons) == 255


def test_every_shape_checks_its_witness():
    for label in S.CASES:
        circ = S.case(label)
        if circ.n_vars > circ.n_public + 1:
            assert circ.unsatisfied(circ.broken_witness()), label
    with pytest.raises(ValueError, match="does not satisfy"):
        class Bad(S.Circuit):
            name = "bad"

            def build(self):
                self.add([(0, 1)], [(0, 1)], [(0, 2)])
        Bad(O.BN254)


def _prove_and_verify(zkey, witness_bytes, public, curve):
    ci = O.CURVES[curve]
    proof, pub = O.groth16_prove(zkey, witness_bytes, ci.fr_to_mont(1234567), ci.fr_to_mont(7654321))
    assert [int(x) for x in pub] == list(public)
    vk = O.zkey_vk(zkey)
    assert O.groth16_verify(vk, [int(x) for x in pub], proof)
    return vk, proof, [int(x) for x in pub]


@pytest.mark.parametrize("label", ["bits", "coeffs", "empty", "public0", "public17", "fit_exact", "fit_double", "tiny1", "tiny2",
                                   "tiny49", "bls_coeffs", "bls_public17", "bls_tiny363"])
def test_structured_proofs_verify(label):
    circ = S.case(label)
    vk, proof, pub = _prove_and_verify(S.case_zkey(label), circ.wtns(), circ.public(), circ.curve)
    for i in sorted({0, len(pub) - 1} if pub else ()):     # an output and a public input
        bad = list(pub)
        bad[i] = (bad[i] + 1) % circ.r
        assert not O.groth16_verify(vk, bad, proof), (label, i)
    if not pub:   # nothing public to change: a proof of another witness's A must fail
        tampered = dict(proof, pi_a=proof["pi_c"])
        assert not O.groth16_verify(vk, pub, tampered)


@pytest.mark.parametrize("tag", ["c2048", "c8"])
def test_reference_circuits_set_up_for_groth16_verify(golden, tag):
    """circuit2 (1000 constraints, 4 public signals: domain 1024) and c8 (a constraint with empty A and B sides) from the
    reference's PLONK fixtures, given a Groth16 key by zkey_new over a prepared powers of tau."""
    g = golden("plonk_setup_cases.npz")
    r1 = O.read_r1cs(bytes(g[f"{tag}_r1cs"]))
    nc, npub = r1["nConstraints"], r1["nOutputs"] + r1["nPubInputs"]
    if tag == "c8":
        assert any(not a and not b for a, b, _c in r1["constraints"])
    domain = 1 << (nc + npub).bit_length()
    zkey = O.zkey_new(bytes(g[f"{tag}_r1cs"]), S.prepared_ptau(O.BN254, domain))
    _, W = O.read_wtns(bytes(g[f"{tag}_wtns"]))
    w = [int.from_bytes(W[i:i + 32], "little") for i in range(0, len(W), 32)]
    ok = lambda lc: sum(v * w[s] for s, v in lc) % O.P_BN_R
    assert all(ok(a) * ok(b) % O.P_BN_R == ok(c) for a, b, c in r1["constraints"])
    vk, proof, pub = _prove_and_verify(zkey, bytes(g[f"{tag}_wtns"]), w[1:npub + 1], O.BN254)
    assert not O.groth16_verify(vk, [pub[0] + 1] + pub[1:], proof)


def test_shuffled_section4_gives_the_same_oracle_proof():
    circ = S.case("coeffs")
    zkey = S.case_zkey("coeffs")
    ci = O.CURVES[circ.curve]
    r, s = ci.fr_to_mont(5), ci.fr_to_mont(6)
    assert O.groth16_prove(S.shuffle(zkey, 9), circ.wtns(), r, s) == O.groth16_prove(zkey, circ.wtns(), r, s)
