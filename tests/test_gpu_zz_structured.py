"""GPU: Groth16 proofs from sb_groth16_prove on structured synthetic keys (oracle/synth_setup.py) equal the oracle's and
VERIFY under the pairing check — on BN254 and on BLS12-381, where the reference ships no fixtures."""
import pytest

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", ["bn128", "bls12381"])
def test_groth16_structured_key_proof_verifies(name):
    import snarkjs_b200
    from oracle import oracle as orc
    from oracle import synth_setup as ss
    from oracle.plonk import wtns_bytes
    cid = orc.BN254 if name == "bn128" else orc.BLS12_381
    ci = orc.CURVES[cid]
    r1cs, wit = ss.chain_r1cs(cid, 1000)
    ptau = ss.prepared_ptau(cid, 1024, tau=0x1234567890ABCDEF, alpha=0xAAAA5555, beta=0xBBBB7777)
    zkey = orc.zkey_new(r1cs, ptau)
    wtns = wtns_bytes(wit, ci.r)
    r, s = ci.fr_to_mont(11), ci.fr_to_mont(13)
    curve = snarkjs_b200.getCurveFromName(name)
    try:
        pk = snarkjs_b200.groth16.ProvingKey(zkey, curve=curve)
        proof, public = snarkjs_b200.groth16.prove(pk, wtns, r, s)
        pk.release()
    finally:
        curve.terminate()
    want, wpub = orc.groth16_prove(zkey, wtns, r, s)
    assert proof == want and [int(p) for p in public] == [int(p) for p in wpub]
    assert orc.groth16_verify(orc.zkey_vk(zkey), [int(p) for p in public], proof)
