"""GPU: Groth16 proofs of the circuits in tests/r1cs_shapes.py (Num2Bits rows, 2^14-term rows, edge coefficients, empty
sides, 0 to 300 public signals, full and just-overflowing domains, nVars far from the domain, and 1 to 400 signals)
are the oracle's bytes; the proofs from structured keys verify.  A subset repeats every proof in each way the library
can run it: the overlapped pipeline, serialised, without window tables, in small MSM chunks, as three point-range
shards, and from a wtns container with a second proof from the resident witness."""
import contextlib
import functools

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import oracle as O  # noqa: E402

from tests import r1cs_shapes as S  # noqa: E402

R, S_ = 0x5EED_0001, 0x5EED_0002


@pytest.fixture(scope="module")
def curves():
    import snarkjs_b200
    cs = {O.BN254: snarkjs_b200.getCurveFromName("bn128"), O.BLS12_381: snarkjs_b200.getCurveFromName("bls12381")}
    yield cs
    for c in cs.values():
        c.terminate()


def _rs(curve, r=R, s=S_):
    ci = O.CURVES[curve]
    return ci.fr_to_mont(r), ci.fr_to_mont(s)


@functools.lru_cache(maxsize=None)
def _oracle(label, r=R, s=S_, broken=False):
    circ = S.case(label)
    return O.groth16_prove(S.case_zkey(label), circ.wtns(circ.broken_witness() if broken else None), *_rs(circ.curve, r, s))


def _want(label, r=R, s=S_):
    proof, pub = _oracle(label, r, s)
    return proof, [str(x) for x in pub]


@contextlib.contextmanager
def _tuning(lib, settings):
    try:
        for k, v in settings:
            assert lib.sb_set_tuning(k, v) == 0
        yield
    finally:
        for k, _v in settings:
            lib.sb_set_tuning(k, 0)


def _prove(c, zkey, wtns, r, s):
    from snarkjs_b200 import groth16
    pk = groth16.ProvingKey(zkey, curve=c)
    try:
        return groth16.prove(pk, wtns, r, s)
    finally:
        pk.release()


@pytest.mark.parametrize("label", list(S.CASES))
def test_proof_equals_oracle(curves, label):
    circ = S.case(label)
    c = curves[circ.curve]
    proof, pub = _prove(c, S.case_zkey(label), circ.wtns(), *_rs(circ.curve))
    assert (proof, pub) == _want(label), repr(circ)
    if S.CASES[label][3]:
        assert O.groth16_verify(O.zkey_vk(S.case_zkey(label)), [int(x) for x in pub], proof), label


MODE_CASES = ["coeffs", "empty", "public300", "tiny1", "tiny7", "wide", "ratio_vars", "ratio_rows", "ratio_both",
              "bls_tiny200", "bls_ratio_both"]
TUNINGS = {"serial": [(2, 1)], "no_tables": [(3, 1)], "chunked": [(6, 8)]}


@pytest.mark.parametrize("mode", list(TUNINGS))
@pytest.mark.parametrize("label", MODE_CASES)
def test_tuned_modes_equal_oracle(curves, label, mode):
    """sb_set_tuning(2, 1) serialises the pipeline on one stream, (3, 1) ignores the window tables (at load and at
    proving time), (6, 8) cuts every MSM into chunks of 256 points (the chunked path of the prover)."""
    circ = S.case(label)
    c = curves[circ.curve]
    with _tuning(c.lib, TUNINGS[mode]):
        got = _prove(c, S.case_zkey(label), circ.wtns(), *_rs(circ.curve))
    assert got == _want(label), (label, mode)


@pytest.mark.parametrize("label", MODE_CASES)
def test_three_shards_equal_oracle(curves, label):
    """Three keys each loaded with one point range; the public signals' rows (C bases are padded for them) straddle a
    shard boundary in public300."""
    from snarkjs_b200 import groth16
    circ = S.case(label)
    c = curves[circ.curve]
    zkey = S.case_zkey(label)
    if label == "public300":
        per = -(-circ.n_vars // 3)
        assert per < circ.n_public + 1 < circ.n_vars and (circ.n_public + 1) % per
    r, s = _rs(circ.curve)
    keys = [groth16.ProvingKey(zkey, curve=c, shard=i, n_shards=3) for i in range(3)]
    try:
        w = circ.witness_array()
        parts = np.concatenate([keys[i].prove_shard(w, i, 3) for i in range(3)])
        assert groth16.proof_to_object(c, keys[0].finish(parts, 3, r, s)) == _want(label)[0], label
    finally:
        for k in keys:
            k.release()


@pytest.mark.parametrize("label", MODE_CASES)
def test_wtns_container_and_resident_witness_equal_oracle(curves, label):
    from snarkjs_b200 import groth16
    from snarkjs_b200.curve import _ptr
    circ = S.case(label)
    c = curves[circ.curve]
    pk = groth16.ProvingKey(S.case_zkey(label), curve=c)
    try:
        out = np.empty(8 * c.n8q, np.uint8)
        wt = np.frombuffer(circ.wtns(), np.uint8)
        c.check(c.lib.sb_groth16_prove_wtns(c.handle, pk.handle, _ptr(wt), wt.size, *_rs(circ.curve), _ptr(out)))
        assert groth16.proof_to_object(c, out.tobytes()) == _want(label)[0], label
        c.check(c.lib.sb_groth16_prove_resident(c.handle, pk.handle, *_rs(circ.curve, 11, 13), _ptr(out)))
        assert groth16.proof_to_object(c, out.tobytes()) == _want(label, 11, 13)[0], label
    finally:
        pk.release()


@pytest.mark.parametrize("label", ["bits", "coeffs", "empty", "public17", "ratio_vars", "ratio_both", "bls_coeffs"])
def test_shuffled_section4_gives_identical_bytes(curves, label):
    circ = S.case(label)
    got = _prove(curves[circ.curve], S.shuffle(S.case_zkey(label), 17), circ.wtns(), *_rs(circ.curve))
    assert got == _want(label), label


@pytest.mark.parametrize("label", ["coeffs", "empty", "tiny7", "ratio_rows", "bls_coeffs"])
def test_unsatisfying_witness_gives_the_oracle_bytes(curves, label):
    """The reference proves whatever witness it is given; so does the library, and the proof is the oracle's."""
    circ = S.case(label)
    bad = circ.broken_witness()
    got = _prove(curves[circ.curve], S.case_zkey(label), circ.wtns(bad), *_rs(circ.curve))
    proof, pub = _oracle(label, broken=True)
    assert got == (proof, [str(x) for x in pub]), label
    if S.CASES[label][3]:
        assert not O.groth16_verify(O.zkey_vk(S.case_zkey(label)), [int(x) for x in pub], proof)
