"""GPU: PLONK and fflonk proofs of the keys plonk_setup / fflonk_setup build from the circuits in tests/r1cs_shapes.py
(PLONK_CASES: the minimum domain of 8, 0 to 300 public signals, Num2Bits' 252-addition chain, edge coefficients in the
selectors, gate counts that fill or just overflow the domain, commitments on both sides of the window-table threshold,
domain 2^14, BLS12-381) are the oracle's bytes with the same blinders, and verify where the key is structured.  PLONK
proofs also run from the resident witness, without window tables, serialised, and in batches (sb_plonk_prove_batch) with a
refused proof in the middle; keys the reference refuses (a repeated signal, nPublic = 0) fail with its text on every path.
fflonk proves every BN254 case, including nPublic = 0, and a key whose section 17 is not the interleave of sections 7-14."""
import contextlib
import ctypes
import functools
import re

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import fflonk as OF  # noqa: E402
from oracle import oracle as O  # noqa: E402
from oracle import plonk as OP  # noqa: E402

from tests import r1cs_shapes as S  # noqa: E402

BN, BLS = O.BN254, O.BLS12_381
CODES = {3: "Copy constraints does not match", 4: "Polynomial is not divisible", 5: "T Polynomial is not well calculated",
         6: "Evaluations.getEvaluation() out of bounds"}

PLONK_LABELS = list(S.PLONK_CASES)
FFLONK_LABELS = [label for label, c in S.PLONK_CASES.items() if c[1] == BN]
PLONK_GOOD = [label for label in PLONK_LABELS if label not in S.PLONK_ERRORS]
# domains 8 and 32, 300 Lagrange terms, a 252-addition chain, 4102 / 8198 commitment points (window tables) and 2^14
TUNED = ["tiny2", "tiny4", "tiny7", "public2", "tiny48", "tiny64", "public300", "bits", "gates12+0", "gates12+1", "wide4096"]
TUNINGS = {"no_tables": [(3, 1)], "serial": [(2, 1)]}
BATCH = TUNED + ["bls_bits", "bls_public17", "bls_tiny362", "bls_tiny363", "bls_ratio_rows"]
BROKEN = ["tiny7", "tiny64", "public300", "bits", "gates12+0", "wide4096", "bls_bits", "bls_tiny362"]


@pytest.fixture(scope="module")
def curves():
    import snarkjs_b200
    cs = {BN: snarkjs_b200.getCurveFromName("bn128"), BLS: snarkjs_b200.getCurveFromName("bls12381")}
    yield cs
    for c in cs.values():
        c.terminate()


@contextlib.contextmanager
def _tuning(lib, settings):
    try:
        for k, v in settings:
            assert lib.sb_set_tuning(k, v) == 0, (k, v)
        yield
    finally:
        for k, _v in settings:
            lib.sb_set_tuning(k, 0)


def _plonk_blinders(k):
    return [0x7000 + 104729 * i + 15485863 * k for i in range(11)]


def _fflonk_blinders(k):
    return [0x8000 + 1299709 * i + 7919 * k for i in range(9)]


def _mont(curve, ints):
    ci = O.CURVES[curve]
    return b"".join(ci.fr_to_mont(x) for x in ints)


def _witness(label, broken=False):
    circ = S.case(label)
    return circ.wtns(circ.broken_witness() if broken else None)


def _payload(wtns):
    return np.frombuffer(O.read_wtns(wtns)[1], np.uint8)


@functools.lru_cache(maxsize=None)
def _plonk_oracle(label, k=0, broken=False):
    """(proof, public signals) of oracle.plonk with blinder set k, or the text of the reference's error"""
    try:
        return OP.plonk_prove(S.plonk_zkey(label), _witness(label, broken), _plonk_blinders(k))
    except ValueError as e:
        return str(e)


@functools.lru_cache(maxsize=None)
def _fflonk_oracle(label, k=0):
    try:
        return OF.fflonk_prove(S.fflonk_zkey(label), _witness(label), _fflonk_blinders(k))
    except ValueError as e:
        return str(e)


@contextlib.contextmanager
def _plonk_key(c, label):
    from snarkjs_b200 import plonk
    pk = plonk.ProvingKey(S.plonk_zkey(label), curve=c)
    try:
        yield pk
    finally:
        pk.release()


def _raw_batch(pk, ws, bls):
    """sb_plonk_prove_batch through the ABI: (rc, proof bytes per witness, status per witness)"""
    lib, c = pk.curve.lib, pk.curve
    w = np.concatenate([_payload(x) for x in ws])
    bl = np.frombuffer(b"".join(bls), np.uint8)
    pb = lib.sb_plonk_proof_bytes(c.handle)
    out = np.full(len(ws) * pb, 0xA5, np.uint8)
    status = np.full(len(ws), -7, np.int32)
    rc = lib.sb_plonk_prove_batch(c.handle, pk.handle, w.ctypes.data_as(ctypes.c_void_p), w.size // 32 // len(ws), len(ws),
                                  bl.ctypes.data_as(ctypes.c_void_p), out.ctypes.data_as(ctypes.c_void_p), status.ctypes.data_as(ctypes.c_void_p))
    return rc, [out[i * pb:(i + 1) * pb].tobytes() for i in range(len(ws))], [int(s) for s in status]


# ------------------------------------------------------------------------------------------------------------ PLONK
@pytest.mark.parametrize("label", PLONK_LABELS)
def test_plonk_proof_and_resident_proof_equal_oracle(curves, label):
    """plonk.prove with blinder set 0, then sb_plonk_prove_resident with set 1; keys the reference refuses fail with its
    text on both paths (the refused witness stays resident)."""
    from snarkjs_b200 import SbError, plonk
    circ = S.case(label)
    c = curves[circ.curve]
    with _plonk_key(c, label) as pk:
        want = _plonk_oracle(label)
        if isinstance(want, str):
            assert want == S.PLONK_ERRORS[label]
            with pytest.raises(SbError, match=f"^{re.escape(want)}$"):
                plonk.prove(pk, circ.wtns(), _mont(circ.curve, _plonk_blinders(0)))
            with pytest.raises(SbError, match=f"^{re.escape(want)}$"):
                pk.prove_raw(None, _mont(circ.curve, _plonk_blinders(1)))
            return
        got = plonk.prove(pk, circ.wtns(), _mont(circ.curve, _plonk_blinders(0)))
        assert got == want, label
        if S.PLONK_CASES[label][3]:
            assert OP.plonk_verify(OP.plonk_vk(S.plonk_zkey(label)), got[1], got[0]), label
        raw = pk.prove_raw(None, _mont(circ.curve, _plonk_blinders(1)))
        assert plonk.proof_to_object(c, raw) == _plonk_oracle(label, 1)[0], label


@pytest.mark.parametrize("mode", list(TUNINGS))
@pytest.mark.parametrize("label", TUNED)
def test_plonk_tuned_modes_equal_oracle(curves, label, mode):
    """sb_set_tuning(3, 1) loads and proves without window tables; (2, 1) serialises the pipeline on one stream."""
    from snarkjs_b200 import plonk
    circ = S.case(label)
    c = curves[circ.curve]
    with _tuning(c.lib, TUNINGS[mode]), _plonk_key(c, label) as pk:
        got = plonk.prove(pk, circ.wtns(), _mont(circ.curve, _plonk_blinders(0)))
    assert got == _plonk_oracle(label), (label, mode)


@pytest.mark.parametrize("label", BATCH)
def test_plonk_batch_equals_single_proofs(curves, label):
    """Three proofs with distinct blinders in one batch, then in sub-batches of one proof (sb_set_tuning(14, 1))."""
    from snarkjs_b200 import plonk
    circ = S.case(label)
    c = curves[circ.curve]
    ws = [_payload(circ.wtns())] * 3
    bls = [_mont(circ.curve, _plonk_blinders(k)) for k in range(3)]
    with _plonk_key(c, label) as pk:
        got = pk.prove_batch_raw(ws, bls)
        assert got == [pk.prove_raw(w, b) for w, b in zip(ws, bls)], label
        assert len(set(got)) == 3
        assert plonk.proof_to_object(c, got[0]) == _plonk_oracle(label)[0], label
        with _tuning(c.lib, [(14, 1)]):
            assert pk.prove_batch_raw(ws, bls) == got, label


@pytest.mark.parametrize("label", BROKEN)
def test_plonk_batch_refused_proof_in_the_middle(curves, label):
    """broken_witness() at index 2 of 5: its slot is zero-filled with the oracle's error as status and text; the others
    are the single proofs."""
    from snarkjs_b200 import SbError, plonk
    circ = S.case(label)
    c = curves[circ.curve]
    want_bad = _plonk_oracle(label, 2, broken=True)
    assert isinstance(want_bad, str), label
    ws = [_witness(label)] * 2 + [_witness(label, broken=True)] + [_witness(label)] * 2
    bls = [_mont(circ.curve, _plonk_blinders(k)) for k in range(5)]
    with _plonk_key(c, label) as pk:
        rc, proofs, status = _raw_batch(pk, ws, bls)
        assert rc != 0 and status[:2] == [0, 0] and status[3:] == [0, 0], status
        assert CODES[status[2]] == want_bad == c.lib.sb_last_error(c.handle).decode()
        assert proofs[2] == bytes(len(proofs[2]))
        for k in (0, 1, 3, 4):
            assert proofs[k] == pk.prove_raw(_payload(ws[k]), bls[k]), k
        assert plonk.proof_to_object(c, proofs[0]) == _plonk_oracle(label)[0]
        with pytest.raises(SbError, match=f"^{re.escape(want_bad)}$"):
            plonk.prove_batch(pk, ws, bls)


@pytest.mark.parametrize("label", list(S.PLONK_ERRORS))
def test_plonk_batch_of_a_refused_key(curves, label):
    """A key no witness proves (a repeated signal; nPublic = 0): every proof of a batch fails with the reference's text and
    a zero-filled slot, and the context then proves another key."""
    from snarkjs_b200 import plonk
    circ = S.case(label)
    c = curves[circ.curve]
    want = _plonk_oracle(label)
    assert want == S.PLONK_ERRORS[label]
    ws = [_witness(label)] * 3
    bls = [_mont(circ.curve, _plonk_blinders(k)) for k in range(3)]
    with _plonk_key(c, label) as pk:
        rc, proofs, status = _raw_batch(pk, ws, bls)
        assert rc != 0 and [CODES[s] for s in status] == [want] * 3
        assert c.lib.sb_last_error(c.handle).decode() == want
        assert proofs == [bytes(len(proofs[0]))] * 3
    with _plonk_key(c, "tiny2") as pk:
        assert plonk.prove(pk, _witness("tiny2"), _mont(BN, _plonk_blinders(0))) == _plonk_oracle("tiny2")


# ------------------------------------------------------------------------------------------------------------ fflonk
@pytest.mark.parametrize("label", FFLONK_LABELS)
def test_fflonk_proof_and_resident_proof_equal_oracle(curves, label):
    from snarkjs_b200 import SbError, fflonk
    circ = S.case(label)
    c = curves[BN]
    zkey = S.fflonk_zkey(label)
    pk = fflonk.ProvingKey(zkey, curve=c)
    try:
        want = _fflonk_oracle(label)
        if isinstance(want, str):
            assert want == S.FFLONK_ERRORS[label]
            with pytest.raises(SbError, match=f"^{re.escape(want)}$"):
                fflonk.prove(pk, circ.wtns(), _mont(BN, _fflonk_blinders(0)))
            return
        got = fflonk.prove(pk, circ.wtns(), _mont(BN, _fflonk_blinders(0)))
        assert got == want, label
        if S.PLONK_CASES[label][3]:
            assert OF.fflonk_verify(OF.fflonk_vk(zkey), got[1], got[0]), label
        raw = pk.prove_raw(None, _mont(BN, _fflonk_blinders(1)))
        assert fflonk.proof_to_object(c, raw) == _fflonk_oracle(label, 1)[0], label
    finally:
        pk.release()


def test_fflonk_c0_section_not_the_interleave(curves):
    """One flipped bit in section 17: the prover evaluates C0 from section 17 itself, as the reference does, instead of
    from sections 7-14 (the GPU side of tests/test_host_fflonk.py's test of the same name)."""
    from snarkjs_b200 import fflonk
    zkey = bytearray(S.fflonk_zkey("bits"))
    data, secs = O.read_binfile(bytes(zkey), "zkey", 2)
    zkey[secs[17][0][0] + 5 * 32] ^= 1
    zkey = bytes(zkey)
    wtns = _witness("bits")
    want = OF.fflonk_prove(zkey, wtns, _fflonk_blinders(0))
    pk = fflonk.ProvingKey(zkey, curve=curves[BN])
    try:
        assert fflonk.prove(pk, wtns, _mont(BN, _fflonk_blinders(0))) == want
    finally:
        pk.release()
    assert not OF.fflonk_verify(OF.fflonk_vk(zkey), want[1], want[0])
