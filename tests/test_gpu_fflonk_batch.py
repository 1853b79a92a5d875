"""GPU: sb_fflonk_prove_batch.  Every batch proof is byte-identical to prove_raw of the same witness and blinders, and the
oracle's where checked (and verifies where the key is structured).  Covered: the reference fixture, chain keys of 13 to
2000 gates (2000: window-table commitments), an unstructured 2^14 key, every BN254 shape key of tests/r1cs_shapes.py
(refused ones with the single path's text), a key whose C0 is not the interleave of its parts; every way of running
(sub-batches of 1 and 3, no window tables, serialised, MSM chunks shorter than a row); a witness the reference rejects in
the middle of a batch; the resident witness of sb_fflonk_prove_resident; and launches that do not grow with K."""
import contextlib
import ctypes
import functools

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import fflonk as OF  # noqa: E402
from oracle import oracle as O  # noqa: E402
from oracle import plonk as OP  # noqa: E402

from tests import r1cs_shapes as S  # noqa: E402

from .test_host_plonk_batch import chain_witnesses  # noqa: E402

BN = O.BN254
KS = (1, 2, 7, 32)
# (label, n_gates, structured, n_pub, with_additions, deep)
SYNTH = [("g13", 13, True, 1, True, False), ("g120", 120, True, 3, True, False), ("g500", 500, True, 1, False, False),
         ("deep", 100, True, 1, True, True), ("g2000", 2000, True, 1, True, False), ("g16000", 16000, False, 1, True, False)]


@pytest.fixture(scope="module")
def curve():
    import snarkjs_b200
    c = snarkjs_b200.getCurveFromName("bn128")
    yield c
    c.terminate()


@contextlib.contextmanager
def tuning(lib, settings):
    try:
        for k, v in settings:
            assert lib.sb_set_tuning(k, v) == 0, (k, v)
        yield
    finally:
        for k, _v in settings:
            lib.sb_set_tuning(k, 0)


def blinder_ints(k):
    return [0x6000 + 15485863 * i + 7919 * k for i in range(9)]


def blinders(count):
    ci = O.CURVES[BN]
    return [b"".join(ci.fr_to_mont(b) for b in blinder_ints(k)) for k in range(count)]


@functools.lru_cache(maxsize=None)
def synth_case(label):
    """(zkey, [wtns, ...] of max(KS) distinct valid witnesses, structured)"""
    _, n_gates, structured, n_pub, with_add, deep = next(s for s in SYNTH if s[0] == label)
    gates, adds, n_vars, n_pub, wit = OP.chain_gates(n_gates, n_pub=n_pub, with_additions=with_add, deep_additions=deep)
    zkey = OF.fflonk_setup_synth(gates, adds, n_vars, n_pub, tau=0xFF0B + n_gates, structured=structured)
    return zkey, tuple(OP.wtns_bytes(w) for w in chain_witnesses(wit, max(KS), O.P_BN_R)), structured


def payload(wtns):
    return np.frombuffer(O.read_wtns(wtns)[1], np.uint8)


def raw_batch(pk, ws, bls):
    """sb_fflonk_prove_batch straight through the ABI: (rc, proof bytes per witness, status per witness)"""
    lib, c = pk.curve.lib, pk.curve
    w = np.concatenate([payload(x) for x in ws])
    bl = np.frombuffer(b"".join(bls), np.uint8)
    pb = lib.sb_fflonk_proof_bytes(c.handle)
    out = np.full(len(ws) * pb, 0xA5, np.uint8)
    status = np.full(len(ws), -7, np.int32)
    rc = lib.sb_fflonk_prove_batch(c.handle, pk.handle, w.ctypes.data_as(ctypes.c_void_p), w.size // 32 // len(ws), len(ws),
                                   bl.ctypes.data_as(ctypes.c_void_p), out.ctypes.data_as(ctypes.c_void_p), status.ctypes.data_as(ctypes.c_void_p))
    return rc, [out[i * pb:(i + 1) * pb].tobytes() for i in range(len(ws))], list(status)


def check_equal(pk, zkey, ws, verify, oracle=True, bls=None):
    import snarkjs_b200
    bls = bls or blinders(len(ws))
    got = pk.prove_batch_raw([payload(x) for x in ws], bls)
    for k, (x, b) in enumerate(zip(ws, bls)):
        assert got[k] == pk.prove_raw(payload(x), b), k
    if oracle:
        for k in range(min(2, len(ws))):
            obj = snarkjs_b200.fflonk.proof_to_object(pk.curve, got[k])
            want, public = OF.fflonk_prove(zkey, ws[k], blinder_ints(k))
            assert obj == want, k
            if verify:
                assert OF.fflonk_verify(OF.fflonk_vk(zkey), public, obj)
    return got


@pytest.mark.parametrize("count", KS)
@pytest.mark.parametrize("label", [s[0] for s in SYNTH])
def test_synthetic_batches_equal_single_proofs(curve, label, count):
    import snarkjs_b200
    zkey, wl, structured = synth_case(label)
    pk = snarkjs_b200.fflonk.ProvingKey(zkey, curve)
    try:
        small = label not in ("g2000", "g16000")
        got = check_equal(pk, zkey, list(wl[:count]), verify=structured and small, oracle=(count == 2 and label != "g16000"))
        assert len(set(got)) == count
    finally:
        pk.release()


@pytest.mark.parametrize("count", KS)
def test_reference_fixture(curve, golden, count):
    import snarkjs_b200
    g = golden("fflonk_case.npz")
    zkey, wtns = bytes(g["zkey"]), bytes(g["wtns"])
    pk = snarkjs_b200.fflonk.ProvingKey(zkey, curve)
    try:
        check_equal(pk, zkey, [wtns] * count, verify=True, oracle=(count == 2))
    finally:
        pk.release()


@pytest.mark.parametrize("label", [label for label, c in S.PLONK_CASES.items() if c[1] == BN])
def test_shape_keys(curve, label):
    """Batches of three of every BN254 shape key; keys the reference rejects fail with the single path's text."""
    import snarkjs_b200
    zkey, wtns = S.fflonk_zkey(label), S.case(label).wtns()
    pk = snarkjs_b200.fflonk.ProvingKey(zkey, curve)
    try:
        bls = blinders(3)
        if label in S.FFLONK_ERRORS:
            rc, proofs, status = raw_batch(pk, [wtns] * 3, bls)
            assert rc != 0 and all(s != 0 for s in status)
            assert curve.lib.sb_last_error(curve.handle).decode() == S.FFLONK_ERRORS[label]
            assert proofs == [bytes(len(proofs[0]))] * 3
            with pytest.raises(snarkjs_b200.SbError, match=S.FFLONK_ERRORS[label]):
                pk.prove_raw(payload(wtns), bls[0])
        else:
            check_equal(pk, zkey, [wtns] * 3, verify=False, oracle=False, bls=bls)
    finally:
        pk.release()


def test_c0_not_the_interleave(curve):
    """A key whose section 17 differs from the interleave of sections 7-14: C0's eight opening values join round 3's
    reduction; batch, single path and oracle agree."""
    import snarkjs_b200
    zkey = bytearray(S.fflonk_zkey("bits"))
    _, secs = O.read_binfile(bytes(zkey), "zkey", 2)
    zkey[secs[17][0][0] + 5 * 32] ^= 1
    zkey = bytes(zkey)
    wtns = S.case("bits").wtns()
    pk = snarkjs_b200.fflonk.ProvingKey(zkey, curve)
    try:
        check_equal(pk, zkey, [wtns] * 3, verify=False, oracle=True)
    finally:
        pk.release()


def test_prove_batch_objects(curve):
    """fflonk.prove_batch: the objects and public signals fflonk.prove gives, in order."""
    import snarkjs_b200
    zkey, wl, _ = synth_case("g120")
    pk = snarkjs_b200.fflonk.ProvingKey(zkey, curve)
    try:
        bls = blinders(3)
        got = snarkjs_b200.fflonk.prove_batch(pk, list(wl[:3]), bls)
        assert got == [snarkjs_b200.fflonk.prove(pk, w, b) for w, b in zip(wl[:3], bls)]
        assert len(snarkjs_b200.fflonk.prove_batch(pk, list(wl[:2]))) == 2          # drawn blinders
    finally:
        pk.release()


def log_n(pk):
    """log2 of the key's domain size n, from sb_fflonk_info"""
    lib, c = pk.curve.lib, pk.curve
    nv, npub, ds, na = (ctypes.c_uint32() for _ in range(4))
    assert lib.sb_fflonk_info(c.handle, pk.handle, ctypes.byref(nv), ctypes.byref(npub), ctypes.byref(ds), ctypes.byref(na)) == 0
    return ds.value.bit_length() - 1


# MSM chunks of 2^(log2(n) + offset) points, shorter than the batch's rows of 9n: the batch commits row by row, chunk by
# chunk, instead of one sorted MSM over all rows.  A row of 9n is then exactly 9 chunks (n), 4.5 chunks (2n), or one whole
# chunk and n points (8n, where C1's 8n is exactly one chunk).
CHUNKED = {"chunked-n": 0, "chunked-2n": 1, "chunked-8n": 3}


@pytest.mark.parametrize("mode", ["sub1", "sub3", "no_tables", "serial"] + list(CHUNKED))
def test_every_way_of_running_gives_the_same_bytes(curve, mode):
    import snarkjs_b200
    zkey, wl, _ = synth_case("g2000")
    ws = list(wl[:7])
    bls = blinders(7)
    pk = snarkjs_b200.fflonk.ProvingKey(zkey, curve)
    try:
        want = [pk.prove_raw(payload(x), b) for x, b in zip(ws, bls)]
        if mode in CHUNKED:
            chunk = [(6, log_n(pk) + CHUNKED[mode])]
            with tuning(curve.lib, chunk):                                # a key loaded before the setting
                assert pk.prove_batch_raw([payload(x) for x in ws], bls) == want
    finally:
        pk.release()
    # chunked: also without window tables, which makes the commitments plain-mode MSMs past a chunk
    runs = ([chunk, chunk + [(3, 1)]] if mode in CHUNKED else
            [{"sub1": [(14, 1)], "sub3": [(14, 3)], "no_tables": [(3, 1)], "serial": [(2, 1)]}[mode]])
    for settings in runs:
        with tuning(curve.lib, settings):
            pk = snarkjs_b200.fflonk.ProvingKey(zkey, curve)        # loaded under the setting: no window tables in no_tables
            try:
                assert pk.prove_batch_raw([payload(x) for x in ws], bls) == want, settings
            finally:
                pk.release()


def test_errors_and_state(curve):
    import snarkjs_b200
    SbError = snarkjs_b200.SbError
    zkey, wl, _ = synth_case("g120")
    ws = list(wl[:5])
    bls = blinders(5)
    pk = snarkjs_b200.fflonk.ProvingKey(zkey, curve)
    lib, c = curve.lib, curve
    try:
        first = pk.prove_raw(payload(ws[0]), bls[0])
        res_before = pk.prove_raw(None, bls[1])
        # a wrong witness length: the reference's text, nothing written
        w = np.concatenate([payload(x)[:-32] for x in ws[:2]])
        out = np.full(2 * lib.sb_fflonk_proof_bytes(c.handle), 0xA5, np.uint8)
        bl = np.frombuffer(b"".join(bls[:2]), np.uint8)
        rc = lib.sb_fflonk_prove_batch(c.handle, pk.handle, w.ctypes.data_as(ctypes.c_void_p), w.size // 64, 2,
                                       bl.ctypes.data_as(ctypes.c_void_p), out.ctypes.data_as(ctypes.c_void_p), None)
        assert rc != 0 and (out == 0xA5).all()
        assert lib.sb_last_error(c.handle).decode().startswith("Invalid witness length. Circuit: ")
        assert lib.sb_fflonk_prove_batch(c.handle, pk.handle, None, w.size // 64, 0, None, None, None) != 0   # length first
        assert lib.sb_fflonk_prove_batch(c.handle, pk.handle, None, w.size // 64 + 1, 0, None, None, None) == 0  # count == 0
        assert lib.sb_fflonk_prove_batch(c.handle, pk.handle, None, w.size // 64 + 1, 2, None, None, None) != 0  # null pointers
        assert lib.sb_fflonk_prove_batch(c.handle, 999, None, 0, 0, None, None, None) != 0                   # bad handle
        # index 2 of 5 breaks a copy constraint
        wit = list(O.read_wtns(ws[2])[1])
        bad_ints = [int.from_bytes(bytes(wit[i * 32:(i + 1) * 32]), "little") for i in range(len(wit) // 32)]
        bad_ints[4] = (bad_ints[4] + 1) % O.P_BN_R
        bad = list(ws)
        bad[2] = OP.wtns_bytes(bad_ints)
        with pytest.raises(SbError) as single_err:
            pk.prove_raw(payload(bad[2]), bls[2])
        rc, proofs, status = raw_batch(pk, bad, bls)
        assert rc != 0
        assert [s != 0 for s in status] == [False, False, True, False, False]
        assert status[2] in (3, 4) and lib.sb_last_error(c.handle).decode() == str(single_err.value)
        assert proofs[2] == bytes(len(proofs[2]))
        for k in (0, 1, 3, 4):
            assert proofs[k] == pk.prove_raw(payload(bad[k]), bls[k]), k
        assert pk.prove_batch_raw([payload(x) for x in bad], bls)[2] is None
        with pytest.raises(SbError, match=str(single_err.value)):
            snarkjs_b200.fflonk.prove_batch(pk, bad, bls)
        # the key still proves, and the single path's resident witness is the one it left
        assert pk.prove_batch_raw([payload(ws[0])], [bls[0]]) == [first]
        assert pk.prove_raw(payload(ws[0]), bls[0]) == first
        assert pk.prove_raw(None, bls[1]) == res_before
        pk.prove_batch_raw([payload(x) for x in ws], bls)
        assert pk.prove_raw(None, bls[1]) == res_before
    finally:
        pk.release()


def test_launches_scale_with_work_not_with_k(curve):
    import snarkjs_b200
    zkey, wl, _ = synth_case("g13")
    pk = snarkjs_b200.fflonk.ProvingKey(zkey, curve)
    lib, c = curve.lib, curve
    try:
        with tuning(lib, [(14, 16)]):
            ws = [payload(x) for x in wl[:16]]
            bls = blinders(16)
            pk.prove_batch_raw(ws[:1], bls[:1])                       # warm: tables, cub scratch, buffers
            counts = []
            for k in (1, 16):
                before = lib.sb_launch_count(c.handle)
                pk.prove_batch_raw(ws[:k], bls[:k])
                counts.append(lib.sb_launch_count(c.handle) - before)
        assert counts[1] <= 1.25 * counts[0], counts
    finally:
        pk.release()
