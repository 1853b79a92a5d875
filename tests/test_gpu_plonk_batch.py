"""GPU: sb_plonk_prove_batch.  Every batch proof is byte-identical to prove_raw of the same witness and blinders, and the
oracle's where checked (and verifies where the key is structured).  Covered: the reference fixture and circuit2, chain keys
of 13 to 16000 gates (4090: window-table commitments; 16000: 2^14 on unstructured points), several public inputs, deep
additions and BLS12-381; every way of running (sub-batches of 1 and 3, no window tables, MSM chunks shorter than a
row); a witness the reference rejects in the middle of a batch; the resident witness of sb_plonk_prove_resident; and launches that do not grow with K."""
import contextlib
import ctypes
import functools

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import oracle as O  # noqa: E402
from oracle import plonk as OP  # noqa: E402

from .test_host_plonk_batch import chain_witnesses  # noqa: E402

BN, BLS = O.BN254, O.BLS12_381
KS = (1, 2, 7, 32)
# (label, curve, n_gates, structured, n_pub, with_additions, deep)
SYNTH = [("g13", BN, 13, True, 1, True, False), ("g120", BN, 120, True, 1, True, False), ("g1000", BN, 1000, True, 1, True, False),
         ("g4090", BN, 4090, True, 1, True, False), ("g16000", BN, 16000, False, 1, True, False),
         ("pub5", BN, 60, True, 5, False, False), ("pub3", BN, 29, True, 3, True, False), ("deep", BN, 100, True, 1, True, True),
         ("bls", BLS, 120, True, 1, True, False)]


@pytest.fixture(scope="module")
def curves():
    import snarkjs_b200
    cs = {BN: snarkjs_b200.getCurveFromName("bn128"), BLS: snarkjs_b200.getCurveFromName("bls12381")}
    yield cs
    for c in cs.values():
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
    return [0x9000 + 104729 * i + 7919 * k for i in range(11)]


def blinders(cid, count):
    ci = O.CURVES[cid]
    return [b"".join(ci.fr_to_mont(b) for b in blinder_ints(k)) for k in range(count)]


@functools.lru_cache(maxsize=None)
def synth_case(label):
    """(zkey, [wtns, ...] of max(KS) distinct valid witnesses, structured)"""
    _, cid, n_gates, structured, n_pub, with_add, deep = next(s for s in SYNTH if s[0] == label)
    r = O.CURVES[cid].r
    gates, adds, n_vars, n_pub, wit = OP.chain_gates(n_gates, r=r, n_pub=n_pub, with_additions=with_add, deep_additions=deep)
    zkey = OP.plonk_setup_synth(gates, adds, n_vars, n_pub, tau=0xB47C + n_gates, structured=structured, curve=cid)
    return zkey, tuple(OP.wtns_bytes(w, r) for w in chain_witnesses(wit, max(KS), r)), structured


def payload(wtns):
    return np.frombuffer(O.read_wtns(wtns)[1], np.uint8)


def raw_batch(pk, ws, bls):
    """sb_plonk_prove_batch straight through the ABI: (rc, proof bytes per witness, status per witness)"""
    lib, c = pk.curve.lib, pk.curve
    w = np.concatenate([payload(x) for x in ws])
    bl = np.frombuffer(b"".join(bls), np.uint8)
    pb = lib.sb_plonk_proof_bytes(c.handle)
    out = np.full(len(ws) * pb, 0xA5, np.uint8)
    status = np.full(len(ws), -7, np.int32)
    rc = lib.sb_plonk_prove_batch(c.handle, pk.handle, w.ctypes.data_as(ctypes.c_void_p), w.size // 32 // len(ws), len(ws),
                                  bl.ctypes.data_as(ctypes.c_void_p), out.ctypes.data_as(ctypes.c_void_p), status.ctypes.data_as(ctypes.c_void_p))
    return rc, [out[i * pb:(i + 1) * pb].tobytes() for i in range(len(ws))], list(status)


def check_equal(pk, zkey, ws, cid, verify, oracle=True):
    import snarkjs_b200
    bls = blinders(cid, len(ws))
    got = pk.prove_batch_raw([payload(x) for x in ws], bls)
    for k, (x, b) in enumerate(zip(ws, bls)):
        assert got[k] == pk.prove_raw(payload(x), b), k
    if oracle:
        for k in range(min(2, len(ws))):
            obj = snarkjs_b200.plonk.proof_to_object(pk.curve, got[k])
            want, public = OP.plonk_prove(zkey, ws[k], blinder_ints(k))
            assert obj == want, k
            if verify:
                assert OP.plonk_verify(OP.plonk_vk(zkey), public, obj)
    return got


@pytest.mark.parametrize("count", KS)
@pytest.mark.parametrize("label", [s[0] for s in SYNTH])
def test_synthetic_batches_equal_single_proofs(curves, label, count):
    import snarkjs_b200
    zkey, wl, structured = synth_case(label)
    cid = next(s[1] for s in SYNTH if s[0] == label)
    pk = snarkjs_b200.plonk.ProvingKey(zkey, curves[cid])
    try:
        small = label not in ("g4090", "g16000")
        got = check_equal(pk, zkey, list(wl[:count]), cid, verify=structured and small, oracle=(count == 2 and (small or label == "g4090")))
        assert len(set(got)) == count
    finally:
        pk.release()


@pytest.mark.parametrize("count", KS)
def test_reference_keys(curves, golden, reference_plonk_key, count):
    """The reference's fixture key and its circuit2 key (domain 2048, 1001 additions, 4 public signals) with their own
    witnesses, repeated with distinct blinders."""
    import snarkjs_b200
    g = golden("plonk_case.npz")
    for zkey, wtns in ((bytes(g["zkey"]), bytes(g["wtns"])), reference_plonk_key(golden("plonk_setup_cases.npz"), "c2048")):
        pk = snarkjs_b200.plonk.ProvingKey(zkey, curves[BN])
        try:
            check_equal(pk, zkey, [wtns] * count, BN, verify=True, oracle=(count == 2))
        finally:
            pk.release()


def test_prove_batch_objects(curves):
    """plonk.prove_batch: the objects and public signals plonk.prove gives, in order."""
    import snarkjs_b200
    zkey, wl, _ = synth_case("pub3")
    pk = snarkjs_b200.plonk.ProvingKey(zkey, curves[BN])
    try:
        bls = blinders(BN, 3)
        got = snarkjs_b200.plonk.prove_batch(pk, list(wl[:3]), bls)
        assert got == [snarkjs_b200.plonk.prove(pk, w, b) for w, b in zip(wl[:3], bls)]
        assert len(snarkjs_b200.plonk.prove_batch(pk, list(wl[:2]))) == 2          # drawn blinders
    finally:
        pk.release()


def log_n(pk):
    """log2 of the key's domain size n, from sb_plonk_info"""
    lib, c = pk.curve.lib, pk.curve
    nv, npub, ds, na = (ctypes.c_uint32() for _ in range(4))
    assert lib.sb_plonk_info(c.handle, pk.handle, ctypes.byref(nv), ctypes.byref(npub), ctypes.byref(ds), ctypes.byref(na)) == 0
    return ds.value.bit_length() - 1


# MSM chunks of 2^(log2(n) + offset) points, shorter than the batch's rows of n + 6: the batch commits row by row, chunk by
# chunk, instead of one sorted MSM over all rows.  n / 2 puts a row over three chunks, n over two (the last of 6 points);
# either way the single path's T1 and T2 (n + 1 points) end one point into a chunk.
CHUNKED = {"chunked-half": -1, "chunked-n": 0}


@pytest.mark.parametrize("label", ["g1000", "g4090"])
@pytest.mark.parametrize("mode", ["sub1", "sub3", "no_tables"] + list(CHUNKED))
def test_every_way_of_running_gives_the_same_bytes(curves, label, mode):
    import snarkjs_b200
    zkey, wl, _ = synth_case(label)
    ws = list(wl[:7])
    bls = blinders(BN, 7)
    lib = curves[BN].lib
    pk = snarkjs_b200.plonk.ProvingKey(zkey, curves[BN])
    try:
        want = [pk.prove_raw(payload(x), b) for x, b in zip(ws, bls)]
        if mode in CHUNKED:
            chunk = [(6, log_n(pk) + CHUNKED[mode])]
            with tuning(lib, chunk):                                      # a key loaded before the setting
                assert pk.prove_batch_raw([payload(x) for x in ws], bls) == want
    finally:
        pk.release()
    # chunked: also without window tables, which makes g4090's commitments plain-mode MSMs past a chunk
    runs = [chunk, chunk + [(3, 1)]] if mode in CHUNKED else [{"sub1": [(14, 1)], "sub3": [(14, 3)], "no_tables": [(3, 1)]}[mode]]
    for settings in runs:
        with tuning(lib, settings):
            pk = snarkjs_b200.plonk.ProvingKey(zkey, curves[BN])        # loaded under the setting: no window tables in no_tables
            try:
                assert pk.prove_batch_raw([payload(x) for x in ws], bls) == want, settings
            finally:
                pk.release()


def test_errors_and_state(curves):
    import snarkjs_b200
    SbError = snarkjs_b200.SbError
    zkey, wl, _ = synth_case("g120")
    ws = list(wl[:5])
    bls = blinders(BN, 5)
    pk = snarkjs_b200.plonk.ProvingKey(zkey, curves[BN])
    lib, c = curves[BN].lib, curves[BN]
    try:
        # the resident witness of the single path, before any batch
        first = pk.prove_raw(payload(ws[0]), bls[0])
        res_before = pk.prove_raw(None, bls[1])
        # a wrong witness length: the reference's text, nothing written
        short = [payload(x)[:-32] for x in ws[:2]]
        w = np.concatenate(short)
        out = np.full(2 * lib.sb_plonk_proof_bytes(c.handle), 0xA5, np.uint8)
        bl = np.frombuffer(b"".join(bls[:2]), np.uint8)
        rc = lib.sb_plonk_prove_batch(c.handle, pk.handle, w.ctypes.data_as(ctypes.c_void_p), w.size // 64, 2,
                                      bl.ctypes.data_as(ctypes.c_void_p), out.ctypes.data_as(ctypes.c_void_p), None)
        assert rc != 0 and (out == 0xA5).all()
        assert lib.sb_last_error(c.handle).decode().startswith("Invalid witness length. Circuit: ")
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
        assert {3: "Copy constraints does not match", 4: "Polynomial is not divisible", 5: "T Polynomial is not well calculated"}[status[2]] == str(single_err.value)
        assert lib.sb_last_error(c.handle).decode() == str(single_err.value)
        assert proofs[2] == bytes(len(proofs[2]))
        for k in (0, 1, 3, 4):
            assert proofs[k] == pk.prove_raw(payload(bad[k]), bls[k]), k
        assert pk.prove_batch_raw([payload(x) for x in bad], bls)[2] is None
        with pytest.raises(SbError, match=str(single_err.value)):
            snarkjs_b200.plonk.prove_batch(pk, bad, bls)
        # the key still proves, and the single path's resident witness is the one it left
        assert pk.prove_batch_raw([payload(ws[0])], [bls[0]]) == [first]
        assert pk.prove_raw(payload(ws[0]), bls[0]) == first
        assert pk.prove_raw(None, bls[1]) == res_before
        pk.prove_batch_raw([payload(x) for x in ws], bls)
        assert pk.prove_raw(None, bls[1]) == res_before
    finally:
        pk.release()


def test_launches_scale_with_work_not_with_k(curves):
    import snarkjs_b200
    zkey, wl, _ = synth_case("g13")
    pk = snarkjs_b200.plonk.ProvingKey(zkey, curves[BN])
    lib, c = curves[BN].lib, curves[BN]
    try:
        with tuning(lib, [(14, 16)]):
            ws = [payload(x) for x in wl[:16]]
            bls = blinders(BN, 16)
            pk.prove_batch_raw(ws[:1], bls[:1])                       # warm: tables, cub scratch, buffers
            counts = []
            for k in (1, 16):
                before = lib.sb_launch_count(c.handle)
                pk.prove_batch_raw(ws[:k], bls[:k])
                counts.append(lib.sb_launch_count(c.handle) - before)
        assert counts[1] <= 1.25 * counts[0], counts
    finally:
        pk.release()
