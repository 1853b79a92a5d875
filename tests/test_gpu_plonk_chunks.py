"""GPU: the PLONK and fflonk batch provers with rows longer than one MSM chunk.  A batch commits a sub-batch as one sorted
MSM over all its rows only while a row (n + 6 points for PLONK, 9n for fflonk) fits in one chunk; longer rows go one at a
time through msm_dev_accumulate, chunk by chunk.  fflonk takes that path unforced from n = 2^20 (9n > 2^23, the batch in
test_gpu_zz_bench_workloads.py); here sb_set_tuning(6, c) shrinks the chunk to 2^c points so that small keys take it too.
The expected bytes are always the unchunked prove_raw of the same witness and blinders, computed before the setting, and
the oracle's proof where stated.  test_gpu_plonk_batch.py and test_gpu_fflonk_batch.py run their mode tables at chunk sizes
at the rows' edges; this file holds what those tables cannot: a refused proof in a chunked batch, the fflonk key whose C0
is not the interleave, PLONK on BLS12-381, many tiny chunks, and the launch count that shows the row-by-row path runs."""
import pytest

pytestmark = pytest.mark.gpu

from oracle import fflonk as OF  # noqa: E402
from oracle import oracle as O  # noqa: E402
from oracle import plonk as OP  # noqa: E402

from tests import r1cs_shapes as S  # noqa: E402

from . import test_gpu_fflonk_batch as FB  # noqa: E402
from . import test_gpu_plonk_batch as PB  # noqa: E402

BN, BLS = O.BN254, O.BLS12_381
tuning = PB.tuning                    # sets (key, value) pairs for the block, then every key back to 0
payload = PB.payload
# the first error of a witness that breaks a copy constraint, by status code
STATUS_TEXT = {3: "Copy constraints does not match", 4: "Polynomial is not divisible"}


@pytest.fixture(scope="module")
def curves():
    import snarkjs_b200
    cs = {BN: snarkjs_b200.getCurveFromName("bn128"), BLS: snarkjs_b200.getCurveFromName("bls12381")}
    yield cs
    for c in cs.values():
        c.terminate()


def proto_of(proto):
    """(prover module, batch test module, blinders(count), blinder_ints(k), oracle prove, oracle vk, oracle verify)"""
    import snarkjs_b200
    if proto == "plonk":
        return (snarkjs_b200.plonk, PB, lambda k: PB.blinders(BN, k), PB.blinder_ints, OP.plonk_prove, OP.plonk_vk, OP.plonk_verify)
    return snarkjs_b200.fflonk, FB, FB.blinders, FB.blinder_ints, OF.fflonk_prove, OF.fflonk_vk, OF.fflonk_verify


def broken(wtns):
    """the witness with signal 4 off by one: it breaks a copy constraint of the chain keys"""
    wit = O.read_wtns(wtns)[1]
    ints = [int.from_bytes(bytes(wit[i * 32:(i + 1) * 32]), "little") for i in range(len(wit) // 32)]
    ints[4] = (ints[4] + 1) % O.P_BN_R
    return OP.wtns_bytes(ints)


@pytest.mark.parametrize("proto", ["plonk", "fflonk"])
def test_refused_proof_in_a_chunked_batch(curves, proto):
    """Index 2 of 5 breaks a copy constraint, with chunks of n / 2 (PLONK rows of two chunks and 6 points, fflonk rows of
    18 chunks): the same status, zero-filled slot and text as an unchunked batch, the other slots the unchunked single
    proofs, and the single path's resident witness untouched."""
    import snarkjs_b200
    mod, B, bls_of, *_ = proto_of(proto)
    zkey, wl, _ = B.synth_case("g120")
    ws = list(wl[:5])
    bls = bls_of(5)
    bad = ws[:2] + [broken(ws[2])] + ws[3:]
    c = curves[BN]
    pk = mod.ProvingKey(zkey, c)
    try:
        with pytest.raises(snarkjs_b200.SbError) as single_err:
            pk.prove_raw(payload(bad[2]), bls[2])
        want = [pk.prove_raw(payload(bad[k]), bls[k]) for k in (0, 1, 3, 4)]
        first = pk.prove_raw(payload(ws[0]), bls[0])                  # leaves ws[0] resident
        res_before = pk.prove_raw(None, bls[1])
        with tuning(c.lib, [(6, B.log_n(pk) - 1)]):
            rc, proofs, status = B.raw_batch(pk, bad, bls)
            err = c.lib.sb_last_error(c.handle).decode()
            assert pk.prove_raw(None, bls[1]) == res_before
        assert rc != 0
        assert [s != 0 for s in status] == [False, False, True, False, False], status
        assert STATUS_TEXT[status[2]] == str(single_err.value) == err
        assert proofs[2] == bytes(len(proofs[2]))
        assert proofs[:2] + proofs[3:] == want
        assert pk.prove_raw(None, bls[0]) == first
    finally:
        pk.release()


def test_c0_not_the_interleave_in_chunks(curves):
    """The fflonk key whose section 17 is not the interleave of sections 7-14 (14 power slots, C0's opening values in round
    3, W2 through commit_plain), batched with chunks of 2n: rows of 4.5 chunks.  Every slot is the unchunked single proof,
    and slot 0 the oracle's."""
    import snarkjs_b200
    zkey = bytearray(S.fflonk_zkey("bits"))
    _, secs = O.read_binfile(bytes(zkey), "zkey", 2)
    zkey[secs[17][0][0] + 5 * 32] ^= 1
    zkey = bytes(zkey)
    wtns = S.case("bits").wtns()
    c = curves[BN]
    bls = FB.blinders(3)
    pk = snarkjs_b200.fflonk.ProvingKey(zkey, c)
    try:
        want = [pk.prove_raw(payload(wtns), b) for b in bls]
        with tuning(c.lib, [(6, FB.log_n(pk) + 1)]):
            got = pk.prove_batch_raw([payload(wtns)] * 3, bls)
        assert got == want
        assert snarkjs_b200.fflonk.proof_to_object(c, got[0]) == OF.fflonk_prove(zkey, wtns, FB.blinder_ints(0))[0]
    finally:
        pk.release()


@pytest.mark.parametrize("label", ["bls", "bls-2^12"])
def test_plonk_bls12381_in_chunks(curves, label):
    """PLONK on BLS12-381 with chunks of n / 2: "bls" (n = 128, plain-mode commitments; slot 0 is also the oracle's proof,
    which verifies) and a 2^12 synthetic key (PTau of n + 6 >= 2^12 points: window-table commitments)."""
    import snarkjs_b200
    from snarkjs_b200 import synth
    c = curves[BLS]
    if label == "bls":
        zkey, wl, _ = PB.synth_case("bls")
        ws = [payload(x) for x in wl[:3]]
    else:
        zkey, wit = synth.synth_plonk_zkey(c, 12)
        ws = [wit] * 3
    bls = PB.blinders(BLS, 3)
    pk = snarkjs_b200.plonk.ProvingKey(zkey, c)
    try:
        want = [pk.prove_raw(w, b) for w, b in zip(ws, bls)]
        with tuning(c.lib, [(6, PB.log_n(pk) - 1)]):
            got = pk.prove_batch_raw(ws, bls)
        assert got == want
        if label == "bls":
            obj = snarkjs_b200.plonk.proof_to_object(c, got[0])
            oracle, public = OP.plonk_prove(zkey, wl[0], PB.blinder_ints(0))
            assert obj == oracle
            assert OP.plonk_verify(OP.plonk_vk(zkey), public, obj)
    finally:
        pk.release()


@pytest.mark.parametrize("proto", ["plonk", "fflonk"])
def test_many_tiny_chunks(curves, proto):
    """The smallest chain key (13 gates, n = 16) with chunks of 8 points: PLONK rows of n + 6 = 22 points are three chunks,
    the last of 6; fflonk rows of 9n are 18.  A batch of 7 equals the unchunked single proofs; slots 0 and 1 are the oracle's
    proofs and verify."""
    mod, B, bls_of, bl_ints, oprove, ovk, overify = proto_of(proto)
    zkey, wl, _ = B.synth_case("g13")
    ws = list(wl[:7])
    bls = bls_of(7)
    c = curves[BN]
    pk = mod.ProvingKey(zkey, c)
    try:
        want = [pk.prove_raw(payload(x), b) for x, b in zip(ws, bls)]
        with tuning(c.lib, [(6, 3)]):
            got = pk.prove_batch_raw([payload(x) for x in ws], bls)
        assert got == want
        for k in range(2):
            obj = mod.proof_to_object(c, got[k])
            oracle, public = oprove(zkey, ws[k], bl_ints(k))
            assert obj == oracle, k
            assert overify(ovk(zkey), public, obj), k
    finally:
        pk.release()


@pytest.mark.parametrize("proto", ["plonk", "fflonk"])
def test_launches_grow_with_k_in_chunks(curves, proto):
    """The mirror of test_launches_scale_with_work_not_with_k: with rows that fit a chunk, a batch of 4 launches about as many
    kernels as a batch of 1; with chunks of 8 points (rows of 3 chunks for PLONK, 18 for fflonk on the 13-gate key), every
    row is its own chain of MSMs, so a batch of 4 launches well over twice as many.  This is what tells the row-by-row path
    from the sorted one, which give the same bytes."""
    mod, B, bls_of, *_ = proto_of(proto)
    zkey, wl, _ = B.synth_case("g13")
    ws = [payload(x) for x in wl[:4]]
    bls = bls_of(4)
    c = curves[BN]
    lib = c.lib
    pk = mod.ProvingKey(zkey, c)

    def launches(k):
        before = lib.sb_launch_count(c.handle)
        pk.prove_batch_raw(ws[:k], bls[:k])
        return lib.sb_launch_count(c.handle) - before

    try:
        with tuning(lib, [(14, 4)]):
            pk.prove_batch_raw(ws[:1], bls[:1])                       # warm: tables, cub scratch, buffers
            whole = [launches(1), launches(4)]
        with tuning(lib, [(14, 4), (6, 3)]):
            pk.prove_batch_raw(ws[:1], bls[:1])
            chunked = [launches(1), launches(4)]
        print(f"{proto} launches, K = 1 and 4: rows in one chunk {whole}, rows of several chunks {chunked}")
        assert whole[1] <= 1.25 * whole[0], whole
        assert chunked[1] >= 2 * chunked[0], chunked
    finally:
        pk.release()
