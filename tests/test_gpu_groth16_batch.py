"""GPU: sb_groth16_prove_batch and sb_msm_registered_batch.  Every batch proof is byte-identical to prove_raw of the same
witness and (r, s), and the oracle's where checked; every batched MSM row equals multiExpRegistered on that row and the
oracle.  Covered: synthetic chain keys on both sides of the 2^12 window-table threshold, real circuit shapes (with a
duplicate witness and one whose private part is zero), every way of running (no tables, forced window sizes, sub-batches
of 1 and 3), the state the batch leaves (the resident witness) and the argument errors."""
import contextlib
import functools

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import oracle as O  # noqa: E402
from tests import msm_sets as MS  # noqa: E402
from tests import r1cs_shapes as S  # noqa: E402

BN, BLS = O.BN254, O.BLS12_381
KS = (1, 2, 7, 32)
SYNTH = [(BN, L) for L in (6, 11, 12, 14, 16)] + [(BLS, L) for L in (8, 12, 14)]


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


def rs_pairs(cid, count, seed=0):
    ci = O.CURVES[cid]
    return [(ci.fr_to_mont(1000 + 7 * i + seed), ci.fr_to_mont(5000 + 11 * i + seed)) for i in range(count)]


@functools.lru_cache(maxsize=None)
def chain_witnesses(cid, L, count=max(KS)):
    from snarkjs_b200 import synth
    r = O.CURVES[cid].r
    return tuple(synth.chain_witness(r, L, x0=3 + i, b=7 + 2 * i) for i in range(count))


_ZKEYS = {}


def synth_zkey(curves, cid, L):
    """The chain circuit's key with bases from the GPU generator (deterministic: the same bytes in every call)."""
    from snarkjs_b200 import synth
    if (cid, L) not in _ZKEYS:
        _ZKEYS[(cid, L)] = synth.synth_groth16_zkey(curves[cid], L)
    return _ZKEYS[(cid, L)]


def load(curves, cid, zkey):
    from snarkjs_b200 import groth16
    return groth16.ProvingKey(zkey, curve=curves[cid])


def singles(pk, ws, rs):
    return [pk.prove_raw(w, r, s) for w, (r, s) in zip(ws, rs)]


@pytest.mark.parametrize("cid,L", SYNTH, ids=[f"{'bn' if c == BN else 'bls'}-L{L}" for c, L in SYNTH])
def test_synthetic_batches_equal_single_proofs(curves, cid, L):
    from snarkjs_b200 import groth16, synth
    zkey = synth_zkey(curves, cid, L)
    ws = chain_witnesses(cid, L)
    rs = rs_pairs(cid, max(KS))
    pk = load(curves, cid, zkey)
    try:
        want = singles(pk, ws, rs)
        for K in KS:
            got = pk.prove_batch_raw(ws[:K], rs[:K])
            assert got == want[:K], (L, K, [i for i in range(K) if got[i] != want[i]])
        c = curves[cid]
        r = O.CURVES[cid].r
        for i in (0, max(KS) - 1):
            proof, _pub = O.groth16_prove(zkey, synth.wtns_container(r, ws[i]), *rs[i])
            assert groth16.proof_to_object(c, want[i]) == proof, (L, i)
    finally:
        pk.release()


SHAPE_CASES = ["empty", "bits", "public300", "bls_public17", "tiny1", "tiny2", "tiny4", "tiny7", "tiny49", "bls_tiny49",
               "ratio_both"]


def shape_witnesses(circ):
    """The circuit's witness, a copy of it, the private part zeroed, and the broken witness (which the reference proves)."""
    w = list(circ.w)
    zero = w[:circ.n_public + 1] + [0] * (circ.n_vars - circ.n_public - 1)
    out = [w, list(w), zero]
    try:
        out.append(circ.broken_witness())
    except ValueError:
        pass
    return out


@pytest.mark.parametrize("label", SHAPE_CASES)
def test_shape_batches_equal_oracle(curves, label):
    from snarkjs_b200 import groth16
    circ = S.case(label)
    c = curves[circ.curve]
    zkey = S.case_zkey(label)
    wl = shape_witnesses(circ)
    rs = rs_pairs(circ.curve, len(wl), seed=3)
    pk = groth16.ProvingKey(zkey, curve=c)
    try:
        got = groth16.prove_batch(pk, [circ.wtns(w) for w in wl], rs)
    finally:
        pk.release()
    for i, (w, (r, s)) in enumerate(zip(wl, rs)):
        proof, pub = O.groth16_prove(zkey, circ.wtns(w), r, s)
        assert got[i] == (proof, [str(x) for x in pub]), (label, i)


# (1, 1) and c = 22 (2^21 buckets per window, beyond the axis-sum design) take the running-sum reduction, which returns one
# window sum per window instead of five parts; (6, 8) cuts MSMs into 256-point chunks, which sends the 2^12 keys through
# the single-proof path proof by proof (the 2^6 key stays batched); (2, 1) runs every stream serialised on one.
MODES = {"no_tables": [(3, 1)], "c3": [(13, 3)], "c8": [(13, 8)], "c16": [(13, 16)], "c22": [(13, 22)],
         "force_reduce": [(1, 1)], "chunked": [(6, 8)], "split1": [(14, 1)], "split3": [(14, 3)], "serial": [(2, 1)]}
MODE_KEYS = [(BN, 6), (BN, 12), (BLS, 12)]
# c = 22 without window tables (the 2^6 key) would allocate 12 windows of 2^21 buckets per MSM and proof: not run
MODE_CASES = [(cid, L, m) for cid, L in MODE_KEYS for m in MODES if not (L == 6 and m == "c22")]


@pytest.mark.parametrize("cid,L,mode", MODE_CASES, ids=[f"{'bn' if c == BN else 'bls'}-L{L}-{m}" for c, L, m in MODE_CASES])
def test_every_way_of_running_gives_the_same_bytes(curves, cid, L, mode):
    """Tables and window sizes are chosen when the key is loaded, so the key is loaded under the setting; the single
    proofs are the reference bytes (a proof does not depend on how it was computed)."""
    from snarkjs_b200 import groth16
    zkey = synth_zkey(curves, cid, L)
    ws = chain_witnesses(cid, L)[:7]
    rs = rs_pairs(cid, 7, seed=5)
    pk = load(curves, cid, zkey)
    try:
        want = singles(pk, ws, rs)
    finally:
        pk.release()
    c = curves[cid]
    with tuning(c.lib, MODES[mode]):
        pk = groth16.ProvingKey(zkey, curve=c)
        try:
            assert pk.prove_batch_raw(ws, rs) == want, mode
        finally:
            pk.release()


def test_resident_witness_and_errors(curves):
    from snarkjs_b200 import groth16, SbError
    from snarkjs_b200.curve import _ptr
    cid, L = BN, 12
    c = curves[cid]
    zkey = synth_zkey(curves, cid, L)
    ws = chain_witnesses(cid, L)
    rs = rs_pairs(cid, 4, seed=9)
    pk = load(curves, cid, zkey)
    try:
        first = pk.prove_raw(ws[0], *rs[0])
        pk.prove_batch_raw(ws[1:4], rs[1:4])
        out = np.empty(8 * c.n8q, np.uint8)
        c.check(c.lib.sb_groth16_prove_resident(c.handle, pk.handle, *rs[0], _ptr(out)))
        assert out.tobytes() == first
        # a wrong witness length gives the reference's message
        w = np.concatenate([ws[0], ws[1]])
        with pytest.raises(SbError, match=f"Invalid witness length. Circuit: {pk.nVars}, witness: {pk.nVars - 1}"):
            c.check(c.lib.sb_groth16_prove_batch(c.handle, pk.handle, _ptr(w), pk.nVars - 1, 2, _ptr(np.zeros(64, np.uint8)),
                                                 _ptr(np.zeros(64, np.uint8)), _ptr(np.empty(16 * c.n8q, np.uint8))))
        # count = 0 writes nothing
        sentinel = np.full(8 * c.n8q, 0xA5, np.uint8)
        assert c.lib.sb_groth16_prove_batch(c.handle, pk.handle, None, pk.nVars, 0, None, None, _ptr(sentinel)) == 0
        assert (sentinel == 0xA5).all()
        assert pk.prove_batch_raw(np.zeros(0, np.uint8), []) == []
    finally:
        pk.release()
    # the per-proof path of keys longer than one MSM chunk does not touch the resident witness
    with tuning(c.lib, [(6, 8)]):
        pk = load(curves, cid, zkey)
        try:
            with pytest.raises(SbError, match="no witness resident"):
                c.check(c.lib.sb_groth16_prove_resident(c.handle, pk.handle, *rs[0], _ptr(out)))
            got = pk.prove_batch_raw(ws[1:3], rs[1:3])
            with pytest.raises(SbError, match="no witness resident"):
                c.check(c.lib.sb_groth16_prove_resident(c.handle, pk.handle, *rs[0], _ptr(out)))
            assert got == singles(pk, ws[1:3], rs[1:3])
            assert pk.prove_raw(ws[0], *rs[0]) == first
            pk.prove_batch_raw(ws[1:4], rs[1:4])
            c.check(c.lib.sb_groth16_prove_resident(c.handle, pk.handle, *rs[0], _ptr(out)))
            assert out.tobytes() == first
        finally:
            pk.release()
    # the Python wrapper's own checks
    pk = load(curves, cid, zkey)
    try:
        with pytest.raises(SbError, match="2 witnesses but 3"):
            pk.prove_batch_raw(ws[:2], rs[:3])
        with pytest.raises(SbError, match=f"Invalid witness length. Circuit: {pk.nVars}, witness: {pk.nVars - 1}"):
            pk.prove_batch_raw([ws[0], ws[1][:-32]], rs[:2])
        with pytest.raises(SbError, match="not 2 witnesses"):
            pk.prove_batch_raw(np.concatenate([ws[0], ws[1]])[:-16], rs[:2])
    finally:
        pk.release()
    shard = groth16.ProvingKey(zkey, curve=c, shard=0, n_shards=2)
    try:
        with pytest.raises(SbError, match="sharded"):
            shard.prove_batch_raw([ws[0]], [rs[0]])
    finally:
        shard.release()


MSM_N = (1, 100, 4096, 1 << 16)
MSM_COUNTS = (1, 3, 17)


def msm_rows(cid, n, count):
    """Rows of boundary scalars (0, 1, r - 1, 2^256 - 1 and the recoding edges), uniform and zero rows, interleaved."""
    kinds = ("boundary", "uniform", "zero", "uniform256")
    rows = [MS.scalar_set(cid, kinds[i % 4], n, 32, 8, seed=11 + i) for i in range(count)]
    return np.concatenate(rows)


@pytest.mark.parametrize("grp", (1, 2))
@pytest.mark.parametrize("cid", (BN, BLS), ids=["bn", "bls"])
def test_batched_msm_equals_row_by_row_and_oracle(curves, cid, grp):
    c = curves[cid]
    G = c.G1 if grp == 1 else c.G2
    for n in MSM_N:
        sets = ["random"] + list(MS.BASE_SETS) if n >= 100 else ["random"]
        for bs in sets:
            if n == 1 << 16 and bs != "random":
                continue
            bases = MS.random_bases(cid, grp, n) if bs == "random" else MS.base_set(cid, grp, bs, n)
            h = G.registerBases(bases)
            try:
                for count in MSM_COUNTS:
                    sc = msm_rows(cid, n, count)
                    got = G.multiExpRegisteredBatch(h, sc, count)
                    for k in range(count):
                        row = sc[k * n * 32:(k + 1) * n * 32]
                        assert got[k].tobytes() == G.multiExpRegistered(h, row).tobytes(), (n, bs, count, k)
                    if n <= 4096 and count == MSM_COUNTS[-1]:
                        for k in {0, count - 1}:
                            row = sc[k * n * 32:(k + 1) * n * 32]
                            want = O.g_to_affine(cid, grp, O.multiexp_affine(cid, grp, bases, row))
                            assert G.toAffine(got[k]).tobytes() == want, (n, bs, count, k)
                # a sub-range of the set, split into sub-batches of 2
                if n >= 100:
                    first, m = 17, n - 40
                    sc = msm_rows(cid, m, 5)
                    with tuning(c.lib, [(14, 2)]):
                        got = G.multiExpRegisteredBatch(h, sc, 5, first=first, n=m)
                    for k in range(5):
                        row = sc[k * m * 32:(k + 1) * m * 32]
                        assert got[k].tobytes() == G.multiExpRegistered(h, row, first=first, n=m).tobytes(), (n, bs, k)
            finally:
                c.lib.sb_bases_release(c.handle, h)
    assert G.multiExpRegisteredBatch(1, np.zeros(0, np.uint8), 0).shape == (0, G.sJacobian)


@pytest.mark.parametrize("grp", (1, 2))
@pytest.mark.parametrize("cid", (BN, BLS), ids=["bn", "bls"])
def test_batched_msm_on_the_running_sum_reduction(curves, cid, grp):
    """sb_set_tuning(1, 1), and a 2^12-point table built with c = 22, reduce with k_reduce / k_window_sum: one window sum
    per window, so the rows' window sums are packed more tightly than on the default path."""
    c = curves[cid]
    G = c.G1 if grp == 1 else c.G2
    for settings, ns in (([(1, 1)], (100, 4096)), ([(13, 22)], (4096,))):
        with tuning(c.lib, settings):
            for n in ns:
                bases = MS.random_bases(cid, grp, n)
                h = G.registerBases(bases)
                try:
                    sc = msm_rows(cid, n, 5)
                    got = G.multiExpRegisteredBatch(h, sc, 5)
                    for k in range(5):
                        row = sc[k * n * 32:(k + 1) * n * 32]
                        assert got[k].tobytes() == G.multiExpRegistered(h, row).tobytes(), (settings, n, k)
                    row = sc[4 * n * 32:]
                    want = O.g_to_affine(cid, grp, O.multiexp_affine(cid, grp, bases, row))
                    assert G.toAffine(got[4]).tobytes() == want, (settings, n)
                finally:
                    c.lib.sb_bases_release(c.handle, h)
