"""GPU: sb_plonk_verify_batch and sb_fflonk_verify_batch, with the Python wrappers plonk.verify / verify_batch and
fflonk.verify / verify_batch.

Proofs come from the device provers: on the reference's fixture keys they verify under the reference's vk.json and
public.json; on the synthetic keys of test_gpu_plonk_batch.py (BLS12-381 and 5 public inputs included), and on keys whose
public signals end the first Keccak absorb on a block boundary or number 1000, whole prove_batch batches verify.  Every
status is provoked at its reference priority by editing proof bytes through the ABI (every public index included), and a
sample of distinct items is compared with the oracle's verifiers on the wrapper-decoded proof, including BLS12-381
commitments that are on the curve but outside the r-subgroup.  Large batches repeat a checked pool, so every expected
status is known; at 1000 public signals the per-proof memory budget, not the proof count, splits them into sub-batches."""
import contextlib
import ctypes
import functools
import json
import os
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import fflonk as OF  # noqa: E402
from oracle import oracle as O  # noqa: E402
from oracle import pairing_bls as PB  # noqa: E402
from oracle import plonk as OP  # noqa: E402

BN, BLS = O.BN254, O.BLS12_381
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SB_ERR_ARG = -1
# label: (protocol, curve, gates, public inputs).  The rate labels put the first challenge's absorb on a whole number of
# Keccak blocks, so its padding takes a block of its own; the pub1000 labels run the per-proof public-input loops (PI(xi)
# and the transcript) far past the small counts.
SYNTH = {"plonk-g13": ("plonk", BN, 13, 1), "plonk-pub5": ("plonk", BN, 60, 5), "plonk-bls": ("plonk", BLS, 120, 1),
         "plonk-bls-pub5": ("plonk", BLS, 29, 5), "fflonk-g13": ("fflonk", BN, 13, 1), "fflonk-pub5": ("fflonk", BN, 60, 5),
         "plonk-rate12": ("plonk", BN, 60, 12), "plonk-bls-rate18": ("plonk", BLS, 60, 18), "fflonk-rate13": ("fflonk", BN, 60, 13),
         "plonk-pub1000": ("plonk", BN, 3000, 1000), "plonk-bls-pub1000": ("plonk", BLS, 3000, 1000),
         "fflonk-pub1000": ("fflonk", BN, 3000, 1000)}
KECCAK_RATE = 136


@pytest.fixture(scope="module")
def curves():
    import snarkjs_b200
    cs = {BN: snarkjs_b200.getCurveFromName("bn128"), BLS: snarkjs_b200.getCurveFromName("bls12381")}
    yield cs
    for c in cs.values():
        c.terminate()


@contextlib.contextmanager
def batch_cap(lib, v):
    assert lib.sb_set_tuning(14, v) == 0
    try:
        yield
    finally:
        lib.sb_set_tuning(14, 0)


def _golden(name):
    g = np.load(os.path.join(ROOT, "tests", "golden", name))
    return {k: bytes(g[k]) for k in g.files}


def mod(proto):
    import snarkjs_b200
    return snarkjs_b200.plonk if proto == "plonk" else snarkjs_b200.fflonk


def raw(c, proto, vkb, n_public, power, pubs: bytes, proofs: bytes, count: int):
    st = (ctypes.c_int32 * max(1, count))(*([-7] * max(1, count)))
    fn = c.lib.sb_plonk_verify_batch if proto == "plonk" else c.lib.sb_fflonk_verify_batch
    rc = fn(c.handle, vkb, len(vkb), n_public, power, pubs or None, proofs or None, count, st)
    return rc, list(st)[:count]


@functools.lru_cache(maxsize=None)
def synth(label):
    """(zkey, wtns, vk) of a synthetic structured key"""
    proto, cid, n_gates, n_pub = SYNTH[label]
    r = O.CURVES[cid].r
    gates, adds, n_vars, n_pub, wit = OP.chain_gates(n_gates, r=r, n_pub=n_pub)
    if proto == "plonk":
        zkey = OP.plonk_setup_synth(gates, adds, n_vars, n_pub, tau=0xC0DE + n_gates, curve=cid)
    else:
        zkey = OF.fflonk_setup_synth(gates, adds, n_vars, n_pub, tau=0xC0DE + n_gates)
    return zkey, OP.wtns_bytes(wit, r), mod(proto).verification_key(zkey)


def prove(curves, proto, cid, zkey, wtns, count):
    m = mod(proto)
    pk = m.ProvingKey(zkey, curves[cid])
    try:
        return m.prove_batch(pk, [wtns] * count)
    finally:
        pk.release()


# ---- reference fixtures --------------------------------------------------------------------------------------------------
def test_reference_fixtures(curves):
    g = _golden("plonk_case.npz")
    vk, pub = json.loads(g["vk_json"]), json.loads(g["public_json"])
    (proof, p2), = prove(curves, "plonk", BN, g["zkey"], g["wtns"], 1)
    assert p2 == pub
    assert mod("plonk").verify(vk, pub, proof, curve=curves[BN])
    stale = json.loads(g["proof_json"])
    assert not OP.plonk_verify(vk, pub, stale)
    assert mod("plonk").verify_status(vk, [(pub, stale)], curve=curves[BN]) == [1]     # passes every check, fails the pairing
    f = _golden("fflonk_case.npz")
    fvk, fpub = json.loads(f["vk_json"]), json.loads(f["public_json"])
    (fproof, fp2), = prove(curves, "fflonk", BN, f["zkey"], f["wtns"], 1)
    assert fp2 == fpub
    assert mod("fflonk").verify(fvk, fpub, fproof, curve=curves[BN])


def first_absorb(proto, cid, n_pub):
    """Bytes absorbed before the first challenge: PLONK's 8 key points, the publics and A, B, C; fflonk's C0, the publics
    and C1 (points uncompressed, signals 32 bytes)."""
    return (11 if proto == "plonk" else 2) * 2 * O.CURVES[cid].n8q + 32 * n_pub


@pytest.mark.parametrize("label", ["plonk-bls", "plonk-rate12", "plonk-bls-rate18", "fflonk-rate13"])
def test_rate_labels_fill_whole_keccak_blocks(label):
    proto, cid, _g, n_pub = SYNTH[label]
    assert first_absorb(proto, cid, n_pub) % KECCAK_RATE == 0


@pytest.mark.parametrize("label", list(SYNTH))
def test_prove_batch_verifies(curves, label):
    proto, cid, _g, _p = SYNTH[label]
    zkey, wtns, vk = synth(label)
    items = prove(curves, proto, cid, zkey, wtns, 5)
    assert mod(proto).verify_batch(vk, [(pub, p) for p, pub in items], curve=curves[cid]) == [True] * 5
    assert len({json.dumps(p, sort_keys=True) for p, _ in items}) == 5


# ---- statuses through the ABI --------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=None)
def pool(label):
    """(vk bytes, n_public, power, [(publics bytes, proof bytes, expected status), ...]): good proofs and edits of them, one
    per status cause, each at its reference priority."""
    import snarkjs_b200
    proto, cid, _g, n_pub = SYNTH[label]
    ci = O.CURVES[cid]
    n8, q, r = ci.n8q, ci.q, ci.r
    m = mod(proto)
    zkey, wtns, vk = synth(label)
    c = snarkjs_b200.getCurveFromName("bn128" if cid == BN else "bls12381")
    try:
        items = prove({cid: c}, proto, cid, zkey, wtns, 3)
    finally:
        c.terminate()
    out = []
    npts, nev, nchk = len(m.POINTS), len(m.EVALS), (6 if proto == "plonk" else 15)
    evb = 2 * n8 * npts
    for k, (proof, pub) in enumerate(items):
        pb = b"".join(int(s).to_bytes(32, "little") for s in pub)
        prf = m.proof_bytes(proof, n8, q, r)
        out.append((pb, prf, 0))
        if k:
            continue
        put = lambda b, o, v: b[:o] + v + b[o + len(v):]
        for i in range(npts):
            x = int.from_bytes(prf[2 * n8 * i:2 * n8 * i + n8], "little")
            y = int.from_bytes(prf[2 * n8 * i + n8:2 * n8 * (i + 1)], "little")
            out.append((pb, put(prf, 2 * n8 * i + n8, ((y + 1) % q).to_bytes(n8, "little")), 3))        # off the curve
            out.append((pb, put(prf, 2 * n8 * i, (x + q).to_bytes(n8, "little") if x + q < 1 << (8 * n8) else q.to_bytes(n8, "little")), 3))
            out.append((pb, put(prf, 2 * n8 * i, bytes(2 * n8)), 1))                                     # infinity
        for i in range(nchk):
            e = int.from_bytes(prf[evb + 32 * i:evb + 32 * (i + 1)], "little")
            out.append((pb, put(prf, evb + 32 * i, ((e + 1) % r).to_bytes(32, "little")), 1))
            out.append((pb, put(prf, evb + 32 * i, (e + r if e + r < 1 << 256 else r).to_bytes(32, "little")), 4))
        if proto == "fflonk":                                                                            # inv is not read
            out.append((pb, put(prf, evb + 32 * 15, (12345).to_bytes(32, "little")), 0))
        off = put(prf, n8, ((int.from_bytes(prf[n8:2 * n8], "little") + 1) % q).to_bytes(n8, "little"))
        big_ev = put(prf, evb, r.to_bytes(32, "little"))
        for j in range(n_pub):
            s = int(pub[j])
            out.append((put(pb, 32 * j, ((s + 1) % r).to_bytes(32, "little")), prf, 1))
            out.append((put(pb, 32 * j, r.to_bytes(32, "little")), prf, 2))
            out.append((put(pb, 32 * j, ((1 << 256) - 1).to_bytes(32, "little")), prf, 2))
            out.append((put(pb, 32 * j, r.to_bytes(32, "little")), big_ev, 4))                           # 4 before 2
            out.append((put(pb, 32 * j, r.to_bytes(32, "little")), off, 3))                              # 3 before 2
        out.append((pb, put(off, evb, r.to_bytes(32, "little")), 3))                                     # 3 before 4
    return m.vk_bytes(vk), n_pub, int(vk["power"]), out


@pytest.mark.parametrize("label", list(SYNTH))
def test_every_status_at_its_priority(curves, label):
    proto, cid, _g, _p = SYNTH[label]
    vkb, n_pub, power, items = pool(label)
    rc, st = raw(curves[cid], proto, vkb, n_pub, power, b"".join(i[0] for i in items), b"".join(i[1] for i in items), len(items))
    assert rc == 0
    assert st == [i[2] for i in items]


def _decoded(label, pb, prf):
    proto, cid, _g, n_pub = SYNTH[label]
    import snarkjs_b200
    ci = O.CURVES[cid]

    class C:   # what proof_to_object reads of a curve
        n8q, q, r, name = ci.n8q, ci.q, ci.r, "bn128" if cid == BN else "bls12381"
    pub = [str(int.from_bytes(pb[32 * j:32 * (j + 1)], "little")) for j in range(n_pub)]
    return pub, mod(proto).proof_to_object(C, prf)


def _off_subgroup(rng):
    q = O.P_BLS_Q
    while True:
        x = rng.randrange(q)
        rhs = (x ** 3 + 4) % q
        y = pow(rhs, (q + 1) // 4, q)
        if y * y % q == rhs and PB.g1_mul((x, y), O.P_BLS_R) is not None:
            return [str(x), str(y), "1"]


@pytest.mark.parametrize("label", ["plonk-pub5", "fflonk-pub5", "plonk-bls"])
def test_verdicts_match_the_oracle(curves, label):
    """Distinct items whose encodings are valid JSON (no coordinate >= q, no evaluation >= r), decoded by the wrapper's
    proof_to_object and checked by the oracle's verifier; BLS12-381 adds commitments outside the r-subgroup."""
    proto, cid, _g, _p = SYNTH[label]
    vkb, n_pub, power, items = pool(label)
    _zkey, _wtns, vk = synth(label)
    n8 = O.CURVES[cid].n8q
    rng = random.Random(11)
    picked = [it for it in items if it[2] == 0][:2] + rng.sample([it for it in items if it[2] == 1], 6 if cid == BN else 2)
    cases = [_decoded(label, pb, prf) for pb, prf, _ in picked]
    if cid == BLS:
        pub, proof = cases[0]
        for keys in (("T2",), ("Wxi", "T3")):
            bad = dict(proof)
            for k in keys:
                bad[k] = _off_subgroup(rng)
            cases.append((pub, bad))
    got = mod(proto).verify_batch(vk, cases, curve=curves[cid])
    oracle = OP.plonk_verify if proto == "plonk" else OF.fflonk_verify
    assert got == [oracle(vk, pub, proof) for pub, proof in cases]
    assert got[0] and got[1]


def test_wrong_counts_through_the_wrapper(curves):
    vkb, n_pub, power, items = pool("plonk-pub5")
    pub, proof = _decoded("plonk-pub5", items[0][0], items[0][1])
    _z, _w, vk = synth("plonk-pub5")
    st = mod("plonk").verify_status(vk, [(pub, proof), (pub[:4], proof), (pub + ["0"], proof), ([str(1 << 256)] + pub[1:], proof)],
                                    curve=curves[BN])
    assert st == [0, 5, 5, 2]
    fpub, fproof = _decoded("fflonk-pub5", pool("fflonk-pub5")[3][0][0], pool("fflonk-pub5")[3][0][1])
    _z, _w, fvk = synth("fflonk-pub5")
    assert mod("fflonk").verify_status(fvk, [(fpub, fproof), (fpub[:4], fproof)], curve=curves[BN]) == [0, 5]


# ---- large batches, sub-batches, edges -----------------------------------------------------------------------------------
@pytest.mark.parametrize("label", ["plonk-pub5", "plonk-bls", "fflonk-g13"])
def test_large_batches_across_sub_batches(curves, label):
    proto, cid, _g, _p = SYNTH[label]
    c = curves[cid]
    vkb, n_pub, power, items = pool(label)
    rng = random.Random(7)
    for cap, count in ((1, 9), (3, 200), (1000, 1 << 16), (0, 1 << 16)):
        order = [rng.randrange(len(items)) for _ in range(count)]
        pubs = b"".join(items[i][0] for i in order)
        prfs = b"".join(items[i][1] for i in order)
        with batch_cap(c.lib, cap):
            rc, st = raw(c, proto, vkb, n_pub, power, pubs, prfs, count)
        assert rc == 0
        assert st == [items[i][2] for i in order], (cap, count)
        assert c.lib.sb_last_ms(c.handle, 0) > 0


# the verify entries' sub-batch (api_verify.inl): min(count, VERIFY_CHUNK, VERIFY_BUDGET / per_proof); the scalars and
# point terms per proof (verify_plonk.cuh): PLONK 18 and 17, fflonk 5 and 5; launches per sub-batch: PLONK 4, fflonk 3
VERIFY_CHUNK, VERIFY_BUDGET = 1 << 15, 512 << 20
PV_SHAPE = {"plonk": (18, 17, 4), "fflonk": (5, 5, 3)}


@pytest.mark.parametrize("label", ["plonk-pub1000", "fflonk-pub1000"])
def test_budget_sub_batches(curves, label):
    """1000 public inputs: the 512 MiB budget, not the 2^15 chunk or a tuning cap, splits 2 chunk + 1 proofs into three
    sub-batches (seen in the launch count); tampered signals at the last and first index sit on both sides of each split."""
    proto, cid, _g, n_pub = SYNTH[label]
    c = curves[cid]
    vkb, n_pub, power, items = pool(label)
    n_sc, n_terms, launches = PV_SHAPE[proto]
    pb, prf, _ = items[0]
    per_proof = len(prf) + 32 * n_pub + 32 * n_sc + n_terms * 4 * c.n8q + 4     # proof, publics, scalars, XYZZ terms, status
    chunk = VERIFY_BUDGET // per_proof
    count = 2 * chunk + 1
    assert chunk < count < VERIFY_CHUNK
    r = O.CURVES[cid].r
    sig = lambda j, v: pb[:32 * j] + v.to_bytes(32, "little") + pb[32 * (j + 1):]
    last, first = int.from_bytes(pb[-32:], "little"), int.from_bytes(pb[:32], "little")
    edits = {chunk - 1: (sig(n_pub - 1, r), prf, 2), chunk: (sig(n_pub - 1, (last + 1) % r), prf, 1),
             2 * chunk - 1: (sig(0, (first + 1) % r), prf, 1), 2 * chunk: (sig(0, r), prf, 2)}
    valid = [it for it in items if it[2] == 0]
    rng = random.Random(13)
    order = [edits[k] if k in edits else valid[rng.randrange(len(valid))] for k in range(count)]
    before = c.lib.sb_launch_count(c.handle)
    with batch_cap(c.lib, 0):
        rc, st = raw(c, proto, vkb, n_pub, power, b"".join(i[0] for i in order), b"".join(i[1] for i in order), count)
    assert rc == 0
    assert c.lib.sb_launch_count(c.handle) - before == 1 + 3 * launches     # prepare, then each sub-batch's kernels
    assert [st[k] for k in sorted(edits)] == [edits[k][2] for k in sorted(edits)]
    assert st == [i[2] for i in order]


def test_batch_of_one_equals_verify_and_count_zero(curves):
    vkb, n_pub, power, items = pool("plonk-g13")
    _z, _w, vk = synth("plonk-g13")
    c = curves[BN]
    # good, off the curve, infinity, off the curve with an evaluation = r; not the coordinate >= q edit (items[2]), which
    # JSON cannot carry: G.fromObject takes coordinates mod q
    for pb, prf, want in (items[0], items[1], items[3], items[-1]):
        pub, proof = _decoded("plonk-g13", pb, prf)
        assert mod("plonk").verify(vk, pub, proof, curve=c) == (want == 0)
        assert raw(c, "plonk", vkb, n_pub, power, pb, prf, 1) == (0, [want])
    st = (ctypes.c_int32 * 2)(-7, -7)
    assert c.lib.sb_plonk_verify_batch(c.handle, vkb, len(vkb), n_pub, power, items[0][0], items[0][1], 0, st) == 0
    assert list(st) == [-7, -7]


def test_argument_errors(curves):
    c = curves[BN]
    vkb, n_pub, power, items = pool("plonk-g13")
    pb, prf, _ = items[0]

    def refused(proto, vk, n_public, pw, pubs, proofs, match, cv=c):
        st = (ctypes.c_int32 * 1)(-7)
        fn = cv.lib.sb_plonk_verify_batch if proto == "plonk" else cv.lib.sb_fflonk_verify_batch
        assert fn(cv.handle, vk, len(vk) if vk else 0, n_public, pw, pubs, proofs, 1, st) == SB_ERR_ARG
        assert match in cv.lib.sb_last_error(cv.handle).decode()
        assert st[0] == -7

    refused("plonk", vkb[:-1], n_pub, power, pb, prf, "vk_len")
    refused("plonk", None, n_pub, power, pb, prf, "vk_len")
    refused("plonk", vkb, n_pub, power, None, prf, "null buffer")
    refused("plonk", vkb, n_pub, power, pb, None, "null buffer")
    for pw in (29, 1 << 31, 0xFFFFFFFF):          # unsigned: no power wraps below the 2-adicity
        refused("plonk", vkb, n_pub, pw, pb, prf, "2-adicity")
    off = vkb[:32] + ((int.from_bytes(vkb[32:64], "little") + 1) % O.P_BN_Q).to_bytes(32, "little") + vkb[64:]
    refused("plonk", off, n_pub, power, pb, prf, "not on its curve")
    big = vkb[:20 * 32 - 128] + O.P_BN_Q.to_bytes(32, "little") + vkb[20 * 32 - 96:]       # X_2.x.c0 = q
    refused("plonk", big, n_pub, power, pb, prf, "not on its curve")
    fvkb, fn_pub, fpower, fitems = pool("fflonk-g13")
    refused("fflonk", fvkb, fn_pub, 0xFFFFFFFF, fitems[0][0], fitems[0][1], "2-adicity")
    refused("fflonk", fvkb[:-32], fn_pub, fpower, fitems[0][0], fitems[0][1], "vk_len")
    refused("fflonk", fvkb, fn_pub, fpower, fitems[0][0], fitems[0][1], "bn128 only", cv=curves[BLS])
    # through the wrappers: a power of -1 reaches the C entry as 2^32 - 1 and is refused, not read as an index
    _z, _w, vk = synth("plonk-g13")
    pub, proof = _decoded("plonk-g13", pb, prf)
    with pytest.raises(mod("plonk").SbError, match="2-adicity"):
        mod("plonk").verify(dict(vk, power=-1), pub, proof, curve=c)
    _z, _w, fvk = synth("fflonk-g13")
    fpub, fproof = _decoded("fflonk-g13", fitems[0][0], fitems[0][1])
    with pytest.raises(mod("fflonk").SbError, match="2-adicity"):
        mod("fflonk").verify_batch(dict(fvk, power=-1), [(fpub, fproof)], curve=c)
    # a key point off its curve raises (the reference would decode it unchecked and return a verdict)
    bad_x2 = dict(vk, X_2=[vk["X_2"][0], [vk["X_2"][1][0], str((int(vk["X_2"][1][1]) + 1) % O.P_BN_Q)], ["1", "0"]])
    with pytest.raises(mod("plonk").SbError, match="not on its curve"):
        mod("plonk").verify(bad_x2, pub, proof, curve=c)
    assert curves[BLS].lib.sb_plonk_verify_batch(curves[BLS].handle, vkb, len(vkb), n_pub, power, pb, prf, 1,
                                                 (ctypes.c_int32 * 1)()) == SB_ERR_ARG    # a BN254 key on BLS12-381: wrong length
