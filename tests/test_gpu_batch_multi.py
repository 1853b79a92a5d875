"""GPU: batches of one key split over several contexts (sb_*_load_replicas / sb_*_prove_batch_multi).  The contexts sit on
device 0 unless stated, and every proof must be the single-context batch's proof of the same witness and randomness, byte
for byte.  Covered: Groth16 on BN254 and BLS12-381 at 2^10 and 2^14, PLONK on both curves and fflonk, over 1, 2 and 3
contexts, with counts of 0, 1, 2 (fewer proofs than contexts), 7 and 33, with and without sub-batches of 2; refused
PLONK / fflonk witnesses in two ranks' ranges; the argument refusals; what replica handles do on the other entries; and
distinct devices when there are several."""
import contextlib
import ctypes
import functools

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import fflonk as OF  # noqa: E402
from oracle import oracle as O  # noqa: E402
from oracle import plonk as OP  # noqa: E402

BN, BLS = O.BN254, O.BLS12_381
NAME = {BN: "bn128", BLS: "bls12381"}
RANKS = (1, 2, 3)
COUNTS = (0, 1, 2, 7, 33)
TUNINGS = {"free": (), "sub2": ((14, 2),)}
# (label, protocol, curve, size: log2 of the Groth16 domain, or the PLONK / fflonk chain's gate count)
KEYS = [("g16-bn-10", "groth16", BN, 10), ("g16-bn-14", "groth16", BN, 14), ("g16-bls-10", "groth16", BLS, 10),
        ("g16-bls-14", "groth16", BLS, 14), ("plonk-bn", "plonk", BN, 120), ("plonk-bls", "plonk", BLS, 120),
        ("fflonk-bn", "fflonk", BN, 120)]
N_BLINDERS = {"plonk": 11, "fflonk": 9}


@pytest.fixture(scope="module")
def ctxs():
    """three contexts per curve, all on device 0"""
    import snarkjs_b200
    cs = {cid: [snarkjs_b200.getCurveFromName(NAME[cid]) for _ in range(3)] for cid in (BN, BLS)}
    yield cs
    for lst in cs.values():
        for c in lst:
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


def module(proto):
    from snarkjs_b200 import fflonk, groth16, plonk
    return {"groth16": groth16, "plonk": plonk, "fflonk": fflonk}[proto]


def blinder_ints(proto, k):
    return [0x7100 + 104729 * i + 7919 * k for i in range(N_BLINDERS[proto])]


@functools.lru_cache(maxsize=None)
def case(label):
    """(zkey, witness payloads, randomness) of max(COUNTS) proofs: Groth16 (r, s) pairs over distinct chain witnesses, or
    PLONK / fflonk blinder strings over one chain witness"""
    _, proto, cid, size = next(k for k in KEYS if k[0] == label)
    ci = O.CURVES[cid]
    count = max(COUNTS)
    if proto == "groth16":
        import snarkjs_b200
        from snarkjs_b200 import synth
        c = snarkjs_b200.getCurveFromName(NAME[cid])
        try:
            zkey = synth.synth_groth16_zkey(c, size)
        finally:
            c.terminate()
        ws = tuple(synth.chain_witness(ci.r, size, x0=3 + i, b=7 + 2 * i).tobytes() for i in range(count))
        rand = tuple((ci.fr_to_mont(1000 + 7 * i), ci.fr_to_mont(5000 + 11 * i)) for i in range(count))
        return zkey, ws, rand
    gates, adds, n_vars, n_pub, wit = OP.chain_gates(size, r=ci.r)
    if proto == "plonk":
        zkey = OP.plonk_setup_synth(gates, adds, n_vars, n_pub, tau=0xB47C + size, curve=cid)
    else:
        zkey = OF.fflonk_setup_synth(gates, adds, n_vars, n_pub, tau=0xB47C + size)
    w = bytes(O.read_wtns(OP.wtns_bytes(wit, ci.r))[1])
    rand = tuple(b"".join(ci.fr_to_mont(b) for b in blinder_ints(proto, k)) for k in range(count))
    return zkey, (w,) * count, rand


def oracle_proof(label, k):
    """proof k of the case as the CPU oracle makes it, as the module's proof object"""
    _, proto, cid, _size = next(x for x in KEYS if x[0] == label)
    zkey, ws, rand = case(label)
    ci = O.CURVES[cid]
    if proto == "groth16":
        from snarkjs_b200 import synth
        return O.groth16_prove(zkey, synth.wtns_container(ci.r, np.frombuffer(ws[k], np.uint8)), *rand[k])[0]
    from snarkjs_b200 import synth
    wtns = synth.wtns_container(ci.r, np.frombuffer(ws[k], np.uint8))
    return (OP.plonk_prove if proto == "plonk" else OF.fflonk_prove)(zkey, wtns, blinder_ints(proto, k))[0]


def batch(key, proto, ws, rand):
    """prove_batch_raw of a ProvingKey or a ReplicatedProvingKey"""
    arrs = [np.frombuffer(w, np.uint8) for w in ws]
    return key.prove_batch_raw(arrs, list(rand))


@functools.lru_cache(maxsize=None)
def single_batch(label):
    """the single-context batch of every proof of the case (tuning-independent: the batch tests prove it)"""
    import snarkjs_b200
    _, proto, cid, _size = next(k for k in KEYS if k[0] == label)
    zkey, ws, rand = case(label)
    c = snarkjs_b200.getCurveFromName(NAME[cid])
    pk = module(proto).ProvingKey(zkey, c)
    try:
        return tuple(batch(pk, proto, ws, rand))
    finally:
        pk.release()
        c.terminate()


@pytest.mark.parametrize("tune", list(TUNINGS))
@pytest.mark.parametrize("n", RANKS)
@pytest.mark.parametrize("label", [k[0] for k in KEYS])
def test_batches_equal_the_single_context_batch(ctxs, label, n, tune):
    _, proto, cid, _size = next(k for k in KEYS if k[0] == label)
    zkey, ws, rand = case(label)
    want = single_batch(label)
    cs = ctxs[cid]
    rk = module(proto).ReplicatedProvingKey(zkey, cs[:n])
    try:
        with tuning(cs[0].lib, TUNINGS[tune]):
            for count in COUNTS:
                got = batch(rk, proto, ws[:count], rand[:count])
                assert got == list(want[:count]), (count, [i for i in range(count) if got[i] != want[i]])
                if count and n == 3 and tune == "free":
                    assert module(proto).proof_to_object(cs[0], got[-1]) == oracle_proof(label, count - 1), count
                if count:
                    # rank i's own time where it had proofs; the whole call on rank 0
                    ms = [c.last_ms(0) for c in cs[:n]]
                    assert ms[0] > 0 and all((t > 0) == (i < count) for i, t in enumerate(ms[1:], 1)), ms
    finally:
        rk.release()


def test_distinct_devices():
    import torch
    import snarkjs_b200
    nd = torch.cuda.device_count()
    if nd < 2:
        pytest.skip("one device")
    cs = [snarkjs_b200.getCurveFromName("bn128", d) for d in range(nd)]
    try:
        for label in ("g16-bn-14", "plonk-bn", "fflonk-bn"):
            proto = next(k[1] for k in KEYS if k[0] == label)
            zkey, ws, rand = case(label)
            rk = module(proto).ReplicatedProvingKey(zkey, cs)
            try:
                assert batch(rk, proto, ws, rand) == list(single_batch(label)), label
            finally:
                rk.release()
    finally:
        for c in cs:
            c.terminate()


# ------------------------------------------------------------------------------------------------------------ refusals
def arr_of(curves):
    return (ctypes.c_void_p * len(curves))(*[c.handle.value for c in curves])


def raw_batch_multi(proto, curves, handles, ws, rand, n_witness=None, status=True):
    """sb_*_prove_batch_multi straight through the ABI, proofs prefilled with 0xA5 and statuses with -7:
    (rc, error text of curves[0], proof bytes per witness, statuses)"""
    lib = curves[0].lib
    count = len(ws)
    w = np.frombuffer(b"".join(ws) or b"\0", np.uint8)
    nw = len(ws[0]) // 32 if n_witness is None else n_witness
    pb = 8 * curves[0].n8q if proto == "groth16" else getattr(lib, f"sb_{proto}_proof_bytes")(curves[0].handle)
    out = np.full(max(count, 1) * pb, 0xA5, np.uint8)
    st = np.full(max(count, 1), -7, np.int32)
    hs = (ctypes.c_uint64 * len(handles))(*handles)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    if proto == "groth16":
        r = np.frombuffer(b"".join(x[0] for x in rand) or b"\0", np.uint8)
        s = np.frombuffer(b"".join(x[1] for x in rand) or b"\0", np.uint8)
        rc = lib.sb_groth16_prove_batch_multi(arr_of(curves), hs, len(curves), p(w), nw, count, p(r), p(s), p(out))
    else:
        bl = np.frombuffer(b"".join(rand) or b"\0", np.uint8)
        rc = getattr(lib, f"sb_{proto}_prove_batch_multi")(arr_of(curves), hs, len(curves), p(w), nw, count, p(bl), p(out),
                                                            p(st) if status else None)
    return rc, lib.sb_last_error(curves[0].handle).decode(), [out[i * pb:(i + 1) * pb].tobytes() for i in range(count)], list(st[:count])


def raw_single_batch(pk, proto, ws, rand):
    """sb_*_prove_batch of one context, as raw_batch_multi reports it"""
    lib, c = pk.curve.lib, pk.curve
    count = len(ws)
    w = np.frombuffer(b"".join(ws), np.uint8)
    pb = getattr(lib, f"sb_{proto}_proof_bytes")(c.handle)
    out = np.full(count * pb, 0xA5, np.uint8)
    st = np.full(count, -7, np.int32)
    bl = np.frombuffer(b"".join(rand), np.uint8)
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    rc = getattr(lib, f"sb_{proto}_prove_batch")(c.handle, pk.handle, p(w), len(ws[0]) // 32, count, p(bl), p(out), p(st))
    return rc, lib.sb_last_error(c.handle).decode(), [out[i * pb:(i + 1) * pb].tobytes() for i in range(count)], list(st)


def broken(w, r):
    """the chain witness with signal 4 moved by one: a copy constraint no longer holds"""
    ints = [int.from_bytes(w[i * 32:(i + 1) * 32], "little") for i in range(len(w) // 32)]
    ints[4] = (ints[4] + 1) % r
    return b"".join(v.to_bytes(32, "little") for v in ints)


@pytest.mark.parametrize("bad_at", [(1, 5), (4, 6)], ids=["ranks-0-1", "ranks-1-2"])
@pytest.mark.parametrize("label", ["plonk-bn", "plonk-bls", "fflonk-bn"])
def test_refused_witnesses_in_two_ranks(ctxs, label, bad_at):
    """7 proofs over 3 ranks ([0, 3), [3, 6), [6, 7)): the statuses, zero slots, code and text of the single batch"""
    _, proto, cid, _size = next(k for k in KEYS if k[0] == label)
    zkey, ws, rand = case(label)
    cs = ctxs[cid]
    bad = list(ws[:7])
    for k in bad_at:
        bad[k] = broken(bad[k], O.CURVES[cid].r)
    pk = module(proto).ProvingKey(zkey, cs[0])
    rk = module(proto).ReplicatedProvingKey(zkey, cs)
    try:
        want = raw_single_batch(pk, proto, bad, rand[:7])
        assert want[0] == -1 and [s != 0 for s in want[3]] == [k in bad_at for k in range(7)]
        got = raw_batch_multi(proto, cs, list(rk.handles), bad, rand[:7])
        assert got == want
        for k in bad_at:
            assert got[2][k] == bytes(len(got[2][k]))
        # without a status array: the same code and text
        assert raw_batch_multi(proto, cs, list(rk.handles), bad, rand[:7], status=False)[:2] == want[:2]
        assert batch(rk, proto, bad, rand[:7]) == batch(pk, proto, bad, rand[:7])
    finally:
        rk.release()
        pk.release()


def groth16_sharded_handles(curves, zkey):
    lib = curves[0].lib
    hs = (ctypes.c_uint64 * len(curves))()
    buf = np.frombuffer(zkey, np.uint8)
    assert lib.sb_groth16_load_multi(arr_of(curves), len(curves), buf.ctypes.data_as(ctypes.c_void_p), buf.size, hs) == 0
    return list(hs)


@pytest.mark.parametrize("label", ["g16-bn-10", "plonk-bn", "fflonk-bn"])
def test_refused_arguments_write_nothing(ctxs, label):
    _, proto, cid, _size = next(k for k in KEYS if k[0] == label)
    zkey, ws, rand = case(label)
    cs = ctxs[cid]
    M = module(proto)
    a = M.ReplicatedProvingKey(zkey, cs)
    b = M.ReplicatedProvingKey(zkey, cs)
    single = M.ProvingKey(zkey, cs[0])
    if proto == "groth16":
        sharded = groth16_sharded_handles(cs, zkey)
    else:
        sk = M.ShardedProvingKey(zkey, cs)
        sharded = list(sk.handles)
    other = ctxs[BLS if cid == BN else BN][0]
    ha, hb = list(a.handles), list(b.handles)
    untouched = lambda res: all(p == b"\xa5" * len(p) for p in res[2])
    try:
        ok = raw_batch_multi(proto, cs, ha, ws[:4], rand[:4])
        assert ok[0] == 0 and ok[2] == list(single_batch(label)[:4])
        nv = len(ws[0]) // 32
        res = raw_batch_multi(proto, cs, ha, ws[:4], rand[:4], n_witness=nv - 1)
        assert res[0] == -1 and res[1].startswith("Invalid witness length. Circuit: ") and untouched(res)
        res = raw_batch_multi(proto, [cs[0], cs[1], other], ha, ws[:4], rand[:4])
        assert res[0] == -1 and "not all of one curve" in res[1] and untouched(res)
        res = raw_batch_multi(proto, [cs[0], cs[1], cs[0]], ha, ws[:4], rand[:4])
        assert res[0] == -1 and "context 2 is context 0 again" in res[1] and untouched(res)
        for hs, curves in (([ha[0], hb[1], ha[2]], cs), ([ha[0], ha[2], ha[1]], [cs[0], cs[2], cs[1]]), (ha[:2], cs[:2]),
                           ([single.handle, ha[1], ha[2]], cs), (sharded, cs)):
            res = raw_batch_multi(proto, curves, hs, ws[:4], rand[:4])
            assert res[0] == -1 and "do not come from one load_replicas call" in res[1] and untouched(res), hs
        # n = 1 takes replica handles only, too
        res = raw_batch_multi(proto, cs[:1], [single.handle], ws[:4], rand[:4])
        assert res[0] == -1 and "load_replicas" in res[1] and untouched(res)
        assert raw_batch_multi(proto, cs, ha, [], [], n_witness=nv)[0] == 0            # count 0
    finally:
        if proto == "groth16":
            for c, h in zip(cs, sharded):
                c.lib.sb_groth16_release(c.handle, h)
        else:
            sk.release()
        a.release()
        b.release()
        single.release()


def view(proto, curve, handle, key):
    """a ProvingKey object over a replica handle (not owned: release() of the view is not called)"""
    M = module(proto)
    pk = M.ProvingKey.__new__(M.ProvingKey)
    pk.curve, pk.handle, pk._own_curve = curve, handle, False
    for k in key.FIELDS:
        setattr(pk, k, getattr(key, k))
    return pk


def resident(proto, pk, rnd):
    lib, c = pk.curve.lib, pk.curve
    if proto != "groth16":
        return pk.prove_raw(None, rnd)
    out = np.empty(8 * c.n8q, np.uint8)
    c.check(lib.sb_groth16_prove_resident(c.handle, pk.handle, bytes(rnd[0]), bytes(rnd[1]), out.ctypes.data_as(ctypes.c_void_p)))
    return out.tobytes()


def prove_one(proto, pk, w, rnd):
    arr = np.frombuffer(w, np.uint8)
    return pk.prove_raw(arr, *rnd) if proto == "groth16" else pk.prove_raw(arr, rnd)


@pytest.mark.parametrize("label", ["g16-bls-10", "plonk-bls", "fflonk-bn"])
def test_replica_handles_on_the_other_entries(ctxs, label):
    _, proto, cid, _size = next(k for k in KEYS if k[0] == label)
    zkey, ws, rand = case(label)
    cs = ctxs[cid]
    want = single_batch(label)
    rk = module(proto).ReplicatedProvingKey(zkey, cs)
    try:
        views = [view(proto, c, h, rk) for c, h in zip(cs, rk.handles)]
        before = []
        for i, v in enumerate(views):
            assert prove_one(proto, v, ws[i], rand[i]) == want[i]                     # sb_*_prove
            assert batch(v, proto, ws[:3], rand[:3]) == list(want[:3])                 # sb_*_prove_batch
            before.append(resident(proto, v, rand[10 + i]))                          # sb_*_prove_resident
            assert before[i] == prove_one(proto, v, ws[i], rand[10 + i])
        # a multi batch leaves every context's resident witness as it was
        assert batch(rk, proto, ws[:7], rand[:7]) == list(want[:7])
        assert [resident(proto, v, rand[10 + i]) for i, v in enumerate(views)] == before
        # sb_*_prove_multi refuses replica handles
        lib = cs[0].lib
        hs = (ctypes.c_uint64 * 3)(*rk.handles)
        w = np.frombuffer(ws[0], np.uint8)
        out = np.zeros(8 * cs[0].n8q if proto == "groth16" else getattr(lib, f"sb_{proto}_proof_bytes")(cs[0].handle), np.uint8)
        p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
        if proto == "groth16":
            rc = lib.sb_groth16_prove_multi(arr_of(cs), hs, 3, p(w), w.size // 32, rand[0][0], rand[0][1], p(out))
            assert rc == -1 and "sb_groth16_load_replicas" in lib.sb_last_error(cs[0].handle).decode()
        else:
            rc = getattr(lib, f"sb_{proto}_prove_multi")(arr_of(cs), hs, 3, p(w), w.size // 32, rand[0], p(out))
            assert rc == -1 and "do not come from one load_multi call" in lib.sb_last_error(cs[0].handle).decode()
        # releasing one replica leaves the others proving
        assert getattr(lib, f"sb_{proto}_release")(cs[1].handle, rk.handles[1]) == 0
        for i in (0, 2):
            assert prove_one(proto, views[i], ws[i], rand[i]) == want[i]
        res = raw_batch_multi(proto, cs, list(rk.handles), ws[:4], rand[:4])
        assert res[0] == -1 and "invalid handle of rank 1" in res[1]
        res = raw_batch_multi(proto, [cs[0], cs[2]], [rk.handles[0], rk.handles[2]], ws[:4], rand[:4])
        assert res[0] == -1 and "load_replicas" in res[1]                              # no longer one load of these contexts
    finally:
        rk.release()
