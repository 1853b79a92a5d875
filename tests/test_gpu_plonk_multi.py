"""GPU: one PLONK / fflonk proof on several contexts (sb_plonk_load_multi / sb_plonk_prove_multi and the fflonk pair), every
commitment summed from one MSM partial per rank over its PTau range.  All contexts sit on device 0 unless stated, and every
proof must be the single-context proof of the same key, witness and blinders, byte for byte.  Covered: 1, 2, 3 and 8 ranks
on the reference fixtures and on chain keys of 2^4 (ranges of a few points; later ranks get empty parts of the shorter
commitments), 2^10 (plain mode) and 2^14 (window tables), a 2^15 key whose eight ranges mix table and plain mode, forced
plain mode, MSM chunks smaller than a range and ranges that end a few points past a chunk, the bench keys at 2^18 and 2^20
against the committed hashes, distinct devices when there are several, and the refusals."""
import contextlib
import functools

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import oracle as O  # noqa: E402

SHARDS = (1, 2, 3, 8)
# (label, protocol, curve name, source: "fixture" or log2 of the domain)
CASES = [("plonk-bn-fixture", "plonk", "bn128", "fixture"), ("plonk-bn-4", "plonk", "bn128", 4), ("plonk-bn-10", "plonk", "bn128", 10),
         ("plonk-bn-14", "plonk", "bn128", 14), ("plonk-bls-4", "plonk", "bls12381", 4), ("plonk-bls-10", "plonk", "bls12381", 10),
         ("plonk-bls-14", "plonk", "bls12381", 14), ("fflonk-bn-fixture", "fflonk", "bn128", "fixture"), ("fflonk-bn-4", "fflonk", "bn128", 4),
         ("fflonk-bn-10", "fflonk", "bn128", 10), ("fflonk-bn-14", "fflonk", "bn128", 14)]


@pytest.fixture(scope="module")
def ctxs():
    """eight contexts per curve, all on device 0"""
    import snarkjs_b200
    cs = {name: [snarkjs_b200.getCurveFromName(name) for _ in range(8)] for name in ("bn128", "bls12381")}
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
    from snarkjs_b200 import fflonk, plonk
    return plonk if proto == "plonk" else fflonk


def blinders(proto, r, salt=0):
    n = 11 if proto == "plonk" else 9
    return b"".join((((0x51 + 7 * i + salt) << 256) % r).to_bytes(32, "little") for i in range(n))


@functools.lru_cache(maxsize=None)
def key_of(proto, cname, source):
    """(zkey bytes, witness section bytes)"""
    import os
    if source == "fixture":
        g = np.load(os.path.join(os.path.dirname(__file__), "golden", f"{proto}_case.npz"))
        return bytes(g["zkey"]), bytes(O.read_wtns(bytes(g["wtns"]))[1])
    import snarkjs_b200
    from snarkjs_b200 import synth
    c = snarkjs_b200.getCurveFromName(cname)
    try:
        zkey, wit = (synth.synth_plonk_zkey if proto == "plonk" else synth.synth_fflonk_zkey)(c, source)
        return zkey, np.asarray(wit).tobytes()
    finally:
        c.terminate()


def single_proof(curve, proto, zkey, wit, bl):
    pk = module(proto).ProvingKey(zkey, curve)
    try:
        return pk.prove_raw(np.frombuffer(wit, np.uint8), bl)
    finally:
        pk.release()


def sharded_proof(curves, proto, zkey, wit, bl):
    sk = module(proto).ShardedProvingKey(zkey, curves)
    try:
        return sk.prove_raw(np.frombuffer(wit, np.uint8), bl)
    finally:
        sk.release()


@pytest.mark.parametrize("shards", SHARDS)
@pytest.mark.parametrize("label,proto,cname,source", CASES, ids=[c[0] for c in CASES])
def test_sharded_proof_equals_single_proof(ctxs, label, proto, cname, source, shards):
    zkey, wit = key_of(proto, cname, source)
    cs = ctxs[cname]
    bl = blinders(proto, cs[0].r, shards)
    want = single_proof(cs[0], proto, zkey, wit, bl)
    sk = module(proto).ShardedProvingKey(zkey, cs[:shards])
    try:
        assert sk.prove_raw(np.frombuffer(wit, np.uint8), bl) == want
        assert sk.prove_raw(np.frombuffer(wit, np.uint8), bl) == want          # the key proves again
        bl2 = blinders(proto, cs[0].r, 100 + shards)
        assert sk.prove_raw(np.frombuffer(wit, np.uint8), bl2) == single_proof(cs[0], proto, zkey, wit, bl2) != want
        for i, c in enumerate(sk.curves):                                       # sb_*_info on every rank's handle
            import ctypes
            nv, npub, ds, na = (ctypes.c_uint32() for _ in range(4))
            assert getattr(c.lib, f"sb_{proto}_info")(c.handle, sk.handles[i], ctypes.byref(nv), ctypes.byref(npub), ctypes.byref(ds), ctypes.byref(na)) == 0
            assert (nv.value, npub.value, ds.value, na.value) == (sk.nVars, sk.nPublic, sk.domainSize, sk.nAdditions)
    finally:
        sk.release()


def test_ranges_mixing_table_and_plain_mode(ctxs):
    """2^15: eight ranges of n + 6 = 32774 points are seven of 4097 (window tables from 4096 points) and one of 4095 (plain)"""
    zkey, wit = key_of("plonk", "bn128", 15)
    cs = ctxs["bn128"]
    bl = blinders("plonk", cs[0].r)
    assert sharded_proof(cs, "plonk", zkey, wit, bl) == single_proof(cs[0], "plonk", zkey, wit, bl)


def range_past_chunk(lib, points):
    """(shards, c): the fewest shards, then the largest chunk of 2^c >= 2^10 points, for which rank 0's range of the PTau
    points (sb_shard_range) ends 1 to 16 points past a chunk boundary"""
    import ctypes
    for shards in range(2, 9):
        first, count = ctypes.c_uint64(), ctypes.c_uint64()
        lib.sb_shard_range(points, 0, shards, ctypes.byref(first), ctypes.byref(count))
        for c in range(min(count.value.bit_length() - 1, 23), 9, -1):
            if 1 <= count.value % (1 << c) <= 16:
                return shards, c
    raise AssertionError(f"no shard range of {points} points ends just past a chunk")


# "range-past-chunk": the shard count and chunk from range_past_chunk.  The 2^14 keys give PLONK two ranges of 8195 =
# 2^13 + 3 points and fflonk two of 73737 = 9 * 2^13 + 9 (PTau of n + 6 and 9n + 18 points).
@pytest.mark.parametrize("settings", [((3, 1),), ((6, 10),), "range-past-chunk"], ids=["no-tables", "chunks-2^10", "range-past-chunk"])
@pytest.mark.parametrize("proto,cname", [("plonk", "bls12381"), ("fflonk", "bn128")])
def test_forced_modes(ctxs, proto, cname, settings):
    zkey, wit = key_of(proto, cname, 14)
    cs = ctxs[cname]
    bl = blinders(proto, cs[0].r)
    shards = 3
    if settings == "range-past-chunk":
        shards, c = range_past_chunk(cs[0].lib, (1 << 14) + 6 if proto == "plonk" else (9 << 14) + 18)
        settings = ((6, c),)
    with tuning(cs[0].lib, settings):
        got = sharded_proof(cs[:shards], proto, zkey, wit, bl)
        assert got == single_proof(cs[0], proto, zkey, wit, bl)
    assert got == single_proof(cs[0], proto, zkey, wit, bl)


@pytest.mark.parametrize("proto,cname,L", [("plonk", "bls12381", 18), ("fflonk", "bn128", 18), ("plonk", "bls12381", 20), ("fflonk", "bn128", 20)])
def test_bench_keys_on_four_ranks_match_committed_hash(ctxs, proto, cname, L):
    import bench_plonk as B
    from bench import proof_hash
    from snarkjs_b200 import synth
    want = B.golden_hash(proto, cname, L)
    assert want, "no committed hash for this workload"
    cs = ctxs[cname]
    zkey, wit = (synth.synth_plonk_zkey if proto == "plonk" else synth.synth_fflonk_zkey)(cs[0], L)
    sk = module(proto).ShardedProvingKey(zkey, cs[:4])
    del zkey
    try:
        raw = sk.prove_raw(wit, B._blinders(cs[0].r, proto))
        assert proof_hash(module(proto).proof_to_object(cs[0], raw)) == want
    finally:
        sk.release()


@pytest.mark.parametrize("proto", ["plonk", "fflonk"])
def test_distinct_devices(proto):
    import torch
    import snarkjs_b200
    nd = torch.cuda.device_count()
    if nd < 2:
        pytest.skip("one device")
    cs = [snarkjs_b200.getCurveFromName("bn128", d % nd) for d in range(max(nd, 3))]
    try:
        for source in (10, 14):
            zkey, wit = key_of(proto, "bn128", source)
            bl = blinders(proto, cs[0].r)
            assert sharded_proof(cs, proto, zkey, wit, bl) == single_proof(cs[0], proto, zkey, wit, bl)
    finally:
        for c in cs:
            c.terminate()


# ------------------------------------------------------------------------------------------------------------ refusals
def error_of(fn):
    from snarkjs_b200.curve import SbError
    with pytest.raises(SbError) as e:
        fn()
    return str(e.value)


@pytest.mark.parametrize("proto", ["plonk", "fflonk"])
def test_refused_witnesses_match_the_single_path(ctxs, proto):
    zkey, wit = key_of(proto, "bn128", 10)
    cs = ctxs["bn128"]
    bl = blinders(proto, cs[0].r)
    pk = module(proto).ProvingKey(zkey, cs[0])
    sk = module(proto).ShardedProvingKey(zkey, cs[:3])
    try:
        short = np.frombuffer(wit[:-32], np.uint8)
        msg = error_of(lambda: pk.prove_raw(short, bl))
        assert msg.startswith("Invalid witness length. Circuit: ")
        assert error_of(lambda: sk.prove_raw(short, bl)) == msg
        bad = bytearray(wit)
        bad[4 * 32] ^= 1                                            # a private signal of the chain: two gates no longer hold
        msg = error_of(lambda: pk.prove_raw(np.frombuffer(bytes(bad), np.uint8), bl))
        assert error_of(lambda: sk.prove_raw(np.frombuffer(bytes(bad), np.uint8), bl)) == msg
        assert sk.prove_raw(np.frombuffer(wit, np.uint8), bl) == pk.prove_raw(np.frombuffer(wit, np.uint8), bl)   # still proves
    finally:
        sk.release()
        pk.release()


def test_plonk_key_without_public_signals(ctxs):
    from tests import r1cs_shapes as S
    zkey, wtns = S.plonk_zkey("public0"), S.case("public0").wtns()
    wit = np.frombuffer(O.read_wtns(wtns)[1], np.uint8)
    cs = ctxs["bn128"]
    bl = blinders("plonk", cs[0].r)
    pk = module("plonk").ProvingKey(zkey, cs[0])
    sk = module("plonk").ShardedProvingKey(zkey, cs[:2])
    try:
        msg = error_of(lambda: pk.prove_raw(wit, bl))
        assert msg == "Evaluations.getEvaluation() out of bounds"
        assert error_of(lambda: sk.prove_raw(wit, bl)) == msg
    finally:
        sk.release()
        pk.release()


def test_plonk_zkey_to_fflonk_multi_load(ctxs):
    import ctypes
    zkey, _ = key_of("plonk", "bn128", "fixture")
    cs = ctxs["bn128"]
    lib = cs[0].lib
    buf = np.frombuffer(zkey, np.uint8)
    h = ctypes.c_uint64()
    rc1 = lib.sb_fflonk_load(cs[0].handle, buf.ctypes.data_as(ctypes.c_void_p), buf.size, ctypes.byref(h))
    msg1 = lib.sb_last_error(cs[0].handle)
    arr = (ctypes.c_void_p * 3)(*[c.handle.value for c in cs[:3]])
    hs = (ctypes.c_uint64 * 3)(7, 7, 7)
    rc2 = lib.sb_fflonk_load_multi(arr, 3, buf.ctypes.data_as(ctypes.c_void_p), buf.size, hs)
    assert rc1 != 0 and (rc2, lib.sb_last_error(cs[0].handle)) == (rc1, msg1)
    assert list(hs) == [0, 0, 0]


def raw_prove_multi(lib, proto, curves, handles, wit, bl):
    import ctypes
    arr = (ctypes.c_void_p * len(curves))(*[c.handle.value for c in curves])
    hs = (ctypes.c_uint64 * len(handles))(*handles)
    w = np.frombuffer(wit, np.uint8)
    out = np.zeros(getattr(lib, f"sb_{proto}_proof_bytes")(curves[0].handle), np.uint8)
    rc = getattr(lib, f"sb_{proto}_prove_multi")(arr, hs, len(curves), w.ctypes.data_as(ctypes.c_void_p), w.size // 32, bl,
                                                  out.ctypes.data_as(ctypes.c_void_p))
    return rc, lib.sb_last_error(curves[0].handle).decode()


@pytest.mark.parametrize("proto", ["plonk", "fflonk"])
def test_refused_contexts_and_handles(ctxs, proto):
    import ctypes
    zkey, wit = key_of(proto, "bn128", 10)
    cs = ctxs["bn128"]
    lib = cs[0].lib
    bl = blinders(proto, cs[0].r)
    a = module(proto).ShardedProvingKey(zkey, cs[:3])
    b = module(proto).ShardedProvingKey(zkey, cs[:3])
    single = module(proto).ProvingKey(zkey, cs[0])
    try:
        ha, hb = list(a.handles), list(b.handles)
        assert raw_prove_multi(lib, proto, cs[:3], ha, wit, bl)[0] == 0
        # a context twice
        rc, msg = raw_prove_multi(lib, proto, [cs[0], cs[1], cs[0]], ha, wit, bl)
        assert rc == -1 and "context 2 is context 0 again" in msg
        # contexts of another curve
        rc, msg = raw_prove_multi(lib, proto, [cs[0], cs[1], ctxs["bls12381"][0]], ha, wit, bl)
        assert rc == -1 and "not all of one curve" in msg
        # handles swapped, or of two loads, or too few ranks
        for hs, curves in (([ha[0], ha[2], ha[1]], [cs[0], cs[2], cs[1]]), ([ha[0], hb[1], ha[2]], cs[:3]), (ha[:2], cs[:2]),
                           ([single.handle, ha[1], ha[2]], cs[:3])):
            rc, msg = raw_prove_multi(lib, proto, curves, hs, wit, bl)
            assert rc == -1 and "do not come from one load_multi call" in msg, hs
        # the single-proof entries refuse every rank's handle
        w = np.frombuffer(wit, np.uint8)
        out = np.zeros(getattr(lib, f"sb_{proto}_proof_bytes")(cs[0].handle), np.uint8)
        for i in range(3):
            rc = getattr(lib, f"sb_{proto}_prove")(cs[i].handle, ha[i], w.ctypes.data_as(ctypes.c_void_p), w.size // 32, bl, out.ctypes.data_as(ctypes.c_void_p))
            assert rc == -1 and f"sb_{proto}_prove_multi" in lib.sb_last_error(cs[i].handle).decode()
            rc = getattr(lib, f"sb_{proto}_prove_resident")(cs[i].handle, ha[i], bl, out.ctypes.data_as(ctypes.c_void_p))
            assert rc == -1 and f"sb_{proto}_prove_multi" in lib.sb_last_error(cs[i].handle).decode()
            st = np.zeros(1, np.int32)
            rc = getattr(lib, f"sb_{proto}_prove_batch")(cs[i].handle, ha[i], w.ctypes.data_as(ctypes.c_void_p), w.size // 32, 1, bl,
                                                          out.ctypes.data_as(ctypes.c_void_p), st.ctypes.data_as(ctypes.c_void_p))
            assert rc == -1 and f"sb_{proto}_prove_multi" in lib.sb_last_error(cs[i].handle).decode()
        # a released shard
        assert getattr(lib, f"sb_{proto}_release")(cs[1].handle, hb[1]) == 0
        rc, msg = raw_prove_multi(lib, proto, cs[:3], hb, wit, bl)
        assert rc == -1 and "invalid handle of rank 1" in msg
        assert raw_prove_multi(lib, proto, cs[:3], ha, wit, bl)[0] == 0          # the other key is untouched
    finally:
        a.release()
        b.release()
        single.release()
