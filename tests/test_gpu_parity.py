"""GPU parity: the CUDA path (through the C ABI / snarkjs_b200 host mirror) against the CPU oracle, the
reference-produced fixture goldens, and size-independent properties at BASELINE.json sizes.
All integer work: comparisons are bit-exact."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import oracle as O  # noqa: E402  (checker only)

BN, BLS = O.BN254, O.BLS12_381


@pytest.fixture(scope="module")
def bn():
    import snarkjs_b200
    c = snarkjs_b200.getCurveFromName("bn128")
    yield c
    c.terminate()


@pytest.fixture(scope="module")
def bls():
    import snarkjs_b200
    c = snarkjs_b200.getCurveFromName("bls12381")
    yield c
    c.terminate()


def rand_fr(seed, n, curve=BN, mont=True):
    """n uniform Fr elements (canonical; Montgomery bytes are just another uniform residue)."""
    return O.random_scalars(seed, n, O.CURVES[curve].r)


# ----------------------------------------------------------------------------------------------- Fr constants
def test_roots_match_oracle(bn, bls):
    for c, cid in ((bn, BN), (bls, BLS)):
        assert c.Fr.s == O.fr_s(cid)
        for i in range(c.Fr.s + 1):
            assert c.Fr.w[i] == O.fr_root(cid, i)
        assert c.Fr.shift == O.fr_root(cid, -1)
        assert c.Fr.nqr == O.fr_root(cid, -2)


# ----------------------------------------------------------------------------------------------- NTT
def test_ntt_fixture_goldens(bn, golden):
    g = golden("ntt_goldens.npz")
    labels = sorted({k[:-5] for k in g if k.endswith("_coef")})
    for lab in labels:
        coef, evals = g[lab + "_coef"], g[lab + "_evals"]
        n = coef.size // 32
        padded = np.concatenate([coef, np.zeros(3 * n * 32, dtype=np.uint8)])
        assert np.array_equal(bn.Fr.fft(padded), evals), lab
        back = bn.Fr.ifft(evals)
        assert np.array_equal(back[:n * 32], coef) and not back[n * 32:].any(), lab


@pytest.mark.parametrize("L", list(range(0, 15)) + [16, 17, 19, 20, 21])
def test_ntt_vs_oracle_bn(bn, L):
    x = rand_fr(100 + L, 1 << L)
    assert np.array_equal(bn.Fr.fft(x), O.fr_fft(BN, x)), L
    assert np.array_equal(bn.Fr.ifft(x), O.fr_fft(BN, x, inverse=True)), L


@pytest.mark.parametrize("L", [1, 5, 10, 11, 13, 18])
def test_ntt_vs_oracle_bls(bls, L):
    x = rand_fr(200 + L, 1 << L, BLS)
    assert np.array_equal(bls.Fr.fft(x), O.fr_fft(BLS, x)), L
    assert np.array_equal(bls.Fr.ifft(x), O.fr_fft(BLS, x, inverse=True)), L


def test_ntt_roundtrip_2_24(bn):
    """BASELINE config #3: 2^24-element round trip (size-independent property) + linearity spot check."""
    n = 1 << 24
    x = rand_fr(4, n)
    y = bn.Fr.fft(x)
    assert np.array_equal(bn.Fr.ifft(y), x)
    # full-size comparison with the oracle (a few seconds with OpenMP)
    small = O.fr_fft(BN, x)  # oracle at full size takes a few seconds with OpenMP
    assert np.array_equal(small, y)


def test_ntt_errors(bn):
    from snarkjs_b200 import SbError
    with pytest.raises(SbError, match="fft must be multiple of 2"):
        bn.Fr.fft(bytes(32 * 3))
    with pytest.raises(SbError, match="fft must be multiple of 2"):
        bn.Fr.fft(b"")


# ----------------------------------------------------------------------------------------------- element-wise Fr
@pytest.mark.parametrize("n", [1, 7, 1000, 4096, 100003])
def test_apply_key_convert_join(bn, n):
    ci = O.CURVES[BN]
    x, y, z = rand_fr(1, n), rand_fr(2, n), rand_fr(3, n)
    first, inc = ci.fr_to_mont(3), O.fr_root(BN, 11)
    assert np.array_equal(bn.Fr.batchApplyKey(x, first, inc), O.fr_batch_apply_key(BN, x, first, inc))
    assert np.array_equal(bn.Fr.batchToMontgomery(x), O.batch_convert(O.F_BN_FR, True, x))
    assert np.array_equal(bn.Fr.batchFromMontgomery(x), O.batch_convert(O.F_BN_FR, False, x))
    import ctypes
    from snarkjs_b200.curve import _ptr
    out = np.empty_like(x)
    bn.check(bn.lib.sb_qap_join_abc(bn.handle, _ptr(x), _ptr(y), _ptr(z), n, _ptr(out)))
    assert np.array_equal(out, O.qap_join_abc(BN, x, y, z))


# ----------------------------------------------------------------------------------------------- MSM
def _msm_check(curve_obj, cid, grp, bases, scalars):
    G = curve_obj.G1 if grp == 1 else curve_obj.G2
    got = G.toAffine(G.multiExpAffine(bases, scalars)).tobytes()
    want = O.g_to_affine(cid, grp, O.multiexp_affine(cid, grp, bases, scalars))
    assert got == want


def test_msm_g1_fixture_goldens(bn, golden):
    g = golden("msm_g1_goldens.npz")
    for nm in sorted(k[:-7] for k in g if k.endswith("_commit")):
        tag = nm.split("_")[0]
        scal = bn.Fr.batchFromMontgomery(g[nm + "_coef_mont"])      # polynomial.js:973
        n = scal.size // 32
        res = bn.G1.multiExpAffine(g[tag + "_ptau"][:64 * n], scal)
        assert bn.G1.toAffine(res).tobytes() == g[nm + "_commit"].tobytes(), nm


def _lagrange_scalars(k, j):
    ci = O.CURVES[BN]
    n = 1 << k
    winv = pow(ci.fr_from_mont(O.fr_root(BN, k)), -1, ci.r)
    ninv = pow(n, -1, ci.r)
    return b"".join((pow(winv, i * j, ci.r) * ninv % ci.r).to_bytes(32, "little") for i in range(n))


def test_msm_ptau_goldens_g1_g2(bn, golden):
    g = golden("ptau_goldens.npz")
    for grp, key, sz in ((1, "g1", 64), (2, "g2", 128)):
        base = g["tauG1"] if grp == 1 else g["tauG2"]
        G = bn.G1 if grp == 1 else bn.G2
        for idx, (k, j) in enumerate(g[key + "_picks"]):
            n = 1 << int(k)
            res = G.multiExpAffine(base[:sz * n], _lagrange_scalars(int(k), int(j)))
            assert G.toAffine(res).tobytes() == g[key + "_expected"][idx * sz:(idx + 1) * sz].tobytes(), (key, k, j)


@pytest.mark.parametrize("n", [1, 2, 3, 31, 32, 33, 100, 1000, 4097, 1 << 14])
@pytest.mark.parametrize("grp", [1, 2])
def test_msm_vs_oracle_bn(bn, n, grp):
    bases = O.gen_points(BN, grp, 10 + n, n)
    _msm_check(bn, BN, grp, bases, rand_fr(20 + n, n))


@pytest.mark.parametrize("n,grp", [(1, 1), (50, 1), (3000, 1), (1, 2), (50, 2), (3000, 2)])
def test_msm_vs_oracle_bls(bls, n, grp):
    bases = O.gen_points(BLS, grp, 10 + n, n)
    _msm_check(bls, BLS, grp, bases, rand_fr(20 + n, n, BLS))


def test_msm_edge_cases(bn):
    n = 600
    bases = O.gen_points(BN, 1, 77, n).reshape(n, 64).copy()
    sc = rand_fr(78, n).reshape(n, 32).copy()
    # points at infinity, repeated points (forces P+P doubling inside a bucket), P and -P with equal scalars (cancellation)
    bases[5] = 0
    bases[17] = 0
    bases[100:140] = bases[100]
    sc[100:140] = sc[100]
    ci = O.CURVES[BN]
    negy = (ci.q - ci.fq_from_mont(bases[200, 32:].tobytes())) % ci.q
    bases[201, :32] = bases[200, :32]
    bases[201, 32:] = np.frombuffer(ci.fq_to_mont(negy), np.uint8)
    sc[201] = sc[200]
    # scalar values: 0, 1, r-1, 2^256-1 (>= r, the reference accepts any value < 2^(8*sScalar))
    sc[0] = 0
    sc[1] = 0; sc[1, 0] = 1
    sc[2] = np.frombuffer((ci.r - 1).to_bytes(32, "little"), np.uint8)
    sc[3] = 255
    _msm_check(bn, BN, 1, bases.reshape(-1), sc.reshape(-1))
    # all scalars zero -> zero point; all scalars one -> sum of points
    z = bn.G1.multiExpAffine(bases.reshape(-1), np.zeros(n * 32, np.uint8))
    assert bn.G1.toAffine(z).tobytes() == bytes(64)
    ones = np.zeros((n, 32), np.uint8); ones[:, 0] = 1
    _msm_check(bn, BN, 1, bases.reshape(-1), ones.reshape(-1))
    # empty input -> G.zero (14561)
    assert bn.G1.multiExpAffine(b"", b"").tobytes() == O.group_zero(BN, 1)
    assert bn.G2.multiExpAffine(b"", b"").tobytes() == O.group_zero(BN, 2)


@pytest.mark.parametrize("sbytes", [1, 4, 13, 31, 32, 40])
def test_msm_scalar_sizes(bn, sbytes):
    n = 257
    bases = O.gen_points(BN, 1, 5, n)
    rng = np.random.default_rng(sbytes)
    sc = rng.integers(0, 256, size=n * sbytes, dtype=np.uint8)
    _msm_check(bn, BN, 1, bases, sc)


def test_msm_scalar_size_mismatch(bn):
    from snarkjs_b200 import SbError
    with pytest.raises(SbError, match="Scalar size does not match"):
        bn.G1.multiExpAffine(bytes(64 * 3), bytes(32 * 3 + 1))


def test_msm_witness_like_skew(bn):
    """SURVEY §8d: 50% zeros, 25% ones, rest uniform — the bucket-skew case (one giant bucket)."""
    n = 1 << 15
    bases = O.gen_points(BN, 1, 9, n)
    sc = rand_fr(91, n).reshape(n, 32).copy()
    rng = np.random.default_rng(5)
    kind = rng.integers(0, 4, n)
    sc[kind < 2] = 0
    sc[kind == 2] = 0
    sc[kind == 2, 0] = 1
    _msm_check(bn, BN, 1, bases, sc.reshape(-1))


def test_msm_2_20_bn254_g1(bn):
    """BASELINE config #2: 2^20 points, 254-bit scalars — bit-exact affine result vs the oracle's Pippenger."""
    n = 1 << 20
    bases = O.gen_points(BN, 1, 2, n)
    sc = rand_fr(3, n)
    _msm_check(bn, BN, 1, bases, sc)
    # registered-bases route and linearity: MSM(b, s) + MSM(b, s') == MSM(b, s + s' mod r) checked through the oracle adds
    h = bn.G1.registerBases(bases)
    r1 = bn.G1.multiExpRegistered(h, sc)
    assert bn.G1.toAffine(r1).tobytes() == O.g_to_affine(BN, 1, O.multiexp_affine(BN, 1, bases, sc))
    half = n // 2
    a = bn.G1.multiExpRegistered(h, sc[:half * 32], first=0, n=half)
    b = bn.G1.multiExpRegistered(h, sc[half * 32:], first=half, n=half)
    assert O.g_to_affine(BN, 1, O.g_add(BN, 1, a.tobytes(), b.tobytes())) == bn.G1.toAffine(r1).tobytes()


# ----------------------------------------------------------------------------------------------- Groth16
def test_groth16_fused_matches_oracle_and_verifies(bn, golden):
    """BASELINE config #1: proof bytes identical to the CPU oracle for the same (r, s); proof verifies;
    aliased public input rejected (test/fullprocess.js:120-133)."""
    from snarkjs_b200 import groth16
    g = golden("groth16_case.npz")
    zkey, wt = g["zkey"].tobytes(), g["wtns"].tobytes()
    ci = O.CURVES[BN]
    r, s = ci.fr_to_mont(123456789), ci.fr_to_mont(987654321)
    pk = groth16.ProvingKey(zkey, curve=bn)
    proof, pub = groth16.prove(pk, wt, r, s)
    oproof, opub = O.groth16_prove(zkey, wt, r, s)
    assert proof == oproof
    assert pub == [str(x) for x in opub]
    vk = O.zkey_vk(zkey)
    assert O.groth16_verify(vk, [int(x) for x in pub], proof)
    assert not O.groth16_verify(vk, [int(pub[0]) + ci.r] + [int(x) for x in pub[1:]], proof)
    # random (r, s): different proof, still valid
    proof2, _ = groth16.prove(pk, wt)
    assert proof2 != proof and O.groth16_verify(vk, [int(x) for x in pub], proof2)
    # sharded route (multi-GPU exchange unit) on one device: 3 shards summed == unsharded
    _, W = groth16.read_wtns_header(wt)
    parts = np.concatenate([pk.prove_shard(np.frombuffer(W, np.uint8), i, 3) for i in range(3)])
    aff = pk.finish(parts, 3, r, s)
    assert groth16.proof_to_object(bn, aff) == proof
    pk.release()


def test_groth16_errors(bn, golden):
    from snarkjs_b200 import groth16, SbError
    g = golden("groth16_case.npz")
    zkey, wt = g["zkey"].tobytes(), g["wtns"].tobytes()
    pk = groth16.ProvingKey(zkey, curve=bn)
    with pytest.raises(SbError, match="Invalid witness length"):
        pk.prove_raw(np.zeros(32 * 5, np.uint8), bytes(32), bytes(32))
    with pytest.raises(SbError, match="Invalid File format"):
        groth16.ProvingKey(b"nope" + zkey[4:], curve=bn)
    pk.release()


# ----------------------------------------------------------------------------------------------- synthetic workloads


@pytest.mark.parametrize("cname,cid", [("bn128", BN), ("bls12381", BLS)])
def test_gen_points_equal_the_oracle_generator(bn, bls, cname, cid):
    """sb_gen_points and the oracle's incremental generator define the same points (bench.py builds the B200 arm's key
    with the first and the CPU reference arm's key with the second): compared across a 4096-point chunk boundary, and
    spot-checked as (k0 + j*kd)*G against the oracle's scalar multiplication."""
    from snarkjs_b200 import synth
    c = bn if cid == BN else bls
    ci = O.CURVES[cid]
    M = (1 << 64) - 1
    for grp, n in ((1, 9000), (2, 4200)):
        pts = synth.gen_points(c, grp, 42, n)
        assert np.array_equal(pts, O.gen_points(cid, grp, 42, n)), (cname, grp)
        sz = ci.n8q * 2 * grp
        gen = ci.g1_affine_bytes(ci.g1) if grp == 1 else ci.g2_affine_bytes(ci.g2)
        gj = O.g_from_affine(cid, grp, gen)
        kd = (42 * 2654435761 + 12345) & M
        for i in (0, 3, 4095, 4096, 4199):
            ch, j = divmod(i, 4096)
            k = (((42 ^ 0x9E3779B97F4A7C15) + ch * 0xD1B54A32D192ED03) & M) + j * kd
            want = O.g_to_affine(cid, grp, O.g_times(cid, grp, gj, k.to_bytes(16, "little")))
            assert pts.tobytes()[i * sz:(i + 1) * sz] == want, (cname, grp, i)


@pytest.mark.parametrize("L", [12, 16, 18])
def test_bench_key_proof_hash_matches_committed_oracle_hash(bn, L):
    """The key bench.py proves (synth seed 1, r = 5, s = 7): the GPU proof object hashes to the CPU oracle's committed
    hash (tests/golden/bench_proof_hashes.json, written by make_bench_hashes.py without a GPU).  bench.py asserts the
    2^20 / 2^22 entries of the same table on every run."""
    import json, os, hashlib
    from snarkjs_b200 import groth16, synth
    tab = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "bench_proof_hashes.json")))["groth16_bn128_chain_r5_s7"]
    zkey = synth.synth_groth16_zkey(bn, L, seed=1)
    ci = O.CURVES[BN]
    pk = groth16.ProvingKey(zkey, curve=bn)
    aff = pk.prove_raw(synth.chain_witness(bn.r, L), ci.fr_to_mont(5), ci.fr_to_mont(7))
    obj = groth16.proof_to_object(bn, aff)
    pk.release()
    assert hashlib.sha256(json.dumps(obj, sort_keys=True, separators=(",", ":")).encode()).hexdigest() == tab[str(L)]


def test_overlapping_calls_on_one_context_are_serialised(bn):
    """The reference awaits several bulk calls at once (build/snarkjs.js:14653, 14929-14932) and an N-API shim runs them
    on libuv threads: four threads hammer ONE context with NTTs, MSMs and joinABC calls that share its staging and io
    buffers; every result must equal the single-threaded one."""
    import threading
    x = [rand_fr(900 + i, 1 << 14) for i in range(4)]
    bases = O.gen_points(BN, 1, 77, 1 << 12)
    want_ntt = [bn.Fr.fft(v).copy() for v in x]
    want_msm = [bn.G1.toAffine(bn.G1.multiExpAffine(bases, v[:32 << 12])).tobytes() for v in x]
    from snarkjs_b200.curve import _ptr

    def join():
        out = np.empty_like(x[0])
        bn.check(bn.lib.sb_qap_join_abc(bn.handle, _ptr(x[0]), _ptr(x[1]), _ptr(x[2]), x[0].size // 32, _ptr(out)))
        return out
    want_join = join()
    errs = []

    def work(i):
        try:
            for _ in range(6):
                assert np.array_equal(bn.Fr.fft(x[i]), want_ntt[i])
                assert bn.G1.toAffine(bn.G1.multiExpAffine(bases, x[i][:32 << 12])).tobytes() == want_msm[i]
                assert np.array_equal(join(), want_join)
        except Exception as e:  # noqa: BLE001
            errs.append((i, repr(e)))

    th = [threading.Thread(target=work, args=(i,)) for i in range(4)]
    [t.start() for t in th]
    [t.join() for t in th]
    assert not errs, errs


def test_prove_resident_needs_a_witness_and_truncated_containers_fail(bn, golden):
    import ctypes, struct
    from snarkjs_b200 import groth16, SbError
    from snarkjs_b200.curve import _ptr
    g = golden("groth16_case.npz")
    zkey = g["zkey"].tobytes()
    pk = groth16.ProvingKey(zkey, curve=bn)
    out = np.empty(256, np.uint8)
    ci = O.CURVES[BN]
    rc = bn.lib.sb_groth16_prove_resident(bn.handle, pk.handle, ci.fr_to_mont(1), ci.fr_to_mont(2), _ptr(out))
    assert rc != 0 and b"no witness resident" in bn.lib.sb_last_error(bn.handle)
    pk.release()
    # a section length near 2^64 must not wrap the bounds check (ADVICE r1): zkey and wtns containers
    sid, ln = struct.unpack_from("<IQ", zkey, 12)
    bad = bytearray(zkey)
    struct.pack_into("<Q", bad, 16, (1 << 64) - 12 - 12)
    h = ctypes.c_uint64()
    buf = np.frombuffer(bytes(bad), np.uint8)
    assert bn.lib.sb_groth16_load(bn.handle, _ptr(buf), buf.size, ctypes.byref(h)) != 0
    assert b"Invalid file size" in bn.lib.sb_last_error(bn.handle)
    w = bytearray(g["wtns"].tobytes())
    struct.pack_into("<Q", w, 16, (1 << 64) - 24)
    pk = groth16.ProvingKey(zkey, curve=bn)
    wb = np.frombuffer(bytes(w), np.uint8)
    assert bn.lib.sb_groth16_prove_wtns(bn.handle, pk.handle, _ptr(wb), wb.size, ci.fr_to_mont(1), ci.fr_to_mont(2), _ptr(out)) != 0
    pk.release()


def test_groth16_synthetic_2_16_matches_oracle(bn):
    """Synthetic chain circuit at 2^16 (unstructured key): fused GPU proof == oracle proof, byte for byte."""
    from snarkjs_b200 import groth16, synth
    L = 16
    zkey = synth.synth_groth16_zkey(bn, L, seed=3)
    w = synth.chain_witness(bn.r, L)
    wt = synth.wtns_container(bn.r, w)
    ci = O.CURVES[BN]
    r, s = ci.fr_to_mont(99), ci.fr_to_mont(77)
    pk = groth16.ProvingKey(zkey, curve=bn)
    proof, pub = groth16.prove(pk, wt, r, s)
    oproof, opub = O.groth16_prove(zkey, wt, r, s)
    assert proof == oproof and pub == [str(x) for x in opub]
    pk.release()


def test_groth16_bls12_381_synthetic_matches_oracle(bls):
    """BASELINE config #5's G2-MSM + coset-NTT content lives in Groth16 on BLS12-381 (SURVEY §3.4): 12-limb Fq, Fq2
    MSM, Fr with 2-adicity 32.  Synthetic chain circuit at 2^13, unstructured key; proof bytes == oracle's."""
    from snarkjs_b200 import groth16, synth
    L = 13
    zkey = synth.synth_groth16_zkey(bls, L, seed=5)
    w = synth.chain_witness(bls.r, L)
    wt = synth.wtns_container(bls.r, w)
    ci = O.CURVES[BLS]
    r, s = ci.fr_to_mont(31337), ci.fr_to_mont(271828)
    pk = groth16.ProvingKey(zkey, curve=bls)
    proof, pub = groth16.prove(pk, wt, r, s)
    oproof, opub = O.groth16_prove(zkey, wt, r, s)
    assert proof == oproof and pub == [str(x) for x in opub]
    pk.release()


def test_bigbuffer_like_inputs(bn):
    """The reference accepts BigBuffer (paged) inputs at the boundary (build/snarkjs.js:12692-12778)."""
    class BigBuffer:
        def __init__(self, data, page):
            self.buffers = [data[i:i + page] for i in range(0, len(data), page)]
            self.byteLength = len(data)
    n = 3000
    bases = O.gen_points(BN, 1, 8, n)
    sc = rand_fr(9, n)
    res = bn.G1.multiExpAffine(BigBuffer(bases, 64 * 1000), BigBuffer(sc, 32 * 777))
    assert bn.G1.toAffine(res).tobytes() == O.g_to_affine(BN, 1, O.multiexp_affine(BN, 1, bases, sc))
    x = rand_fr(10, 4096)
    assert np.array_equal(bn.Fr.fft(BigBuffer(x, 32 * 1024)), O.fr_fft(BN, x))


def test_msm_plain_vs_table_mode(bn):
    """Registered bases use precomputed window tables; sb_set_tuning(3,1) forces the plain windowed path — same bytes.
    sb_set_tuning(1,1) replaces the axis-sum bucket reduction by k_reduce / k_window_sum (the path for geometries with
    more than 2^20 buckets per window) — same bytes again, in both modes."""
    n = 1 << 14
    bases = O.gen_points(BN, 2, 21, n)
    sc = rand_fr(22, n)
    h1 = bn.G2.registerBases(bases)
    a = bn.G2.multiExpRegistered(h1, sc)
    bn.lib.sb_set_tuning(3, 1)
    try:
        h2 = bn.G2.registerBases(bases)
        b = bn.G2.multiExpRegistered(h2, sc)
        assert bn.lib.sb_set_tuning(1, 2) != 0 and bn.lib.sb_set_tuning(4, 2) != 0   # unknown values and keys are refused
        assert all(bn.lib.sb_set_tuning(13, v) != 0 for v in (1, 2, 23))           # window bits outside 3..22
        assert bn.lib.sb_set_tuning(1, 1) == 0
        try:
            assert bn.G2.multiExpRegistered(h2, sc).tobytes() == a.tobytes()
            assert bn.G2.multiExpRegistered(h1, sc).tobytes() == a.tobytes()
        finally:
            bn.lib.sb_set_tuning(1, 0)
    finally:
        bn.lib.sb_set_tuning(3, 0)
    assert a.tobytes() == b.tobytes()
    assert bn.G2.toAffine(a).tobytes() == O.g_to_affine(BN, 2, O.multiexp_affine(BN, 2, bases, sc))
    # sub-range of a registered table
    c = bn.G2.multiExpRegistered(h1, sc[100 * 32:5100 * 32], first=100, n=5000)
    assert bn.G2.toAffine(c).tobytes() == O.g_to_affine(BN, 2, O.multiexp_affine(BN, 2, bases[100 * 128:5100 * 128], sc[100 * 32:5100 * 32]))


def test_groth16_sharded_keys_match_unsharded(bn):
    """Multi-GPU layout on one device: three proving keys each holding one point-range shard (with their own window
    tables); the gathered partials finish to the same proof as the unsharded key; a sharded key refuses other shards."""
    from snarkjs_b200 import groth16, synth, SbError
    L = 15
    zkey = synth.synth_groth16_zkey(bn, L, seed=9)
    w = synth.chain_witness(bn.r, L)
    ci = O.CURVES[BN]
    r, s = ci.fr_to_mont(4242), ci.fr_to_mont(2424)
    full = groth16.ProvingKey(zkey, curve=bn)
    want = full.prove_raw(w, r, s)
    keys = [groth16.ProvingKey(zkey, curve=bn, shard=i, n_shards=3) for i in range(3)]
    parts = np.concatenate([keys[i].prove_shard(w, i, 3) for i in range(3)])
    assert keys[0].finish(parts, 3, r, s) == want
    with pytest.raises(SbError, match="different shard"):
        keys[0].prove_shard(w, 1, 3)
    with pytest.raises(SbError, match="loaded sharded"):
        keys[0].prove_raw(w, r, s)
    for k in keys + [full]:
        k.release()


def test_plonk_polynomial_wrappers_on_fixture_goldens(bn, golden):
    """SURVEY §8a a10: the PLONK/fflonk call sites (Polynomial.fromEvaluations / to4T / multiExponentiation,
    Evaluations.fromPolynomial) reproduce the reference-written bytes of the committed PLONK zkeys."""
    from snarkjs_b200.polynomial import Polynomial, Evaluations
    gn, gm = golden("ntt_goldens.npz"), golden("msm_g1_goldens.npz")
    for tag, lab, name in (("plonk2048", "QM", "Qm"), ("plonk8", "QM", "Qm"), ("plonk8", "S1", "S1")):
        coef, evals = gn[f"{tag}_{lab}_coef"], gn[f"{tag}_{lab}_evals"]
        p = Polynomial(coef, bn)
        assert np.array_equal(Evaluations.fromPolynomial(p, 4, bn).eval, evals)                      # evaluations.js:29-36
        assert np.array_equal(Polynomial.fromEvaluations(evals, bn).coef[:coef.size], coef)          # polynomial.js:31-35
        assert p.multiExponentiation(gm[f"{tag}_ptau"], name).tobytes() == gm[f"{tag}_{name}_commit"].tobytes()   # :970-977
        n = coef.size // 32
        a, A4 = Polynomial.to4T(O.fr_fft(BN, coef), n, bn.Fr)                                         # :111-119
        assert np.array_equal(a, coef) and np.array_equal(A4, evals)


def test_groth16_streamed_zkey_file(bn, golden, tmp_path):
    """sb_groth16_load_file: the key mapped from disk and streamed through the staging buffers; same proof as the
    in-memory load; malformed files are rejected with the reference's messages."""
    from snarkjs_b200 import groth16, SbError
    g = golden("groth16_case.npz")
    zkey, wt = g["zkey"].tobytes(), g["wtns"].tobytes()
    p = tmp_path / "circuit.zkey"
    p.write_bytes(zkey)
    ci = O.CURVES[BN]
    r, s = ci.fr_to_mont(77), ci.fr_to_mont(88)
    pk_mem = groth16.ProvingKey(zkey, curve=bn)
    pk_file = groth16.ProvingKey.from_file(str(p), bn)
    assert (pk_file.nVars, pk_file.nPublic, pk_file.domainSize) == (pk_mem.nVars, pk_mem.nPublic, pk_mem.domainSize)
    assert groth16.prove(pk_file, wt, r, s) == groth16.prove(pk_mem, wt, r, s)
    (tmp_path / "short.zkey").write_bytes(zkey[:len(zkey) - 100])
    with pytest.raises(SbError, match="Invalid file size"):
        groth16.ProvingKey.from_file(str(tmp_path / "short.zkey"), bn)
    with pytest.raises(SbError, match="cannot open"):
        groth16.ProvingKey.from_file(str(tmp_path / "missing.zkey"), bn)
    pk_mem.release(); pk_file.release()


def test_chunked_paths(bn, golden):
    """Inputs larger than one MSM chunk (2^23 points in production) take the chunk loop of sb_msm_* and the serial
    fallback of the Groth16 pipeline; sb_set_tuning(6, 11) shrinks the chunk to 2^11 so the tests reach them."""
    from snarkjs_b200 import groth16
    n = 9000
    bases = O.gen_points(BN, 1, 51, n)
    sc = rand_fr(52, n)
    want = O.g_to_affine(BN, 1, O.multiexp_affine(BN, 1, bases, sc))
    g = golden("groth16_case.npz")
    zkey, wt = g["zkey"].tobytes(), g["wtns"].tobytes()
    ci = O.CURVES[BN]
    r, s = ci.fr_to_mont(5150), ci.fr_to_mont(1984)
    oproof, _ = O.groth16_prove(zkey, wt, r, s)
    bn.lib.sb_set_tuning(6, 11)
    try:
        assert bn.G1.toAffine(bn.G1.multiExpAffine(bases, sc)).tobytes() == want
        h = bn.G1.registerBases(bases)
        assert bn.G1.toAffine(bn.G1.multiExpRegistered(h, sc)).tobytes() == want
        pk = groth16.ProvingKey(zkey, curve=bn)          # domain 1024 < chunk, nVars 1003 < chunk: shrink further
        bn.lib.sb_set_tuning(6, 8)
        proof, _ = groth16.prove(pk, wt, r, s)
        assert proof == oproof
        pk.release()
    finally:
        bn.lib.sb_set_tuning(6, 0)


def test_staged_host_copies(bn, golden):
    """sb_set_tuning(8, 1): pageable caller buffers >= 1 MiB go through the pinned double-buffered staging path (both
    directions, odd sizes, several chunks); results are unchanged."""
    from snarkjs_b200 import groth16, synth
    x = rand_fr(71, (1 << 19) + 0)                       # 16 MiB: two 8 MiB chunks exactly
    y = rand_fr(72, 300001)                              # 9.2 MiB: one full chunk + remainder
    want_fft = O.fr_fft(BN, x)
    want_conv = O.batch_convert(O.F_BN_FR, True, y)
    n = 40000
    bases = O.gen_points(BN, 1, 73, n)                   # 2.4 MiB of bases, 1.2 MiB of scalars
    sc = rand_fr(74, n)
    want_msm = O.g_to_affine(BN, 1, O.multiexp_affine(BN, 1, bases, sc))
    L = 16
    zkey = synth.synth_groth16_zkey(bn, L, seed=11)
    w = synth.chain_witness(bn.r, L)                     # 2 MiB pageable witness
    ci = O.CURVES[BN]
    r, s = ci.fr_to_mont(3), ci.fr_to_mont(4)
    pk = groth16.ProvingKey(zkey, curve=bn)
    want_proof = pk.prove_raw(w, r, s)
    for mode in (1, 0):                                  # staged (default) and the driver's pageable path
      bn.lib.sb_set_tuning(8, mode)
      try:
        assert np.array_equal(bn.Fr.fft(x), want_fft)
        assert np.array_equal(bn.Fr.batchToMontgomery(y), want_conv)
        assert bn.G1.toAffine(bn.G1.multiExpAffine(bases, sc)).tobytes() == want_msm
        assert pk.prove_raw(w, r, s) == want_proof
        pts = synth.gen_points(bn, 2, 5, 20000)          # 2.5 MiB device -> host
        if mode == 1: ref_pts = pts.tobytes()
        else: assert pts.tobytes() == ref_pts
      finally:
        bn.lib.sb_set_tuning(8, 1)
    pk.release()


def test_table_mode_full_width_scalars_and_bls(bn, bls):
    """Registered bases (precomputed window tables): arbitrary 256-bit scalars (the reference accepts any value
    < 2^(8*sScalar)), short scalars, BLS12-381 G1/G2, and the partial/sum-partials exchange API."""
    import ctypes
    from snarkjs_b200.curve import _ptr
    n = 1 << 13
    rng = np.random.default_rng(99)
    for curve, cid, grp in ((bn, BN, 1), (bn, BN, 2), (bls, BLS, 1), (bls, BLS, 2)):
        G = curve.G1 if grp == 1 else curve.G2
        bases = O.gen_points(cid, grp, 60 + grp, n)
        h = G.registerBases(bases)
        full = rng.integers(0, 256, size=n * 32, dtype=np.uint8)            # uniform 256-bit values, most >= r
        full[:32] = 255
        got = G.multiExpRegistered(h, full)
        assert G.toAffine(got).tobytes() == O.g_to_affine(cid, grp, O.multiexp_affine(cid, grp, bases, full)), (cid, grp)
        short = rng.integers(0, 256, size=n * 5, dtype=np.uint8)             # 5-byte scalars through the table path
        out = np.empty(G.sJacobian, np.uint8)
        curve.check(curve.lib.sb_msm_registered(curve.handle, h, 0, _ptr(short), 5, n, _ptr(out)))
        assert G.toAffine(out).tobytes() == O.g_to_affine(cid, grp, O.multiexp_affine(cid, grp, bases, short)), (cid, grp, "short")
        # exchange unit: two half-range partials summed on the host == whole
        pb = curve.lib.sb_msm_partial_bytes(curve.handle, grp)
        parts = np.empty(2 * pb, np.uint8)
        half = n // 2
        sc = rand_fr(61, n, cid)
        for i in range(2):
            curve.check(curve.lib.sb_msm_registered_partial(curve.handle, h, i * half, _ptr(sc[i * half * 32:(i + 1) * half * 32]), 32, half,
                                                            ctypes.c_void_p(parts.ctypes.data + i * pb)))
        summed = np.empty(G.sJacobian, np.uint8)
        curve.check(curve.lib.sb_msm_sum_partials(curve.handle, grp, _ptr(parts), 2, _ptr(summed)))
        assert G.toAffine(summed).tobytes() == O.g_to_affine(cid, grp, O.multiexp_affine(cid, grp, bases, sc)), (cid, grp, "partials")
        curve.check(curve.lib.sb_bases_release(curve.handle, h))
