"""GPU: the Fr NTT as the provers launch it, compared byte for byte with the CPU oracle, and the device-pointer entry points.

sb_ntt_eval runs the library's own launch functions on host data: fr_ntt_batch (layout 0: up to four transforms, each at its
own device offset, as Groth16 runs A, B and C) and fr_ntt_strided (layout 1: any number back to back, as a batch of proofs
and as PLONK and fflonk run theirs), with the optional pre-multiplier first * inc^i on the first pass and the optional scale
on the last.  The transforms sit apart with sentinel guards between them, so an addressing slip corrupts a neighbour or a
guard (the call then fails) instead of reading the right bytes by chance.

The pass plan depends on L alone: one pass up to NTT_DMAX = 10, where the pre-multiplier and the post-scale meet in one
launch (n = 1 included), two passes up to 20, three from 21, split unevenly (22 = 8 + 7 + 7).  sb_set_tuning(7, 10..12)
changes the tile, hence the columns per CTA, of the passes of degree 8 and more.

Expected values.  One oracle transform per curve and size serves the single-transform cases: x and y = fr_fft(x).  The device
inverse does not scale, so it maps y to n x.  A pre-multiplier p_i = first * inc^i is checked by feeding x / p (or y / p), whose
transform with the pre-multiplier is y (or n x) again, and a post-scale s multiplies the expected values by s; every such
product is the oracle's fr_batch_apply_key.  The Groth16 chain and the PLONK inverse are compared with the oracle's composition,
fr_fft(fr_batch_apply_key(fr_fft(X, inverse=True), one, inc)) and fr_fft(X, inverse=True), row by row.  Up to L = 6 the
expected values are also recomputed with an O(n^2) DFT in Python integers, so the oracle is not their only witness."""
import concurrent.futures
import contextlib
import ctypes
import functools

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import oracle as O  # noqa: E402  (checker only)
from tests import msm_sets as S  # noqa: E402

BN, BLS = O.BN254, O.BLS12_381
CURVE_IDS = {BN: "bn254", BLS: "bls12381"}
TILE_DEFAULT = 11                            # g_ntt_tile_log in fr_kernels.cu; sb_set_tuning(7, 0) is refused
PASS_L = {BN: list(range(23)), BLS: [0, 1, 9, 10, 11, 15, 20, 21, 22]}
CHAIN_L = (1, 4, 10, 11, 16)
CHAIN_BATCHES = ((0, 1), (0, 2), (0, 3), (0, 4), (1, 3), (1, 5), (1, 6), (1, 12))   # (layout, count)
CHAIN_ROWS = 12
DFT_MAX_L = 6
LAYOUTS_MAX_L = 16


@pytest.fixture(scope="module")
def curves():
    import snarkjs_b200
    cs = {BN: snarkjs_b200.getCurveFromName("bn128"), BLS: snarkjs_b200.getCurveFromName("bls12381")}
    yield cs
    for c in cs.values():
        c.terminate()


def _ptr(a):
    from snarkjs_b200.curve import _ptr as p
    return p(a)


# ----------------------------------------------------------------------------------------------- field helpers
def R(cid):
    return O.CURVES[cid].r


def mont(cid, v) -> bytes:
    return O.CURVES[cid].fr_to_mont(v)


@functools.lru_cache(maxsize=None)
def _nqr(r):
    k = 2
    while pow(k, (r - 1) // 2, r) != r - 1:
        k += 1
    return k


def root(cid, L):
    """Plain primitive 2^L-th root of unity Fr.w[L]: w[s] = nqr^((r-1)/2^s) for the first non-residue nqr from 2, w[i] = w[i+1]^2."""
    r = R(cid)
    s = ((r - 1) & -(r - 1)).bit_length() - 1
    return pow(_nqr(r), ((r - 1) >> s) << (s - L), r)


def shift(cid):
    """Plain Fr.shift = nqr^2, the coset generator of a domain of 2^Fr.s points."""
    return _nqr(R(cid)) ** 2 % R(cid)


def consts(cid, L):
    """Pre-multiplier (first, inc) and post-scale for size 2^L: plain, far from 1."""
    r = R(cid)
    return pow(5, 101 + L, r), pow(7, 103 + L, r), pow(11, 107 + L, r)


def passes(L):
    """ntt_plan's pass count: one pass of degree L up to NTT_DMAX = 10, then ceil(L / 10)."""
    return 1 if L <= 10 else (L + 9) // 10


def rand_fr(cid, n, seed):
    """n Fr elements in Montgomery form, uniform below 2^253 (< r on both curves), starting with r - 1, 0 and R mod r (one)."""
    a = np.random.default_rng(seed).integers(0, 256, (n, 32), dtype=np.uint8)
    a[:, 31] &= 0x1F
    for i, v in enumerate((R(cid) - 1, 0, (1 << 256) % R(cid))[:n]):
        a[i] = np.frombuffer(v.to_bytes(32, "little"), np.uint8)
    a = a.reshape(-1)
    a.setflags(write=False)
    return a


def apply_key(cid, data, first, inc=1):
    """The oracle's fr_batch_apply_key, out[i] = data[i] * first * inc^i (first, inc plain; data Montgomery).  Its loop is
    serial, so large inputs go through it in chunks on several threads (ctypes releases the GIL), chunk k from first * inc^lo."""
    r = R(cid)
    n = data.size // 32
    parts = 8 if n >= 1 << 14 else 1
    lo = [n * k // parts for k in range(parts + 1)]

    def run(k):
        return O.fr_batch_apply_key(cid, data[lo[k] * 32:lo[k + 1] * 32], mont(cid, first * pow(inc, lo[k], r)), mont(cid, inc))
    with concurrent.futures.ThreadPoolExecutor(parts) as ex:
        out = np.concatenate(list(ex.map(run, range(parts))))
    out.setflags(write=False)
    return out


def ints(data):
    b = bytes(data)
    return [int.from_bytes(b[i:i + 32], "little") for i in range(0, len(b), 32)]


def enc(vals):
    return np.frombuffer(b"".join(int(v).to_bytes(32, "little") for v in vals), np.uint8)


def dft(cid, L, data, inverse, pre=None, post=None):
    """The rows of `data` through the O(n^2) definition in Python integers:
    out_j = post * sum_i in_i * first * inc^i * w^(+-ij), w = Fr.w[L], no 1/n.  A Montgomery residue times a plain integer is
    the residue of the product, so the matrix applies to the bytes as they are."""
    r, n = R(cid), 1 << L
    w = pow(root(cid, L), -1 if inverse else 1, r)
    f, g = pre or (1, 1)
    s = 1 if post is None else post
    M = np.array([[s * f * pow(g, i, r) * pow(w, i * j, r) % r for i in range(n)] for j in range(n)], dtype=object)
    X = np.array(ints(data), dtype=object).reshape(-1, n).T
    return enc((M.dot(X) % r).T.reshape(-1))


def diff(got, want, what):
    g, w = np.asarray(got).reshape(-1, 32), np.asarray(want).reshape(-1, 32)
    if g.shape != w.shape:
        return f"{what}: {g.shape[0]} elements, expected {w.shape[0]}"
    bad = np.flatnonzero((g != w).any(axis=1))
    return f"{what}: {len(bad)} of {len(w)} elements differ, the first at {bad[0] if len(bad) else '-'}"


# ----------------------------------------------------------------------------------------------- the hook
def ntt_eval(c, L, data, layout, inverse, pre=None, post=None):
    """sb_ntt_eval over the rows of `data` (count = size / 2^L): pre = (first, inc) and post as plain integers."""
    data = np.ascontiguousarray(data, np.uint8).reshape(-1)
    out = np.empty_like(data)
    first, inc = (mont(c.id, pre[0]), mont(c.id, pre[1])) if pre else (None, None)
    scale = mont(c.id, post) if post is not None else None
    c.check(c.lib.sb_ntt_eval(c.handle, L, data.size >> (L + 5), layout, int(inverse), first, inc, scale, _ptr(data), _ptr(out)))
    return out


@contextlib.contextmanager
def ntt_tile(lib, tile):
    try:
        assert lib.sb_set_tuning(7, tile) == 0, tile
        yield
    finally:
        lib.sb_set_tuning(7, TILE_DEFAULT)


# ----------------------------------------------------------------------------------------------- expected values
@functools.lru_cache(maxsize=None)
def plan_case(cid, L):
    """x and the oracle's y = fr_fft(x), one transform of 2^L."""
    x = rand_fr(cid, 1 << L, 100 * cid + L)
    y = O.fr_fft(cid, x)
    y.setflags(write=False)
    return x, y


@functools.lru_cache(maxsize=None)
def plan_cases(cid, L):
    """{name: (inverse, input, pre, post, expected)} for the eight fusions of one transform.  The inverse's post-scale is 1/n,
    the value PLONK and fflonk fold into their inverse transforms."""
    r, n = R(cid), 1 << L
    x, y = plan_case(cid, L)
    f, g, s = consts(cid, L)
    pre, ninv = (f, g), pow(n, -1, r)
    xp = apply_key(cid, x, pow(f, -1, r), pow(g, -1, r))    # x / p: its transform with the pre-multiplier p is y
    yp = apply_key(cid, y, pow(f, -1, r), pow(g, -1, r))
    ys, nx = apply_key(cid, y, s), apply_key(cid, x, n)
    return {"fwd": (False, x, None, None, y),
            "fwd post": (False, x, None, s, ys),
            "fwd pre": (False, xp, pre, None, y),
            "fwd pre post": (False, xp, pre, s, ys),
            "inv": (True, y, None, None, nx),
            "inv post": (True, y, None, ninv, x),
            "inv pre": (True, yp, pre, None, nx),
            "inv pre post": (True, yp, pre, ninv, x)}


@functools.lru_cache(maxsize=None)
def plan_batch(cid, L, name, count):
    """`count` rows for one fusion of plan_cases: row j is (j + 1) times its input, so neighbouring rows differ everywhere,
    and its expected transform is (j + 1) times the expected one."""
    inverse, inp, pre, post, want = plan_cases(cid, L)[name]
    rows = np.concatenate([inp] + [apply_key(cid, inp, j + 1) for j in range(1, count)])
    wants = np.concatenate([want] + [apply_key(cid, want, j + 1) for j in range(1, count)])
    return inverse, rows, pre, post, wants


@functools.lru_cache(maxsize=None)
def chain_case(cid, L, inc_name):
    """CHAIN_ROWS random inputs X_k and the oracle's Groth16 chain of each, fr_fft(fr_batch_apply_key(fr_fft(X_k,
    inverse=True), one, inc)): inc = w_{2n} (Fr.w[L + 1]) or, for a domain of 2^Fr.s, Fr.shift."""
    n = 1 << L
    inc = root(cid, L + 1) if inc_name == "w2n" else shift(cid)
    X = rand_fr(cid, CHAIN_ROWS * n, 7000 + 100 * cid + L)
    one, minc = mont(cid, 1), mont(cid, inc)
    want = np.concatenate([O.fr_fft(cid, O.fr_batch_apply_key(cid, O.fr_fft(cid, X[k * n * 32:(k + 1) * n * 32], inverse=True), one, minc))
                           for k in range(CHAIN_ROWS)])
    return X, inc, want


def groth16_chain(c, L, X, layout, inc):
    """Groth16's launches: the unscaled inverse, then the coset transform with 1/n folded into the pre-multiplier."""
    n = 1 << L
    u = ntt_eval(c, L, X, layout, True)
    return ntt_eval(c, L, u, layout, False, pre=(pow(n, -1, R(c.id)), inc))


def dft_chain(cid, L, X, inc):
    n = 1 << L
    return dft(cid, L, dft(cid, L, X, True), False, pre=(pow(n, -1, R(cid)), inc))


# ----------------------------------------------------------------------------------------------- 1. every pass plan
PLAN = [(cid, L) for cid in (BN, BLS) for L in PASS_L[cid]]


@pytest.mark.parametrize("cid,L", PLAN, ids=[f"{CURVE_IDS[c]}-L{L}" for c, L in PLAN])
def test_pass_plan(curves, cid, L):
    """One transform of 2^L, forward and inverse, with and without the pre-multiplier and the post-scale, in both layouts
    (from 2^17 each fusion in one of them, alternately)."""
    c = curves[cid]
    for i, (name, (inverse, inp, pre, post, want)) in enumerate(plan_cases(cid, L).items()):
        for layout in (0, 1) if L <= LAYOUTS_MAX_L else (i % 2,):
            got = ntt_eval(c, L, inp, layout, inverse, pre, post)
            assert np.array_equal(got, want), diff(got, want, f"{name}, layout {layout}")
        if L <= DFT_MAX_L:
            assert np.array_equal(want, dft(cid, L, inp, inverse, pre, post)), f"{name}: the oracle's values differ from the DFT"


# ----------------------------------------------------------------------------------------------- 2. the Groth16 chain
@pytest.mark.parametrize("L", CHAIN_L)
@pytest.mark.parametrize("cid", (BN, BLS), ids=list(CURVE_IDS.values()))
def test_groth16_chain(curves, cid, L):
    """Unscaled inverse into the coset transform (first = 1/n, inc = w_{2n}) over 1 to 4 transforms by pointer and 3 to 12
    strided ones, each row its own random input."""
    c = curves[cid]
    assert mont(cid, root(cid, L + 1)) == c.Fr.w[L + 1]
    X, inc, want = chain_case(cid, L, "w2n")
    for layout, count in CHAIN_BATCHES:
        m = count << (L + 5)
        got = groth16_chain(c, L, X[:m], layout, inc)
        assert np.array_equal(got, want[:m]), diff(got, want[:m], f"layout {layout}, count {count}")
    if L <= DFT_MAX_L:
        assert np.array_equal(want, dft_chain(cid, L, X, inc)), "the oracle's chain differs from the DFT"


@pytest.mark.parametrize("L", (4, 11))
@pytest.mark.parametrize("cid", (BN, BLS), ids=list(CURVE_IDS.values()))
def test_groth16_chain_shift_coset(curves, cid, L):
    """The chain with inc = Fr.shift: the arithmetic of a 2^Fr.s domain (groth16_qap_ntt's power == Fr.s branch), whose
    keys are too large for a proof test, run at a small size."""
    c = curves[cid]
    assert mont(cid, shift(cid)) == c.Fr.shift
    X, inc, want = chain_case(cid, L, "shift")
    for layout, count in ((0, 3), (1, 5)):
        m = count << (L + 5)
        got = groth16_chain(c, L, X[:m], layout, inc)
        assert np.array_equal(got, want[:m]), diff(got, want[:m], f"layout {layout}, count {count}")
    if L <= DFT_MAX_L:
        assert np.array_equal(want, dft_chain(cid, L, X, inc)), "the oracle's chain differs from the DFT"


# ----------------------------------------------------------------------------------------------- 3. the PLONK / fflonk launch
@functools.lru_cache(maxsize=None)
def plonk_case(cid, L):
    """Seven rows, a random one, all zeros, r - 1 everywhere, then four random ones, and the oracle's Fr.ifft of each."""
    n = 1 << L
    rnd = rand_fr(cid, 5 * n, 9000 + 100 * cid + L).reshape(5, -1)
    full = np.tile(np.frombuffer((R(cid) - 1).to_bytes(32, "little"), np.uint8), n)
    rows = [rnd[0], np.zeros(n * 32, np.uint8), full, rnd[1], rnd[2], rnd[3], rnd[4]]
    return np.concatenate(rows), np.concatenate([O.fr_fft(cid, row, inverse=True) for row in rows])


@pytest.mark.parametrize("L", (3, 10, 11, 14, 18))
@pytest.mark.parametrize("cid", (BN, BLS), ids=list(CURVE_IDS.values()))
def test_plonk_strided_inverse(curves, cid, L):
    """fr_ntt_strided inverse with the 1/n post-scale over 1, 2 and 7 transforms: each row is Fr.ifft of its own row."""
    c = curves[cid]
    X, want = plonk_case(cid, L)
    ninv = pow(1 << L, -1, R(cid))
    for count in (1, 2, 7):
        m = count << (L + 5)
        got = ntt_eval(c, L, X[:m], 1, True, post=ninv)
        assert np.array_equal(got, want[:m]), diff(got, want[:m], f"count {count}")
    if L <= DFT_MAX_L:
        assert np.array_equal(want, dft(cid, L, X, True, post=ninv)), "the oracle's values differ from the DFT"


# ----------------------------------------------------------------------------------------------- 4. the grid's y limit
@pytest.mark.parametrize("L", (1, 2))
@pytest.mark.parametrize("cid", (BN, BLS), ids=list(CURVE_IDS.values()))
def test_strided_grid_limit(curves, cid, L):
    """65535 strided transforms, the most one launch takes (blockIdx.y): the forward with both fusions and the scaled inverse.
    Every row is compared with the DFT, the first, middle and last rows also with the oracle."""
    c = curves[cid]
    r, n, count = R(cid), 1 << L, 65535
    f, g, s = consts(cid, L)
    X = rand_fr(cid, count * n, 11000 + 100 * cid + L)
    for inverse, pre, post in ((False, (f, g), s), (True, None, pow(n, -1, r))):
        got = ntt_eval(c, L, X, 1, inverse, pre, post)
        want = dft(cid, L, X, inverse, pre, post)
        assert np.array_equal(got, want), diff(got, want, f"inverse={inverse}")
        for k in (0, 1, count // 2, count - 2, count - 1):
            row = X[k * n * 32:(k + 1) * n * 32]
            exp = O.fr_fft(cid, row, inverse=True) if inverse else apply_key(cid, O.fr_fft(cid, apply_key(cid, row, f, g)), s)
            assert np.array_equal(got[k * n * 32:(k + 1) * n * 32], exp), (inverse, k)


# ----------------------------------------------------------------------------------------------- 5. tile settings
TILE_L = (10, 11, 12, 13, 14, 20, 21, 22)
TILE_CASES = ("inv", "fwd pre", "inv post", "fwd pre post")   # Groth16's two launches, PLONK's, and both fusions at once
TILE_CASES_LARGE = ("inv post", "fwd pre post")


@pytest.mark.parametrize("tile", (10, 12))
@pytest.mark.parametrize("cid", (BN, BLS), ids=list(CURVE_IDS.values()))
def test_tile_settings(curves, cid, tile):
    """sb_set_tuning(7, tile) around the default 11, at the sizes where the plan or the columns per CTA change: the fused
    launches over 3 transforms by pointer and 5 strided ones (from 2^20: 2 and 2, with both fusions in each direction), and
    the Groth16 chain up to 2^14."""
    c = curves[cid]
    with ntt_tile(c.lib, tile):
        for L in TILE_L:
            for name in TILE_CASES if L <= 14 else TILE_CASES_LARGE:
                for layout, count in ((0, 3), (1, 5)) if L <= 14 else ((0, 2), (1, 2)):
                    inverse, rows, pre, post, want = plan_batch(cid, L, name, count)
                    got = ntt_eval(c, L, rows, layout, inverse, pre, post)
                    assert np.array_equal(got, want), diff(got, want, f"L={L} {name}, layout {layout}, count {count}")
            if L <= 14:
                X, inc, want = chain_case(cid, L, "w2n")
                for layout, count in ((0, 3), (1, 5)):
                    m = count << (L + 5)
                    got = groth16_chain(c, L, X[:m], layout, inc)
                    assert np.array_equal(got, want[:m]), diff(got, want[:m], f"L={L} chain, layout {layout}, count {count}")


# ----------------------------------------------------------------------------------------------- 6. refusals
def test_ntt_eval_refusals(curves):
    """Out-of-range arguments are SB_ERR_ARG before any device work; the smallest valid calls of each layout succeed."""
    buf = np.zeros(8 * 32, np.uint8)
    out = np.zeros(8 * 32, np.uint8)
    one = mont(BN, 1)
    for cid, c in curves.items():
        lib, h, s = c.lib, c.handle, c.Fr.s

        def call(L, count, layout, first=None, inc=None, src=_ptr(buf), dst=_ptr(out)):
            return lib.sb_ntt_eval(h, L, count, layout, 0, first, inc, None, src, dst)
        for L, count, layout in ((s + 1, 1, 0), (s + 1, 1, 1), (-1, 1, 0), (1, 0, 0), (1, 5, 0), (1, -1, 0), (1, 0, 1),
                                 (1, 65536, 1), (1, 1, 2), (1, 1, -1)):
            assert call(L, count, layout) == -1, (cid, L, count, layout)
            assert b"sb_ntt_eval" in lib.sb_last_error(h)
        assert call(1, 1, 0, src=None) == -1 and call(1, 1, 1, dst=None) == -1
        assert call(1, 1, 0, first=one) == -1 and call(1, 1, 1, inc=one) == -1
        assert lib.sb_ntt_eval(None, 1, 1, 0, 0, None, None, None, _ptr(buf), _ptr(out)) == -1
        assert call(1, 4, 0) == 0 and call(2, 2, 1) == 0 and call(0, 1, 0, first=one, inc=one) == 0


# ----------------------------------------------------------------------------------------------- 7. device-pointer entries
@contextlib.contextmanager
def dev_buffers(c, *sizes):
    ptrs = []
    try:
        for b in sizes:
            p = c.lib.sb_dev_alloc(c.handle, b)
            assert p, f"sb_dev_alloc({b}) failed"
            ptrs.append(p)
        yield ptrs
    finally:
        for p in ptrs:
            c.check(c.lib.sb_dev_free(c.handle, p))


@pytest.mark.parametrize("cid", (BN, BLS), ids=list(CURVE_IDS.values()))
def test_ntt_fr_dev(curves, cid):
    """sb_ntt_fr_dev equals Fr.fft / Fr.ifft and returns the buffer the last pass wrote: every pass moves the data to the
    other buffer (one pass up to 2^10, two up to 2^20, three from 2^21); n = 1 is returned as it is."""
    c = curves[cid]
    lib, h = c.lib, c.handle
    for L in (0, 5, 10, 11, 21):
        n = 1 << L
        x, y = plan_case(cid, L)
        for inverse, inp, want in ((False, x, y), (True, y, x)):
            out = np.empty(n * 32, np.uint8)
            with dev_buffers(c, n * 32, n * 32) as (data, scratch):
                c.check(lib.sb_dev_upload(h, data, _ptr(np.ascontiguousarray(inp)), n * 32))
                res = ctypes.c_void_p()
                c.check(lib.sb_ntt_fr_dev(h, data, scratch, n, int(inverse), ctypes.byref(res)))
                assert res.value == (scratch if L and passes(L) % 2 else data), (L, inverse)
                c.check(lib.sb_dev_download(h, _ptr(out), res.value, n * 32))
            assert np.array_equal(out, want), diff(out, want, f"L={L} inverse={inverse}")


GROUPS = [(BN, 1), (BN, 2), (BLS, 1), (BLS, 2)]


@pytest.mark.parametrize("cid,grp", GROUPS, ids=["bn254_g1", "bn254_g2", "bls12381_g1", "bls12381_g2"])
def test_msm_dev(curves, cid, grp):
    """sb_msm_dev on device copies of random bases and of P, -P, P, ... (doublings and cancellations in the buckets), with
    32- and 13-byte scalars, uniform and all equal (zero on the P, -P set), equals the oracle's multiExpAffine."""
    c = curves[cid]
    G = c.G1 if grp == 1 else c.G2
    n = 1500
    for bname in ("random", "p_neg_p"):
        bases = S.random_bases(cid, grp, n) if bname == "random" else S.base_set(cid, grp, "p_neg_p", n)
        for sb in (32, 13):
            for kind in ("uniform", "equal"):
                sc = S.scalar_set(cid, kind, n, sb)
                out = np.empty(G.sJacobian, np.uint8)
                with dev_buffers(c, bases.size, sc.size) as (db, ds):
                    c.check(c.lib.sb_dev_upload(c.handle, db, _ptr(np.ascontiguousarray(bases)), bases.size))
                    c.check(c.lib.sb_dev_upload(c.handle, ds, _ptr(np.ascontiguousarray(sc)), sc.size))
                    c.check(c.lib.sb_msm_dev(c.handle, grp, db, ds, sb, n, _ptr(out)))
                want = O.g_to_affine(cid, grp, O.multiexp_affine(cid, grp, bases, sc))
                assert G.toAffine(out).tobytes() == want, (bname, sb, kind)
