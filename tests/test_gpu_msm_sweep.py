"""The MSM on every path its window size can take.  sb_set_tuning(13, c) forces the window bits c, which decide the bucket
count, the number of windows, whether the bucket reduction splits the buckets into rows and columns (c >= 12) and how
many axis-sum levels each side gets, whether it falls back to k_reduce (c >= 22), and how dense the top window is.
Every c runs on the four (curve, group) pairs, in plain mode (bases passed with the call) and in table mode (registered
bases with precomputed window tables), with both bucket reductions, on degenerate bases and on scalars at the edges of
the signed-digit recoding.  Every result is compared, as toAffine bytes, with the CPU oracle's Pippenger over the same
bases and scalars; the oracle does not depend on c, mode or reduction, so each result is computed once and reused.

Plain mode stops at c = 20: a plain MSM allocates W * 2^(c-1) buckets, 2.6 GB on BLS12-381 G2 at c = 20 and 9.7 GB at
c = 22.  Table mode shares one bucket set between the windows and runs up to c = 22."""
import contextlib
import hashlib
import time

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import oracle as O  # noqa: E402  (checker only)
from tests import msm_sets as S  # noqa: E402

BN, BLS = O.BN254, O.BLS12_381
GROUPS = [(BN, 1), (BN, 2), (BLS, 1), (BLS, 2)]
GROUP_IDS = ["bn254_g1", "bn254_g2", "bls12381_g1", "bls12381_g2"]
N = 4133                                    # >= 2^12 (window tables are built) and not a multiple of 32
PLAIN_C = range(3, 21)
TABLE_C = range(3, 23)
# one c per reduction shape: unsplit (3, 8, 11), split with one / two column levels (12, 14, 16, 20), k_reduce (22)
SHAPE_C = (3, 8, 11, 12, 14, 16, 20, 22)
DEFAULTS = {1: 0, 2: 0, 6: 0, 7: 11, 13: 0}


@contextlib.contextmanager
def tuning(lib, settings):
    """Sets process-wide switches (sb_set_tuning) for the block and restores their defaults afterwards."""
    try:
        for k, v in settings.items():
            assert lib.sb_set_tuning(k, v) == 0, (k, v)
        yield
    finally:
        for k in settings:
            lib.sb_set_tuning(k, DEFAULTS[k])


@pytest.fixture(scope="module")
def curves():
    import snarkjs_b200
    cs = {BN: snarkjs_b200.getCurveFromName("bn128"), BLS: snarkjs_b200.getCurveFromName("bls12381")}
    yield cs
    for c in cs.values():
        c.terminate()


_ORACLE = {}


def want(cid, grp, bases, scalars):
    """toAffine bytes of the oracle's Pippenger, memoised on the content of the bases and scalars."""
    key = (cid, grp, hashlib.sha1(np.ascontiguousarray(bases)).digest(), hashlib.sha1(np.ascontiguousarray(scalars)).digest(),
           len(scalars))
    if key not in _ORACLE:
        _ORACLE[key] = O.g_to_affine(cid, grp, O.multiexp_affine(cid, grp, bases, scalars))
    return _ORACLE[key]


def want_ones(cid, grp, bases, c, sbytes):
    """Oracle result for S.scalar_set("ones"): every scalar is the same value v, so the MSM is v * (sum of the bases)."""
    total = O.multiexp_affine(cid, grp, bases, np.ones(len(bases) // S.point_bytes(cid, grp), np.uint8))   # 1-byte scalars 1
    v = S.ones_value(c, sbytes).to_bytes(sbytes + 1, "little")
    return O.g_to_affine(cid, grp, O.g_times(cid, grp, total, v))


def group(curves, cid, grp):
    c = curves[cid]
    return c, (c.G1 if grp == 1 else c.G2)


def plain(G, bases, sc):
    return G.toAffine(G.multiExpAffine(bases, sc)).tobytes()


def registered(G, h, sc, first=0, n=None):
    n = len(sc) // 32 if n is None else n
    return G.toAffine(G.multiExpRegistered(h, sc, first=first, n=n)).tobytes()


def entries(curve, grp):
    """(digit, point) entries the bucket accumulation consumed in the last MSM call."""
    return curve.lib.sb_last_stat(curve.handle, 4 if grp == 1 else 5)


def other_c(c):
    """A window size with a different window count, set while a table built with c is used."""
    return 3 if c != 3 else 4


# ----------------------------------------------------------------------------------------------- heuristics at real sizes
# First in the file: a 2^20-point table is up to 2.6 GB (BLS12-381 G2), so these run on their own short-lived contexts.
@pytest.mark.parametrize("cid,grp", GROUPS, ids=GROUP_IDS)
def test_heuristic_geometry_at_real_sizes(cid, grp):
    """No forcing.  Plain multiExpAffine at 2^17 points picks c = 13 (a split reduction).  A registered set of 2^20 points
    gets c = 20 tables with stride 2^20; MSMs over its start, middle and end are compared on the matching slices."""
    import snarkjs_b200
    from snarkjs_b200 import synth
    curve = snarkjs_b200.getCurveFromName("bn128" if cid == BN else "bls12381")
    try:
        G = curve.G1 if grp == 1 else curve.G2
        sz = S.point_bytes(cid, grp)
        n = 1 << 17
        bases = synth.gen_points(curve, grp, 31 + grp, n)
        sc = O.random_scalars(32 + grp, n, O.CURVES[cid].r)
        assert plain(G, bases, sc) == want(cid, grp, bases, sc)
        ones = S.scalar_set(cid, "ones", n, 32, 13)                    # W(13) = 20 differs from W(12) and W(14)
        assert plain(G, bases, ones) == want_ones(cid, grp, bases, 13, 32)
        assert entries(curve, grp) == n * S.windows(13, 32)
        m = 1 << 20
        big = synth.gen_points(curve, grp, 41 + grp, m)
        t0 = time.perf_counter()
        h = G.registerBases(big)
        print(f"{GROUP_IDS[GROUPS.index((cid, grp))]}: 2^20-point table built in {time.perf_counter() - t0:.2f} s")
        try:
            sc = O.random_scalars(42 + grp, 3000, O.CURVES[cid].r)
            for first in (0, (m >> 1) - 1500, m - 3000):
                got = registered(G, h, sc, first=first, n=3000)
                assert got == want(cid, grp, big[first * sz:(first + 3000) * sz], sc), first
            # the table's c is 20: digit 1 in every window of 32-byte scalars gives 3000 * 13 entries
            ones = S.scalar_set(cid, "ones", 3000, 32, 20)
            registered(G, h, ones, first=m - 3000, n=3000)
            assert entries(curve, grp) == 3000 * S.windows(20, 32)
        finally:
            curve.check(curve.lib.sb_bases_release(curve.handle, h))
    finally:
        curve.terminate()


# ----------------------------------------------------------------------------------------------- a. geometry sweep
SWEEP = [("plain", c) for c in PLAIN_C] + [("table", c) for c in TABLE_C]


@pytest.mark.parametrize("mode,c", SWEEP, ids=[f"{m}-c{c}" for m, c in SWEEP])
@pytest.mark.parametrize("cid,grp", GROUPS, ids=GROUP_IDS)
def test_geometry_sweep(curves, cid, grp, mode, c):
    import ctypes
    from snarkjs_b200.curve import _ptr
    curve, G = group(curves, cid, grp)
    lib = curve.lib
    bases = S.random_bases(cid, grp, N)
    sets = {k: S.scalar_set(cid, k, N) for k in ("uniform", "uniform256")}
    sets["boundary"] = S.scalar_set(cid, "boundary", N, 32, c)
    ones = S.scalar_set(cid, "ones", N, 32, c)
    expect = {k: want(cid, grp, bases, s) for k, s in sets.items()}
    expect_ones = want_ones(cid, grp, bases, c, 32)
    if mode == "plain":
        with tuning(lib, {13: c}):
            for red in (0, 1):
                with tuning(lib, {1: red}):
                    for k, s in sets.items():
                        assert plain(G, bases, s) == expect[k], (k, red)
            assert plain(G, bases, ones) == expect_ones
            assert entries(curve, grp) == N * S.windows(c, 32)
        return
    with tuning(lib, {13: c}):
        h = G.registerBases(bases)
    try:
        # the table keeps the c it was built with: a different forced c at MSM time changes nothing
        with tuning(lib, {13: other_c(c)}):
            for red in (0, 1):
                with tuning(lib, {1: red}):
                    for k, s in sets.items():
                        assert registered(G, h, s) == expect[k], (k, red)
            assert registered(G, h, ones) == expect_ones
            assert entries(curve, grp) == N * S.windows(c, 32)
            # exchange unit: three uneven ranges starting after point 0, summed on the host
            sc = sets["uniform"]
            cuts = (7, 1290, 1291, N)
            pb = lib.sb_msm_partial_bytes(curve.handle, grp)
            parts = np.empty(3 * pb, np.uint8)
            for i in range(3):
                lo, hi = cuts[i], cuts[i + 1]
                curve.check(lib.sb_msm_registered_partial(curve.handle, h, lo, _ptr(np.ascontiguousarray(sc[lo * 32:hi * 32])), 32,
                                                          hi - lo, ctypes.c_void_p(parts.ctypes.data + i * pb)))
            out = np.empty(G.sJacobian, np.uint8)
            curve.check(lib.sb_msm_sum_partials(curve.handle, grp, _ptr(parts), 3, _ptr(out)))
            sz = S.point_bytes(cid, grp)
            assert G.toAffine(out).tobytes() == want(cid, grp, bases[cuts[0] * sz:], sc[cuts[0] * 32:])
    finally:
        curve.check(lib.sb_bases_release(curve.handle, h))


# ----------------------------------------------------------------------------------------------- b. degenerate bases
DEGEN = [("plain", c) for c in SHAPE_C if c <= 20] + [("table", c) for c in SHAPE_C]


@pytest.mark.parametrize("mode,c", DEGEN, ids=[f"{m}-c{c}" for m, c in DEGEN])
@pytest.mark.parametrize("cid,grp", GROUPS, ids=GROUP_IDS)
def test_degenerate_bases(curves, cid, grp, mode, c):
    """Repeated points, P next to -P, and points at infinity: equal and opposite partial sums meet in the bucket
    accumulation, k_fold, the axis sums, the warp sums and k_reduce, where the full addition takes its doubling and
    cancellation branches; k_precompute sees infinity bases."""
    curve, G = group(curves, cid, grp)
    lib = curve.lib
    zero = bytes(S.point_bytes(cid, grp))
    for bname in S.BASE_SETS:
        bases = S.base_set(cid, grp, bname, N)
        sets = {k: S.scalar_set(cid, k, N) for k in ("uniform", "equal", "zero")}
        sets["boundary"] = S.scalar_set(cid, "boundary", N, 32, c)
        with tuning(lib, {13: c}):
            h = G.registerBases(bases) if mode == "table" else None
            try:
                for k, s in sets.items():
                    got = registered(G, h, s) if h else plain(G, bases, s)
                    assert got == want(cid, grp, bases, s), (bname, k)
                    if k == "zero" or bname == "all_inf" or (bname == "p_neg_p" and k == "equal"):
                        assert got == zero, (bname, k)
            finally:
                if h:
                    curve.check(lib.sb_bases_release(curve.handle, h))


# ----------------------------------------------------------------------------------------------- c. boundary scalars by width
WIDTHS = (1, 4, 5, 13, 31, 32)
WIDTH_C = (3, 8, 11, 12, 16, 20, 22)
# c divides 8*sbytes + 1: the top window has c - 1 bits, so with the carry its digit reaches half
TOP_HALF = ((4, 3), (4, 11), (13, 3), (13, 5), (13, 7), (13, 15), (13, 21))
SUB_FIRST, SUB_N = 1000, 400


def width_cases(mode):
    cmax = 20 if mode == "plain" else 22
    pairs = {(sb, c) for sb in WIDTHS for c in WIDTH_C} | set(TOP_HALF)
    return sorted((sb, c) for sb, c in pairs if c <= cmax)


@pytest.mark.parametrize("mode", ["plain", "table"])
@pytest.mark.parametrize("cid,grp", GROUPS, ids=GROUP_IDS)
def test_boundary_scalars_by_width(curves, cid, grp, mode):
    """Per-c boundary scalars at widths of 1 to 32 bytes, on a 400-point range starting at point 1000 of a registered set
    (table mode) or on the same 400 bases passed with the call (plain mode)."""
    curve, G = group(curves, cid, grp)
    lib = curve.lib
    sz = S.point_bytes(cid, grp)
    bases = S.random_bases(cid, grp, N)
    sub = bases[SUB_FIRST * sz:(SUB_FIRST + SUB_N) * sz]
    cases = width_cases(mode)
    for c in sorted({c for _, c in cases}):
        with tuning(lib, {13: c}):
            h = G.registerBases(bases) if mode == "table" else None
            try:
                for sb in sorted(sb for sb, cc in cases if cc == c):
                    s = S.scalar_set(cid, "boundary", SUB_N, sb, c)
                    got = registered(G, h, s, first=SUB_FIRST, n=SUB_N) if h else plain(G, sub, s)
                    assert got == want(cid, grp, sub, s), (sb, c)
                    assert entries(curve, grp) <= SUB_N * S.windows(c, sb)
            finally:
                if h:
                    curve.check(lib.sb_bases_release(curve.handle, h))


@pytest.mark.parametrize("cid,grp", GROUPS, ids=GROUP_IDS)
def test_wide_scalars_on_registered_bases(curves, cid, grp):
    """Scalars wider than the 32 bytes the window tables cover take the raw-bases path of a registered set (plain Pippenger
    on the registered points from `first`), with the heuristic c and with forced ones.  65 bytes is refused."""
    from snarkjs_b200 import SbError
    curve, G = group(curves, cid, grp)
    lib = curve.lib
    sz = S.point_bytes(cid, grp)
    bases = S.random_bases(cid, grp, N)
    sub = bases[SUB_FIRST * sz:(SUB_FIRST + SUB_N) * sz]
    h = G.registerBases(bases)
    try:
        for sb in (33, 40, 64):
            for c in (0, 3, 8, 11, 12, 16):
                s = S.scalar_set(cid, "boundary", SUB_N, sb, c or 16)
                with tuning(lib, {13: c}):
                    got = registered(G, h, s, first=SUB_FIRST, n=SUB_N)
                assert got == want(cid, grp, sub, s), (sb, c)
                if c:
                    assert entries(curve, grp) <= SUB_N * S.windows(c, sb)
            s = S.scalar_set(cid, "uniform256", SUB_N, sb)
            assert registered(G, h, s, first=SUB_FIRST, n=SUB_N) == want(cid, grp, sub, s), sb
        with pytest.raises(SbError, match="Scalar size does not match"):
            G.multiExpRegistered(h, np.zeros(SUB_N * 65, np.uint8), first=SUB_FIRST, n=SUB_N)
        with pytest.raises(SbError, match="Scalar size does not match"):
            G.multiExpAffine(sub, np.zeros(SUB_N * 65, np.uint8))
    finally:
        curve.check(lib.sb_bases_release(curve.handle, h))


# ----------------------------------------------------------------------------------------------- d. chunk and offset edges
@pytest.mark.parametrize("cid,grp", GROUPS, ids=GROUP_IDS)
def test_chunk_and_offset_edges(curves, cid, grp):
    """sb_set_tuning(6, 11): chunks of 2048 points.  13-byte scalars put every chunk's scalars at an odd address, so k_digits
    reads them byte by byte; on a registered set the chunk offset is added to `first`."""
    curve, G = group(curves, cid, grp)
    lib = curve.lib
    sz = S.point_bytes(cid, grp)
    bases = S.random_bases(cid, grp, N)
    first, n = 101, N - 101
    with tuning(lib, {6: 11}):
        for c in (0, 8, 16):
            with tuning(lib, {13: c}):
                for sb in (13, 32):
                    for k in ("uniform256", "boundary"):
                        s = S.scalar_set(cid, k, N, sb, c or 16)
                        assert plain(G, bases, s) == want(cid, grp, bases, s), (c, sb, k)
                        assert plain(G, bases[first * sz:], s[first * sb:]) == want(cid, grp, bases[first * sz:], s[first * sb:]), (c, sb, k)
                h = G.registerBases(bases)
            try:
                for sb in (13, 32):
                    for k in ("uniform256", "boundary"):
                        s = S.scalar_set(cid, k, N, sb, c or 16)[first * sb:]
                        got = registered(G, h, s, first=first, n=n)
                        assert got == want(cid, grp, bases[first * sz:], s), (c, sb, k)
            finally:
                curve.check(lib.sb_bases_release(curve.handle, h))


# ----------------------------------------------------------------------------------------------- f. raw output format
@pytest.mark.parametrize("cid,grp", GROUPS, ids=GROUP_IDS)
def test_raw_output_is_normalised_jacobian(curves, cid, grp):
    """sb_msm_g?_affine, sb_msm_registered and sb_msm_sum_partials return x || y || 1 (Montgomery) for a non-zero
    result and (0, 1, 0) for zero, byte for byte (include/snarkb200.h)."""
    import ctypes
    from snarkjs_b200.curve import _ptr
    curve, G = group(curves, cid, grp)
    lib = curve.lib
    ci = O.CURVES[cid]
    one = ci.fq_to_mont(1) + bytes(ci.n8q * (grp - 1))
    bases = S.random_bases(cid, grp, N)
    h = G.registerBases(bases)
    try:
        for k in ("uniform", "zero"):
            s = S.scalar_set(cid, k, N)
            aff = want(cid, grp, bases, s)
            expect = O.group_zero(cid, grp) if k == "zero" else aff + one
            assert G.multiExpAffine(bases, s).tobytes() == expect, k
            assert G.multiExpRegistered(h, s).tobytes() == expect, k
            pb = lib.sb_msm_partial_bytes(curve.handle, grp)
            part = np.empty(pb, np.uint8)
            curve.check(lib.sb_msm_registered_partial(curve.handle, h, 0, _ptr(np.ascontiguousarray(s)), 32, N, ctypes.c_void_p(part.ctypes.data)))
            out = np.empty(G.sJacobian, np.uint8)
            curve.check(lib.sb_msm_sum_partials(curve.handle, grp, _ptr(part), 1, _ptr(out)))
            assert out.tobytes() == expect, k
    finally:
        curve.check(lib.sb_bases_release(curve.handle, h))


# ----------------------------------------------------------------------------------------------- g. switches that keep the bytes
BLINDERS = [0x3000 + 104729 * i for i in range(11)]


@pytest.fixture(scope="module")
def groth16_case(curves):
    """Synthetic 2^16 Groth16 key with its witness and the oracle's proof."""
    from snarkjs_b200 import synth
    bn = curves[BN]
    zkey = synth.synth_groth16_zkey(bn, 16, seed=13)
    wt = synth.wtns_container(bn.r, synth.chain_witness(bn.r, 16))
    ci = O.CURVES[BN]
    r, s = ci.fr_to_mont(1357), ci.fr_to_mont(2468)
    return zkey, wt, r, s, O.groth16_prove(zkey, wt, r, s)


@pytest.fixture(scope="module")
def plonk_bls_case():
    """Synthetic BLS12-381 PLONK key (1000 gates: domain 1024, quotient NTTs of 4096 points) and the oracle's proof."""
    from oracle import plonk as op
    ci = O.CURVES[BLS]
    gates, adds, n_vars, n_pub, wit = op.chain_gates(1000, r=ci.r)
    zkey = op.plonk_setup_synth(gates, adds, n_vars, n_pub, tau=0xB15B15, curve=BLS)
    wt = op.wtns_bytes(wit, ci.r)
    return zkey, wt, op.plonk_prove(zkey, wt, BLINDERS)


def test_serialised_prove_same_bytes(curves, groth16_case):
    """sb_set_tuning(2, 1) runs every stream of a Groth16 prove call on one stream (per-kernel-class timing): same proof."""
    from snarkjs_b200 import groth16
    zkey, wt, r, s, (oproof, opub) = groth16_case
    pk = groth16.ProvingKey(zkey, curve=curves[BN])
    try:
        proof, pub = groth16.prove(pk, wt, r, s)
        assert proof == oproof and pub == [str(x) for x in opub]
        with tuning(curves[BN].lib, {2: 1}):
            assert groth16.prove(pk, wt, r, s)[0] == proof
    finally:
        pk.release()


def test_ntt_tile_sizes(curves, groth16_case, plonk_bls_case):
    """sb_set_tuning(7, tile): the largest NTT tile 2^10 or 2^12 instead of 2^11.  Fr.fft at 2^11 .. 2^22 equals the
    oracle's, Fr.ifft inverts the oracle's transform exactly, and a Groth16 and a BLS12-381 PLONK proof (the fused coset
    and scale passes) equal the oracle's proofs."""
    from snarkjs_b200 import groth16, plonk
    lib = curves[BN].lib
    for cid in (BN, BLS):
        c = curves[cid]
        for L in range(11, 23):
            x = O.random_scalars(500 + L, 1 << L, O.CURVES[cid].r, bits=253)
            y = O.fr_fft(cid, x)
            for tile in (10, 12):
                with tuning(lib, {7: tile}):
                    assert np.array_equal(c.Fr.fft(x), y), (cid, L, tile)
                    assert np.array_equal(c.Fr.ifft(y), x), (cid, L, tile)
    zkey, wt, r, s, (oproof, opub) = groth16_case
    zkey_p, wt_p, want_plonk = plonk_bls_case
    bl = b"".join(O.CURVES[BLS].fr_to_mont(b) for b in BLINDERS)
    for tile in (10, 12):
        with tuning(lib, {7: tile}):
            pk = groth16.ProvingKey(zkey, curve=curves[BN])
            try:
                proof, pub = groth16.prove(pk, wt, r, s)
                assert proof == oproof and pub == [str(x) for x in opub], tile
            finally:
                pk.release()
            pk = plonk.ProvingKey(zkey_p, curves[BLS])
            try:
                assert plonk.prove(pk, wt_p, bl) == want_plonk, tile
            finally:
                pk.release()
