"""G1/G2 fft, ifft, lagrangeEvaluations and batchApplyKey on the GPU (csrc/gfft.cuh through sb_group_fft /
sb_group_batch_apply_key and curve.py), and powersoftau prepare phase2 built on them:
  * byte parity with the CPU oracle for n = 2^0..2^12 (BN254 G1) / 2^0..2^10 (the other pairs), both directions, every
    affine / Jacobian input and output combination, with infinity, repeated points, P / -P pairs and the MSM tests'
    degenerate base sets;
  * the bytes the reference wrote into sections 12-15 of powersOfTau15_final.ptau, through lagrangeEvaluations and through
    snarkjs_b200.ptau.prepare_phase2 on a power-10 ptau cut from the fixture;
  * sizes beyond the oracle: fft(ifft(x)) == x at 2^20 / 2^18 / 2^16 points, with sampled ifft outputs checked against
    an MSM of the same points (a validated path) and a known-tau Lagrange check;
  * batchApplyKey against the oracle at 2^12 on all four pairs, and the error texts."""
import ctypes

import numpy as np
import pytest

from oracle import oracle as O
from tests import gfft_cases as GC
from tests import gfft_oracle as GO
from tests import msm_sets as S

pytestmark = pytest.mark.gpu

NAME = {O.BN254: "bn128", O.BLS12_381: "bls12381"}
MAXLOG = {(O.BN254, 1): 12, (O.BN254, 2): 10, (O.BLS12_381, 1): 10, (O.BLS12_381, 2): 10}
BIG = {(O.BN254, 1): 20, (O.BN254, 2): 18, (O.BLS12_381, 1): 18, (O.BLS12_381, 2): 16}
COMBOS = [("affine", "affine"), ("affine", "jacobian"), ("jacobian", "affine"), ("jacobian", "jacobian")]


@pytest.fixture(scope="module")
def curves():
    import snarkjs_b200
    cs = {cid: snarkjs_b200.getCurveFromName(NAME[cid]) for cid in (O.BN254, O.BLS12_381)}
    yield cs
    for c in cs.values():
        c.terminate()


@pytest.fixture(scope="module")
def g():
    return GC.goldens()


def group(curves, cid, grp):
    c = curves[cid]
    return c.G1 if grp == 1 else c.G2


_inputs = {}


def sweep_input(cid, grp):
    """2^MAXLOG points k_i G as un-normalised Jacobian and as affine bytes; every prefix of 8 or more points holds
    infinity, a repeated point and two P / -P pairs."""
    if (cid, grp) not in _inputs:
        jac = GC.points_jac(cid, grp, GC.degenerate_scalars(cid, 1 << MAXLOG[(cid, grp)]))
        _inputs[(cid, grp)] = (jac, O.batch_to_affine(cid, grp, jac))
    return _inputs[(cid, grp)]


def check_all_combos(G, cid, grp, jac, aff, inverse):
    raw = GO.group_fft(cid, grp, aff, inverse=inverse, out_jacobian=True)
    want, want_jac = O.batch_to_affine(cid, grp, raw), GC.normalise_jac(cid, grp, raw)
    fn = G.ifft if inverse else G.fft
    for tin, tout in COMBOS:
        got = fn(jac if tin == "jacobian" else aff, tin, tout)
        ref = want_jac if tout == "jacobian" else want
        assert got.tobytes() == ref.tobytes(), (tin, tout)


@pytest.mark.parametrize("cid,grp", GC.CASES)
@pytest.mark.parametrize("inverse", [False, True])
def test_group_fft_vs_oracle_sweep(curves, cid, grp, inverse):
    G = group(curves, cid, grp)
    jac_all, aff_all = sweep_input(cid, grp)
    sj, sa = 3 * G.n8, 2 * G.n8
    for k in range(MAXLOG[(cid, grp)] + 1):
        n = 1 << k
        check_all_combos(G, cid, grp, jac_all[:n * sj], aff_all[:n * sa], inverse)


@pytest.mark.parametrize("cid,grp", GC.CASES)
@pytest.mark.parametrize("name", S.BASE_SETS)
def test_group_fft_degenerate_base_sets(curves, cid, grp, name):
    G = group(curves, cid, grp)
    n = 128
    aff = np.ascontiguousarray(S.base_set(cid, grp, name, n)).reshape(-1)
    jac = np.frombuffer(b"".join(O.g_from_affine(cid, grp, aff[i * 2 * G.n8:(i + 1) * 2 * G.n8].tobytes()) for i in range(n)), np.uint8)
    for inverse in (False, True):
        check_all_combos(G, cid, grp, jac, aff, inverse)


@pytest.mark.parametrize("sid,src,grp,kmax", GC.SECTIONS)
def test_lagrange_evaluations_match_reference_sections(curves, g, sid, src, grp, kmax):
    G = group(curves, O.BN254, grp)
    pts = GC.section_points(g, src)
    want = GC.block_digests(g, sid)
    for k in range(kmax + 1):
        got = G.lagrangeEvaluations(pts[:(1 << k) * 64 * grp])
        assert GC.digest(got) == want[k].tobytes(), f"section {sid} block 2^{k}"


def test_prepare_phase2_gpu(curves, g):
    from snarkjs_b200 import ptau as P
    src = GC.truncated_ptau(g)
    out = P.prepare_phase2(src)
    s_in, s_out = GC.sections(src), GC.sections(out)
    assert list(O.read_binfile(out, "ptau", 1)[1]) == [1, 2, 3, 4, 5, 6, 7, 12, 13, 14, 15]
    for sid in range(1, 8):
        assert s_out[sid] == s_in[sid]
    power = GC.TRUNC_POWER
    for sid, _src, grp, _k in GC.SECTIONS:
        sg = 64 * grp
        want = GC.block_digests(g, sid)
        for k in range(power + 1):
            assert GC.digest(s_out[sid][((1 << k) - 1) * sg:((2 << k) - 1) * sg]) == want[k].tobytes(), (sid, k)
    top = s_out[12][((1 << (power + 1)) - 1) * 64:]
    assert top == GO.group_fft(O.BN254, 1, s_in[2] + bytes(64), inverse=True).tobytes()


def fr_powers_plain(c, n, first: int, inc: int) -> np.ndarray:
    """first * inc^i, i < n, as plain Fr bytes (GPU Fr.batchApplyKey + batchFromMontgomery, both validated elsewhere)."""
    ci = O.CURVES[c.id]
    ones = np.frombuffer(ci.fr_to_mont(1) * n, np.uint8)
    return c.Fr.batchFromMontgomery(c.Fr.batchApplyKey(ones, ci.fr_to_mont(first), ci.fr_to_mont(inc)))


@pytest.mark.parametrize("cid,grp", GC.CASES)
def test_group_fft_large_roundtrip_and_msm(curves, cid, grp):
    c = curves[cid]
    G = group(curves, cid, grp)
    ci = O.CURVES[cid]
    L = BIG[(cid, grp)]
    n = 1 << L
    x = np.empty(n * 2 * G.n8, np.uint8)
    c.check(c.lib.sb_gen_points(c.handle, grp, 5, n, x.ctypes.data_as(ctypes.c_void_p)))
    x.reshape(n, -1)[3] = 0                              # one point at infinity
    y = G.ifft(x)
    w = ci.fr_from_mont(c.Fr.w[L])
    winv, ninv = pow(w, -1, ci.r), pow(n, -1, ci.r)
    for j in (0, 1, n // 2 + 3, n - 1):
        sc = fr_powers_plain(c, n, ninv, pow(winv, j, ci.r))
        want = G.toAffine(G.multiExpAffine(x, sc))
        assert y[j * 2 * G.n8:(j + 1) * 2 * G.n8].tobytes() == want.tobytes(), j
    assert G.fft(y).tobytes() == x.tobytes()
    yj = G.ifft(x, "affine", "jacobian")
    assert G.fft(yj, "jacobian", "affine").tobytes() == x.tobytes()


@pytest.mark.parametrize("cid,grp", GC.CASES)
def test_known_tau_lagrange(curves, cid, grp):
    G = group(curves, cid, grp)
    c = curves[cid]
    ci = O.CURVES[cid]
    L = 12 if (cid, grp) == (O.BN254, 1) else 10
    n = 1 << L
    gen = O.g_to_affine(cid, grp, GC.generator_jac(cid, grp))
    tau = 0x5EED_0F_7A0 * 1000003 + 17
    powers = G.batchApplyKey(np.frombuffer(gen * n, np.uint8), ci.fr_to_mont(1), ci.fr_to_mont(tau))
    sa = 2 * G.n8
    for i in (0, 1, 2, n - 1):
        want = O.g_to_affine(cid, grp, O.g_times(cid, grp, GC.generator_jac(cid, grp), GC.fr_plain(cid, pow(tau, i, ci.r))))
        assert powers[i * sa:(i + 1) * sa].tobytes() == want
    lag = G.lagrangeEvaluations(powers)
    w = ci.fr_from_mont(c.Fr.w[L])
    for j in (0, 1, 5, n - 1):
        wj = pow(w, j, ci.r)
        lj = (pow(tau, n, ci.r) - 1) * wj * pow(n * (tau - wj), -1, ci.r) % ci.r
        want = O.g_to_affine(cid, grp, O.g_times(cid, grp, GC.generator_jac(cid, grp), GC.fr_plain(cid, lj)))
        assert lag[j * sa:(j + 1) * sa].tobytes() == want, j


@pytest.mark.parametrize("cid,grp", GC.CASES)
def test_batch_apply_key_vs_oracle(curves, cid, grp):
    G = group(curves, cid, grp)
    ci = O.CURVES[cid]
    n = 1 << 12
    aff = np.array(S.random_bases(cid, grp, n, 9)).reshape(n, -1)
    aff[7] = 0
    aff[8] = aff[9]
    aff = aff.reshape(-1)
    first, inc = ci.fr_to_mont(987654321987654321), ci.fr_to_mont(ci.r - 12345)
    want = GO.group_batch_apply_key(cid, grp, aff, first, inc)
    assert G.batchApplyKey(aff, first, inc).tobytes() == want.tobytes()
    want_jac = GC.normalise_jac(cid, grp, GO.group_batch_apply_key(cid, grp, aff, first, inc, out_jacobian=True))
    assert G.batchApplyKey(aff, first, inc, "affine", "jacobian").tobytes() == want_jac.tobytes()
    jac = G.batchApplyKey(aff, ci.fr_to_mont(1), ci.fr_to_mont(1), "affine", "jacobian")
    assert G.batchApplyKey(jac, first, inc, "jacobian", "affine").tobytes() == want.tobytes()
    # the point count is floor(bytes / point size); no points -> empty
    assert G.batchApplyKey(aff[:2 * G.n8 * 3 + 5], first, inc).tobytes() == want[:2 * G.n8 * 3].tobytes()
    assert G.batchApplyKey(aff[:5], first, inc).size == 0


def test_group_fft_errors(curves):
    from snarkjs_b200.curve import SbError
    c = curves[O.BN254]
    G = c.G1
    pts = O.gen_points(O.BN254, 1, 1, 3)
    with pytest.raises(SbError, match="fft must be multiple of 2"):
        G.fft(pts)
    with pytest.raises(SbError, match="fft must be multiple of 2"):
        G.ifft(pts[:10])
    with pytest.raises(SbError, match="lagrangeEvaluations invalid Input size"):
        G.lagrangeEvaluations(pts)
    # log2(n) = Fr.s + 1 is the reference's fftExt path: refused before any input is read
    s = c.Fr.s
    out = np.zeros(64, np.uint8)
    rc = c.lib.sb_group_fft(c.handle, 1, pts.ctypes.data_as(ctypes.c_void_p), 0, 1 << (s + 1), 1, 0, out.ctypes.data_as(ctypes.c_void_p))
    assert rc == -1 and "fftExt path not supported" in c.lib.sb_last_error(c.handle).decode()
    big = np.lib.stride_tricks.as_strided(np.zeros(1, np.uint8), shape=((1 << (s + 2)) * 64,), strides=(0,))
    with pytest.raises(SbError, match="lagrangeEvaluations input too big"):
        G.lagrangeEvaluations(big)
