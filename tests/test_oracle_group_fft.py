"""The CPU reference group FFT and group batchApplyKey (tests/gfft_oracle.py, the checker of the GPU kernels), pinned on
the CPU:
  * its ifft of the fixture's tau / alpha-tau / beta-tau prefixes gives the bytes the reference wrote into sections 12-15
    of powersOfTau15_final.ptau (block digests in tests/golden/ptau_prepare_goldens.npz);
  * fft / ifft equal the naive O(n^2) sum of scalar multiplications on all four (curve, group) pairs, with infinity,
    repeated points and P / -P pairs, for every combination of affine / Jacobian input and output;
  * batchApplyKey equals g_times point by point;
  * snarkjs_b200.ptau.prepare_phase2, run with an oracle-backed stand-in curve on a power-10 ptau cut from the fixture,
    reproduces the fixture's block digests (the container logic without a GPU)."""
import pytest

from oracle import oracle as O
from snarkjs_b200 import ptau as P
from tests import gfft_cases as GC
from tests import gfft_oracle as GO

_memo = {}


def oracle_ifft(cid, grp, pts: bytes) -> bytes:
    key = (cid, grp, GC.digest(pts))
    if key not in _memo:
        _memo[key] = GO.group_fft(cid, grp, pts, inverse=True).tobytes()
    return _memo[key]


@pytest.fixture(scope="module")
def g():
    return GC.goldens()


@pytest.mark.parametrize("sid,src,grp,kmax", GC.SECTIONS)
def test_oracle_ifft_matches_reference_sections(g, sid, src, grp, kmax):
    pts = GC.section_points(g, src)
    sg = 64 * grp
    want = GC.block_digests(g, sid)
    assert len(want) == kmax + 1
    for k in range(kmax + 1):
        got = oracle_ifft(O.BN254, grp, pts[:(1 << k) * sg].tobytes())
        assert GC.digest(got) == want[k].tobytes(), f"section {sid} block 2^{k}"


def naive_dft(cid, grp, pts_jac: bytes, inverse: bool):
    """X[k] = sum_j x[j] w^(jk) (forward), x[k] = n^-1 sum_j X[j] w^(-jk) (inverse), by g_times / g_add."""
    ci = O.CURVES[cid]
    sj = 3 * ci.n8q * grp
    n = len(pts_jac) // sj
    L = n.bit_length() - 1
    w = ci.fr_from_mont(O.fr_root(cid, L))
    if inverse:
        w = pow(w, -1, ci.r)
    ninv = pow(n, -1, ci.r) if inverse else 1
    x = [pts_jac[j * sj:(j + 1) * sj] for j in range(n)]
    out = []
    for k in range(n):
        acc = O.group_zero(cid, grp)
        for j in range(n):
            acc = O.g_add(cid, grp, acc, O.g_times(cid, grp, x[j], GC.fr_plain(cid, pow(w, j * k, ci.r) * ninv)))
        out.append(acc)
    return b"".join(out)


@pytest.mark.parametrize("cid,grp", GC.CASES)
@pytest.mark.parametrize("n", [1, 2, 4, 8, 16])
@pytest.mark.parametrize("inverse", [False, True])
def test_oracle_fft_vs_naive(cid, grp, n, inverse):
    jac = GC.points_jac(cid, grp, GC.degenerate_scalars(cid, n)).tobytes()
    aff = O.batch_to_affine(cid, grp, jac).tobytes()
    want = O.batch_to_affine(cid, grp, naive_dft(cid, grp, jac, inverse))
    for in_jac in (False, True):
        for out_jac in (False, True):
            got = GO.group_fft(cid, grp, jac if in_jac else aff, inverse=inverse, in_jacobian=in_jac, out_jacobian=out_jac)
            if out_jac:
                got = O.batch_to_affine(cid, grp, got)
            assert got.tobytes() == want.tobytes(), (in_jac, out_jac)


def test_oracle_fft_size_errors():
    pts = O.gen_points(O.BN254, 1, 1, 3)
    with pytest.raises(ValueError, match="fft must be multiple of 2"):
        GO.group_fft(O.BN254, 1, pts)


@pytest.mark.parametrize("cid,grp", GC.CASES)
@pytest.mark.parametrize("in_jac,out_jac", [(False, False), (True, True), (False, True), (True, False)])
def test_oracle_batch_apply_key(cid, grp, in_jac, out_jac):
    ci = O.CURVES[cid]
    n = 19
    jac = GC.points_jac(cid, grp, GC.degenerate_scalars(cid, n)).tobytes()
    inp = jac if in_jac else O.batch_to_affine(cid, grp, jac).tobytes()
    first, inc = 0x1234567 * 0x89abcdef + 5, ci.r - 77
    got = GO.group_batch_apply_key(cid, grp, inp, GC.fr_mont(cid, first), GC.fr_mont(cid, inc), in_jacobian=in_jac,
                                  out_jacobian=out_jac)
    if out_jac:
        got = O.batch_to_affine(cid, grp, got)
    sj = 3 * ci.n8q * grp
    want = b"".join(O.g_times(cid, grp, jac[i * sj:(i + 1) * sj], GC.fr_plain(cid, first * pow(inc, i, ci.r))) for i in range(n))
    assert got.tobytes() == O.batch_to_affine(cid, grp, want).tobytes()


class OracleCurve:
    """Stand-in for snarkjs_b200.Curve with the oracle behind G1/G2.lagrangeEvaluations (BN254 only: the fixture's curve)."""

    class _G:
        def __init__(self, grp):
            self.grp = grp

        def lagrangeEvaluations(self, buff, inType="affine", outType="affine", logger=None, loggerTxt=""):
            assert (inType, outType) == ("affine", "affine")
            return oracle_ifft(O.BN254, self.grp, bytes(buff))

    def __init__(self):
        self.q = O.P_BN_Q
        self.n8q = 32
        self.G1, self.G2 = self._G(1), self._G(2)


def test_prepare_phase2_container_with_oracle(g):
    src = GC.truncated_ptau(g)
    out = P.prepare_phase2(src, curve=OracleCurve())
    s_in, s_out = GC.sections(src), GC.sections(out)
    assert list(O.read_binfile(out, "ptau", 1)[1]) == [1, 2, 3, 4, 5, 6, 7, 12, 13, 14, 15]
    assert s_out[1] == s_in[1]
    for sid in range(2, 8):
        assert s_out[sid] == s_in[sid]
    power = GC.TRUNC_POWER
    for sid, _src, grp, _k in GC.SECTIONS:
        sg = 64 * grp
        blocks = power + 2 if sid == 12 else power + 1
        assert len(s_out[sid]) == ((1 << blocks) - 1) * sg
        want = GC.block_digests(g, sid)
        for k in range(power + 1):
            assert GC.digest(s_out[sid][((1 << k) - 1) * sg:((2 << k) - 1) * sg]) == want[k].tobytes(), (sid, k)
    # section 12's extra block at power + 1: the 2^11 - 1 tau points and one point at infinity
    top = s_out[12][((1 << (power + 1)) - 1) * 64:]
    assert top == oracle_ifft(O.BN254, 1, s_in[2] + bytes(64))


def test_prepare_phase2_header_checks(g):
    src = bytearray(GC.truncated_ptau(g))
    with pytest.raises(Exception, match="Invalid File format"):
        P.prepare_phase2(b"xxxx" + bytes(src[4:]), curve=OracleCurve())
