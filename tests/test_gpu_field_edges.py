"""GPU: the field primitives as compiled for sm_90a, pinned bit for bit to Python big-integer results at their carry and
reduction edges (sb_field_eval over every record of tests/field_edges.py), and the element-wise Fr entry points and Fr.fft /
Fr.ifft of both curves on boundary operands, with expected values in closed form."""
import functools

import numpy as np
import pytest

from tests import ec_edges as EC
from tests import field_edges as FE

pytestmark = pytest.mark.gpu

R256 = 1 << 256
CURVES = ("bn128", "bls12381")


@pytest.fixture(scope="module")
def curves():
    import snarkjs_b200
    cs = {name: snarkjs_b200.getCurveFromName(name) for name in CURVES}
    yield cs
    for c in cs.values():
        c.terminate()


def _ptr(a):
    from snarkjs_b200.curve import _ptr as p
    return p(a)


def _enc(vals) -> np.ndarray:
    return np.frombuffer(b"".join(v.to_bytes(32, "little") for v in vals), np.uint8)


def _dec(buf) -> list[int]:
    b = bytes(buf)
    return [int.from_bytes(b[i:i + 32], "little") for i in range(0, len(b), 32)]


def _first_diff(got, want, what):
    g, w = _dec(got), _dec(want)
    bad = [i for i in range(len(w)) if g[i] != w[i]]
    return f"{what}: {len(bad)} of {len(w)} elements differ; first at {bad[0]}: got {hex(g[bad[0]])} expected {hex(w[bad[0]])}"


# ------------------------------------------------------------------------------------- primitives through sb_field_eval
@pytest.mark.parametrize("field,op", FE.all_sets(), ids=[f"{FE.FIELDS[f][0].replace(' ', '_')}-{FE.OP_NAMES[o]}" for f, o in FE.all_sets()])
def test_field_primitive_edges(curves, field, op):
    c = curves["bn128"]                     # the field does not depend on the context's curve
    recs = FE.records(field, op)
    inp, want = FE.pack(field, recs)
    a = np.frombuffer(inp, np.uint8)
    out = np.zeros(len(want), np.uint8)
    c.check(c.lib.sb_field_eval(c.handle, field, op, _ptr(a), len(recs), _ptr(out)))
    if out.tobytes() != want:
        bad = FE.mismatches(field, op, out.tobytes())
        pytest.fail(f"{len(bad)}+ mismatching records, first ones:\n" + "\n".join(bad))


def test_field_eval_refuses_undefined_field_op_pairs(curves):
    """Ops past the last point op, point ops on the Fr fields and Fp ops on Fq2 are SB_ERR_ARG, as are unknown fields."""
    c = curves["bls12381"]
    buf = np.zeros(4 * 48, np.uint8)
    out = np.zeros(4 * 48, np.uint8)
    refused = [(3, FE.FP_OPS["mul2"]), (0, FE.FP2_OPS["mul_i"]), (6, 0), (-1, 0), (0, FE.FE_NOPS), (4, FE.FE_NOPS),
               (0, -1)]
    refused += [(f, op) for f in (4, 5) for op in FE.FP_OPS.values()]           # Fp ops are not defined on Fq2
    refused += [(f, op) for f in (1, 3) for op in EC.EC_OPS.values()]           # no group over Fr
    for field, op in refused:
        assert c.lib.sb_field_eval(c.handle, field, op, _ptr(buf), 1, _ptr(out)) == -1, (field, op)
        assert b"not defined" in c.lib.sb_last_error(c.handle)
    assert c.lib.sb_field_eval(None, 0, 0, _ptr(buf), 1, _ptr(out)) == -1
    assert c.lib.sb_field_eval(c.handle, 0, 0, _ptr(buf), 0, _ptr(out)) == 0


# ------------------------------------------------------------------------------------- element-wise Fr entry points
def _boundary(r):
    F = FE._F(r, 8)
    return list(F.consts().values()), list(F.raw().values())


@pytest.mark.parametrize("name", CURVES)
def test_fr_convert_boundary(curves, name):
    """batchToMontgomery / batchFromMontgomery on the constant set and, since the kernel takes the caller's bytes unchecked,
    on values in [r, 2^256): a*R mod r and a*R^-1 mod r all the same."""
    c = curves[name]
    r = c.r
    consts, raw = _boundary(r)
    vals = consts + raw
    x = _enc(vals)
    got = c.Fr.batchToMontgomery(x)
    want = _enc([v * R256 % r for v in vals])
    assert np.array_equal(got, want), _first_diff(got, want, "batchToMontgomery")
    got = c.Fr.batchFromMontgomery(x)
    want = _enc([v * pow(R256, -1, r) % r for v in vals])
    assert np.array_equal(got, want), _first_diff(got, want, "batchFromMontgomery")


@pytest.mark.parametrize("name", CURVES)
def test_qap_join_abc_boundary(curves, name):
    """out = fromMontgomery(a*b - c) with a*b = c (out 0) and a*b = c - 1 (out = (r-1)*R^-1) over all constant pairs."""
    c = curves[name]
    r = c.r
    Ri = pow(R256, -1, r)
    consts, _ = _boundary(r)
    A, B, C, W = [], [], [], []
    for a in consts:
        for b in consts:
            ab = a * b * Ri % r
            for d in (0, 1):
                A.append(a), B.append(b), C.append((ab + d) % r), W.append((r - d) % r * Ri % r)
    a, b, cc, out = _enc(A), _enc(B), _enc(C), np.zeros(32 * len(W), np.uint8)
    c.check(c.lib.sb_qap_join_abc(c.handle, _ptr(a), _ptr(b), _ptr(cc), len(W), _ptr(out)))
    want = _enc(W)
    assert np.array_equal(out, want), _first_diff(out, want, "joinABC")


@pytest.mark.parametrize("name", CURVES)
@pytest.mark.parametrize("first", [1, -1, 0], ids=["first=1", "first=-1", "first=0"])
@pytest.mark.parametrize("inc", [1, -1, 0], ids=["inc=1", "inc=-1", "inc=0"])
def test_fr_apply_key_boundary(curves, name, first, inc):
    """batchApplyKey(in, first, inc)[i] = in[i] * first * inc^i with first, inc in {Montgomery 1, Montgomery -1, 0} on
    inputs of r-1 (inc^0 = 1); 5000 elements reach several rows of the power tables."""
    c = curves[name]
    r = c.r
    n = 5000
    x = _enc([r - 1] * n)
    mont = lambda v: (v % r) * R256 % r   # noqa: E731
    got = c.Fr.batchApplyKey(x, mont(first).to_bytes(32, "little"), mont(inc).to_bytes(32, "little"))
    want = _enc([(r - 1) * first * pow(inc, i, r) % r for i in range(n)])
    assert np.array_equal(got, want), _first_diff(got, want, "batchApplyKey")


# ------------------------------------------------------------------------------------- Fr.fft / Fr.ifft in closed form
@functools.lru_cache(maxsize=None)
def _root(r: int, L: int) -> int:
    """Plain primitive 2^L-th root Fr.w[L]: w[s] = nqr^((r-1)/2^s) for the first non-residue nqr from 2, w[i] = w[i+1]^2."""
    nqr = 2
    while pow(nqr, (r - 1) // 2, r) != r - 1:
        nqr += 1
    s = ((r - 1) & -(r - 1)).bit_length() - 1
    return pow(pow(nqr, (r - 1) >> s, r), 1 << (s - L), r)


@functools.lru_cache(maxsize=4)
def _powers(r: int, L: int) -> tuple:
    w, t, out = _root(r, L), 1, []
    for _ in range(1 << L):
        out.append(t)
        t = t * w % r
    return tuple(out)


def _fft_expected(r, L, vec, inverse):
    """Closed forms of the transform of the raw residues (the transform is linear, so Montgomery form does not matter):
    X[j] = s * sum_k x[k] w^(+-jk), s = n^-1 for the inverse."""
    n = 1 << L
    s = pow(n, -1, r) if inverse else 1
    m = r - 1
    if vec == "all":
        return [(n * m * s) % r] + [0] * (n - 1)
    k = int(vec[4:]) if vec != "one@n-1" else n - 1
    pw = _powers(r, L)
    sign = -1 if inverse else 1
    return [m * s * pw[(sign * j * k) % n] % r for j in range(n)]


@pytest.mark.parametrize("name", CURVES)
@pytest.mark.parametrize("L", [1, 10, 11, 21])
def test_fr_fft_boundary_closed_form(curves, name, L):
    """L = 1: one pass; 10: the last single-pass size (NTT_DMAX); 11: the first two-pass size; 21: the first three-pass
    size.  Vectors: all entries r-1 (transform n(r-1) at 0, zero elsewhere) and r-1 at one index k in {0, 1, n-1}
    (transform (r-1) w^(jk))."""
    c = curves[name]
    r, n = c.r, 1 << L
    assert c.Fr.w[L] == (_root(r, L) * R256 % r).to_bytes(32, "little")
    for vec in ("all", "one@0", "one@1", "one@n-1"):
        x = [r - 1] * n if vec == "all" else [0] * n
        if vec != "all":
            x[{"one@0": 0, "one@1": 1, "one@n-1": n - 1}[vec]] = r - 1
        xb = _enc(x)
        for inverse in (False, True):
            got = (c.Fr.ifft if inverse else c.Fr.fft)(xb)
            want = _enc(_fft_expected(r, L, vec, inverse))
            assert np.array_equal(got, want), _first_diff(got, want, f"{'ifft' if inverse else 'fft'} L={L} {vec}")
