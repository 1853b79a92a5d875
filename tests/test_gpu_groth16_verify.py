"""GPU: sb_groth16_verify_batch and the device pairing behind it (sb_pairing_eval), on BN254 and BLS12-381.

Forged proofs: a verification key built from known scalars, alpha1 = a G1, beta2 = b G2, gamma2 = g G2, delta2 = d G2,
IC_i = k_i G1, makes (A, B, C) = (x G1, y G2, z G1) verify exactly when -xy + ab + (k_0 + sum s_i k_i) g + z d = 0 (mod r), so
every status of a large batch is known without a Python pairing.  Real proofs come from the device prover and are compared
with the oracle's groth16_verify, including on-curve points outside the r-subgroup.  The pairing itself is pinned against
Python big-integer tower arithmetic (tests/pairing_ref.py), the oracle's pairing raised to the documented c, bilinearity
and the reference's keypair known-answer test."""
import ctypes
import json
import os
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import oracle as O  # noqa: E402
from oracle import keypair as KP  # noqa: E402
from tests import pairing_ref as PR  # noqa: E402

BN, BLS = O.BN254, O.BLS12_381
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def curves():
    import snarkjs_b200
    cs = {BN: snarkjs_b200.getCurveFromName("bn128"), BLS: snarkjs_b200.getCurveFromName("bls12381")}
    yield cs
    for c in cs.values():
        c.terminate()


def _ptr(b):
    return ctypes.c_char_p(bytes(b)) if b else None


def pair_eval(c, op, records: bytes, out_elems: int, n: int):
    out = ctypes.create_string_buffer(max(1, n * out_elems * c.n8q))
    c.check(c.lib.sb_pairing_eval(c.handle, op, _ptr(records), n, out))
    return out.raw[:n * out_elems * c.n8q]


def verify_raw(c, vk: bytes, n_public: int, pubs: bytes, proofs: bytes, count: int):
    st = (ctypes.c_int32 * max(1, count))(*([-7] * max(1, count)))
    rc = c.lib.sb_groth16_verify_batch(c.handle, vk, len(vk), n_public, _ptr(pubs), _ptr(proofs), count, st)
    return rc, list(st)[:count]


# ---- forged keys and proofs --------------------------------------------------------------------------------------------
def g_bytes(cid, group, k):
    """k * generator, affine Montgomery bytes (all zero for k = 0 mod r)."""
    ci = O.CURVES[cid]
    k %= ci.r
    if k == 0:
        return bytes((2 if group == 1 else 4) * ci.n8q)
    gen = ci.g1_affine_bytes(ci.g1) if group == 1 else ci.g2_affine_bytes(ci.g2)
    return O.g_to_affine(cid, group, O.g_times(cid, group, O.g_from_affine(cid, group, gen), k.to_bytes(32, "little")))


class Forged:
    def __init__(self, cid, n_public, seed, zero_k=()):
        rng = random.Random(seed)
        self.cid, self.r, self.n = cid, O.CURVES[cid].r, n_public
        r = self.r
        self.a, self.b, self.g, self.d = (rng.randrange(1, r) for _ in range(4))
        self.k = [0 if i in zero_k else rng.randrange(1, r) for i in range(n_public + 1)]
        self.vk = (g_bytes(cid, 1, self.a) + g_bytes(cid, 2, self.b) + g_bytes(cid, 2, self.g) + g_bytes(cid, 2, self.d)
                   + b"".join(g_bytes(cid, 1, k) for k in self.k))

    def cp(self, s):
        return (self.k[0] + sum(si * ki for si, ki in zip(s, self.k[1:]))) % self.r

    def proof(self, s, x, y, ok=True):
        """(A, B, C) bytes for scalars x, y; C chosen so that the proof verifies, or is off by one G1 when not ok."""
        r = self.r
        z = (x * y - self.a * self.b - self.cp(s) * self.g) * pow(self.d, -1, r) % r
        return g_bytes(self.cid, 1, x) + g_bytes(self.cid, 2, y) + g_bytes(self.cid, 1, z if ok else z + 1)


def pub_bytes(s):
    return b"".join(v.to_bytes(32, "little") for v in s)


def tampered_indices(n):
    """The public indices whose tampering pool() tries: every one up to 300 inputs, else the ends and the middle."""
    return range(n) if n <= 300 else sorted({0, 1, n // 2, n - 2, n - 1})


def pool(f: Forged, m, seed):
    """m forged (publics, proof, expected status) triples: valid and invalid, infinities, boundary signals; then, on one
    valid proof with distinct signals, three edits per index of tampered_indices: s_j + 1 (status 1, or 0 where IC[j+1] is
    infinity), s_j = r (status 2) and s_j swapped with a neighbour (status 1: each signal must meet its own IC point)."""
    rng = random.Random(seed)
    r, out = f.r, []
    if f.n:
        s = [rng.randrange(r) for _ in range(f.n)]
        prf = f.proof(s, rng.randrange(1, r), rng.randrange(1, r))
        out.append((s, prf, 0))
        for j in tampered_indices(f.n):
            s1, s2 = list(s), list(s)
            s1[j] = (s[j] + 1) % r
            s2[j] = r
            out += [(s1, prf, 0 if f.cp(s1) == f.cp(s) else 1), (s2, prf, 2)]
            if f.n > 1:
                i = j + 1 if j + 1 < f.n else j - 1
                sw = list(s)
                sw[i], sw[j] = s[j], s[i]
                assert s[i] != s[j] and f.cp(sw) != f.cp(s)
                out.append((sw, prf, 1))
    for i in range(m):
        kind = i % 8
        s = [rng.choice([0, 1, r - 1, rng.randrange(r)]) for _ in range(f.n)]
        x, y = rng.randrange(1, r), rng.randrange(1, r)
        if kind == 1:
            x = 0                                                   # A = infinity
        elif kind == 2:
            y = 0                                                   # B = infinity
        elif kind == 3:                                             # C = infinity: xy = ab + cp g
            y = (f.a * f.b + f.cp(s) * f.g) * pow(x, -1, r) % r
        ok = kind not in (4, 5)
        prf = f.proof(s, x, y, ok)
        if kind == 5 and f.n:
            s2 = list(s)
            s2[0] = (s2[0] + 1) % r                                  # a perturbed signal
            out.append((s2, f.proof(s, x, y), 1 if f.k[1] else 0))
            continue
        out.append((s, prf, 0 if ok else 1))
    return out


def bad_point(cid, b: bytes, which: str) -> bytes:
    """A proof with A, B or C moved off its curve (y + 1)."""
    ci = O.CURVES[cid]
    n = ci.n8q
    off = {"A": n, "B": 4 * n, "C": 7 * n}[which]
    y = ci.fq_from_mont(b[off:off + n])
    return b[:off] + ci.fq_to_mont(y + 1) + b[off + n:]


def over_q(cid, b: bytes, which: str) -> bytes:
    """A proof whose A, B or C has its first coordinate replaced by q + 5 (not reduced, so not on the curve)."""
    ci = O.CURVES[cid]
    n = ci.n8q
    off = {"A": 0, "B": 2 * n, "C": 6 * n}[which]
    return b[:off] + (ci.q + 5).to_bytes(n, "little") + b[off + n:]


def run_items(c, f: Forged, items):
    pubs = b"".join(pub_bytes(s) for s, _p, _e in items)
    prfs = b"".join(p for _s, p, _e in items)
    rc, st = verify_raw(c, f.vk, f.n, pubs, prfs, len(items))
    assert rc == 0, c.lib.sb_last_error(c.handle)
    return st


CURVE_IDS = [BN, BLS]


@pytest.mark.parametrize("cid", CURVE_IDS, ids=["bn254", "bls12381"])
@pytest.mark.parametrize("n_public", [0, 1, 2, 7, 64, 255, 256, 257, 1000, 4096])
def test_forged_statuses(curves, cid, n_public):
    c = curves[cid]
    f = Forged(cid, n_public, seed=100 + n_public, zero_k=(0, 2) if n_public >= 2 else ())
    items = pool(f, 48, seed=n_public)
    # status 2 (a signal >= r) wins over an off-curve point; status 3 for every bad point
    s0 = [f.r - 1] * n_public
    good = f.proof(s0, 5, 7)
    if n_public:
        items.append(([f.r] + s0[1:], bad_point(cid, good, "A"), 2))
        items.append(([2 ** 256 - 1] + s0[1:], good, 2))
    for w in ("A", "B", "C"):
        items.append((s0, bad_point(cid, good, w), 3))
        items.append((s0, over_q(cid, good, w), 3))
    items.append((s0, good, 0))
    random.Random(7).shuffle(items)
    assert run_items(c, f, items) == [e for _s, _p, e in items]


@pytest.mark.parametrize("cid", CURVE_IDS, ids=["bn254", "bls12381"])
def test_forged_infinities(curves, cid):
    """IC[0] = infinity and all-zero signals give cpub = infinity; proofs with A, B or C at infinity verify."""
    c = curves[cid]
    f = Forged(cid, 3, seed=9, zero_k=(0,))
    r = f.r
    items = [([0, 0, 0], f.proof([0, 0, 0], 3, 4), 0), ([0, 0, 0], f.proof([0, 0, 0], 0, 4), 0),
             ([0, 0, 0], f.proof([0, 0, 0], 3, 0), 0), ([0, 0, 0], f.proof([0, 0, 0], 3, 4, ok=False), 1)]
    x = 11
    s = [1, 2, r - 1]
    y = (f.a * f.b + f.cp(s) * f.g) * pow(x, -1, r) % r
    items.append((s, f.proof(s, x, y), 0))
    assert f.proof(s, x, y)[-2 * c.n8q:] == bytes(2 * c.n8q)
    assert run_items(c, f, items) == [e for _s, _p, e in items]


@pytest.mark.parametrize("cid", CURVE_IDS, ids=["bn254", "bls12381"])
@pytest.mark.parametrize("count,cap", [(0, 0), (1, 0), (31, 32), (32, 32), (33, 32), (1000, 0), (1000, 97), (1 << 16, 0)])
def test_forged_batches(curves, cid, count, cap):
    """Mixed batches, every status in its own slot, across sub-batch boundaries (2^15 proofs by default, or cap)."""
    c = curves[cid]
    f = Forged(cid, 2, seed=21)
    base = pool(f, 200, seed=3)
    s0 = [1, 2]
    good = f.proof(s0, 5, 7)
    base += [([f.r, 1], good, 2), (s0, bad_point(cid, good, "B"), 3), (s0, over_q(cid, good, "C"), 3)]
    rng = random.Random(count)
    items = [base[rng.randrange(len(base))] for _ in range(count)]
    try:
        assert c.lib.sb_set_tuning(14, cap) == 0
        if count == 0:
            rc, st = verify_raw(c, f.vk, f.n, b"", b"", 0)
            assert rc == 0 and st == []
            return
        st = run_items(c, f, items)
    finally:
        c.lib.sb_set_tuning(14, 0)
    want = [e for _s, _p, e in items]
    assert st == want, [i for i in range(count) if st[i] != want[i]][:10]
    assert c.last_ms(0) > 0


# sb_groth16_verify_batch's sub-batch (api_verify.inl): min(count, VERIFY_CHUNK, VERIFY_BUDGET / per_proof)
VERIFY_CHUNK, VERIFY_BUDGET = 1 << 15, 512 << 20


@pytest.mark.parametrize("cid", CURVE_IDS, ids=["bn254", "bls12381"])
def test_forged_budget_sub_batches(curves, cid):
    """16384 public inputs: the 512 MiB budget, not the 2^15 chunk or a tuning cap, splits 2 chunk + 1 proofs into three
    sub-batches (seen in the launch count), and the proofs on both sides of each split get their own statuses."""
    c = curves[cid]
    n8, n = c.n8q, 16384
    per_proof = 8 * n8 + n * (32 + 4 * n8) + 4           # proof, publics, their XYZZ terms, status
    chunk = VERIFY_BUDGET // per_proof
    count = 2 * chunk + 1
    assert chunk < count < VERIFY_CHUNK
    f = Forged(cid, n, seed=41)
    rng = random.Random(41)
    valid = []
    for _ in range(4):
        s = [rng.randrange(f.r) for _ in range(n)]
        valid.append((s, f.proof(s, rng.randrange(1, f.r), rng.randrange(1, f.r)), 0))
    s, prf, _ = valid[0]
    edits = {chunk - 1: (n - 1, f.r, 2), chunk: (n - 1, (s[n - 1] + 1) % f.r, 1), 2 * chunk - 1: (0, (s[0] + 1) % f.r, 1),
             2 * chunk: (0, f.r, 2)}
    items = [valid[rng.randrange(4)] for _ in range(count)]
    for k, (j, v, want) in edits.items():
        items[k] = (s[:j] + [v] + s[j + 1:], prf, want)
    lib = c.lib
    assert lib.sb_set_tuning(14, 0) == 0
    before = lib.sb_launch_count(c.handle)
    st = run_items(c, f, items)
    assert lib.sb_launch_count(c.handle) - before == 1 + 3 * 2     # prepare, then terms and verify per sub-batch
    assert [st[k] for k in sorted(edits)] == [edits[k][2] for k in sorted(edits)]
    assert st == [e for _s, _p, e in items]


@pytest.mark.parametrize("cid", CURVE_IDS, ids=["bn254", "bls12381"])
def test_argument_errors(curves, cid):
    c = curves[cid]
    f = Forged(cid, 1, seed=5)
    pr = f.proof([3], 5, 7)
    rc, _ = verify_raw(c, f.vk[:-1], 1, pub_bytes([3]), pr, 1)
    assert rc == -1 and b"vk_len" in c.lib.sb_last_error(c.handle)
    rc, _ = verify_raw(c, f.vk, 2, pub_bytes([3]), pr, 1)
    assert rc == -1
    bad_vk = bad_point(cid, f.vk[:8 * c.n8q], "A") + f.vk[8 * c.n8q:]          # alpha1's y + 1
    rc, _ = verify_raw(c, bad_vk, 1, pub_bytes([3]), pr, 1)
    assert rc == -1 and b"not on its curve" in c.lib.sb_last_error(c.handle)
    assert c.lib.sb_groth16_verify_batch(c.handle, f.vk, len(f.vk), 1, None, pr, 1, None) == -1
    assert c.lib.sb_pairing_eval(c.handle, 8, None, 0, None) == -1
    assert c.lib.sb_pairing_eval(c.handle, -1, None, 0, None) == -1


# ---- real proofs ------------------------------------------------------------------------------------------------------
def _real(curves, label, n_proofs=3):
    from snarkjs_b200 import groth16
    from tests import r1cs_shapes as S
    circ = S.case(label)
    c = curves[circ.curve]
    zkey = S.case_zkey(label)
    pk = groth16.ProvingKey(zkey, curve=c)
    try:
        ci = O.CURVES[circ.curve]
        rs = [(ci.fr_to_mont(77 + i), ci.fr_to_mont(99 + 3 * i)) for i in range(n_proofs)]
        res = groth16.prove_batch(pk, [circ.wtns()] * n_proofs, rs)
    finally:
        pk.release()
    return c, zkey, res


@pytest.mark.parametrize("label", ["public2", "public17", "bits", "tiny7", "bls_public17", "bls_tiny49"])
def test_real_proofs(curves, label):
    from snarkjs_b200 import groth16
    c, zkey, res = _real(curves, label)
    vk = groth16.verification_key(zkey)
    r = c.r
    items = [(pub, proof) for proof, pub in res]
    want = [True] * len(items)
    if vk["nPublic"]:
        p0, pub0 = res[0]
        items.append(([str(int(pub0[0]) + r)] + pub0[1:], p0))          # aliased signal: status 2
        want.append(False)
        items.append(([str((int(pub0[0]) + 1) % r)] + pub0[1:], p0))    # another statement
        want.append(False)
    swapped = dict(res[0][0], pi_a=res[0][0]["pi_c"], pi_c=res[0][0]["pi_a"])
    items.append((res[0][1], swapped))
    want.append(False)
    assert groth16.verify_batch(vk, items, curve=c) == want
    assert groth16.verify(vk, res[0][1], res[0][0], curve=c)


def test_golden_key_proof(curves):
    from snarkjs_b200 import groth16
    g = np.load(os.path.join(ROOT, "tests", "golden", "groth16_case.npz"))
    c = curves[BN]
    ci = O.CURVES[BN]
    pk = groth16.ProvingKey(g["zkey"].tobytes(), curve=c)
    try:
        proof, pub = groth16.prove(pk, g["wtns"].tobytes(), ci.fr_to_mont(11), ci.fr_to_mont(13))
    finally:
        pk.release()
    vk = groth16.verification_key(g["zkey"].tobytes())

    class Log:
        def __init__(self): self.lines = []
        def error(self, m): self.lines.append(m)
        def info(self, m): self.lines.append(m)
    lg = Log()
    assert groth16.verify(vk, pub, proof, logger=lg, curve=c) and lg.lines == ["OK!"]
    if pub:
        assert not groth16.verify(vk, [str(c.r)] + pub[1:], proof, logger=lg, curve=c)
        assert lg.lines[-1] == "Public inputs are not valid."
    bad = dict(proof, pi_a=[proof["pi_a"][0], str(int(proof["pi_a"][1]) + 1), "1"])
    assert not groth16.verify(vk, pub, bad, logger=lg, curve=c) and lg.lines[-1] == "Proof commitments are not valid."
    bad = dict(proof, pi_c=proof["pi_a"])
    assert not groth16.verify(vk, pub, bad, logger=lg, curve=c) and lg.lines[-1] == "Invalid proof"


def test_bls_structured_setup(curves):
    """A BLS12-381 key from oracle/synth_setup.py's structured setup: its proofs verify."""
    from snarkjs_b200 import groth16
    from oracle import synth_setup as SS
    c = curves[BLS]
    from oracle.plonk import wtns_bytes
    r1cs, wit = SS.chain_r1cs(BLS, 60)
    zkey = O.zkey_new(r1cs, SS.prepared_ptau(BLS, 64, tau=123457, alpha=1111, beta=2222))
    wt = wtns_bytes(wit, O.P_BLS_R)
    ci = O.CURVES[BLS]
    res = groth16.prove_batch(zkey, [wt, wt], [(ci.fr_to_mont(5), ci.fr_to_mont(6)), (ci.fr_to_mont(7), ci.fr_to_mont(8))])
    vk = groth16.verification_key(zkey)
    assert groth16.verify_batch(vk, [(pub, proof) for proof, pub in res], curve=c) == [True, True]


def _fq2_sqrt(a, q):
    """square root in Fq[u]/(u^2 + 1), q = 3 mod 4 (None if a is not a square)."""
    mul = lambda x, y: ((x[0] * y[0] - x[1] * y[1]) % q, (x[0] * y[1] + x[1] * y[0]) % q)

    def pw(x, e):
        r = (1, 0)
        while e:
            if e & 1:
                r = mul(r, x)
            x = mul(x, x)
            e >>= 1
        return r
    a1 = pw(a, (q - 3) // 4)
    alpha = mul(mul(a1, a1), a)
    x0 = mul(a1, a)
    if alpha == (q - 1, 0):
        x = mul((0, 1), x0)
    else:
        x = mul(pw(((1 + alpha[0]) % q, alpha[1]), (q - 1) // 2), x0)
    return x if mul(x, x) == (a[0] % q, a[1] % q) else None


def off_subgroup_g2(cid, rng):
    q = PR.Q[cid]
    b = PR.twist_b(cid)
    while True:
        x = (rng.randrange(q), rng.randrange(q))
        x3 = ((x[0] ** 3 - 3 * x[0] * x[1] ** 2) % q, (3 * x[0] ** 2 * x[1] - x[1] ** 3) % q)
        y = _fq2_sqrt(((x3[0] + b[0]) % q, (x3[1] + b[1]) % q), q)
        if y is not None:
            return (x, y)


def off_subgroup_g1(rng):
    q = O.P_BLS_Q
    while True:
        x = rng.randrange(q)
        y = pow((x ** 3 + 4) % q, (q + 1) // 4, q)
        if (y * y - x ** 3 - 4) % q == 0:
            return (x, y)


@pytest.mark.parametrize("label", ["public2", "bls_public17"])
def test_agrees_with_oracle(curves, label):
    """20 cases per curve through groth16.verify_batch and oracle.groth16_verify, with G2 points outside the subgroup on both
    curves and G1 points outside it on BLS12-381."""
    from snarkjs_b200 import groth16
    c, zkey, res = _real(curves, label, n_proofs=2)
    cid = BN if c.n8q == 32 else BLS
    ci = O.CURVES[cid]
    vk = groth16.verification_key(zkey)
    ovk = O.zkey_vk(zkey)
    rng = random.Random(len(label))
    o1 = lambda p: ["0", "1", "0"] if p is None else [str(p[0]), str(p[1]), "1"]
    o2 = lambda p: [[str(p[0][0]), str(p[0][1])], [str(p[1][0]), str(p[1][1])], ["1", "0"]]
    cases = []
    for i in range(20):
        proof, pub = res[i % 2]
        proof = dict(proof)
        kind = i % 5
        if kind == 1:
            proof["pi_b"] = o2(off_subgroup_g2(cid, rng))
        elif kind == 2 and cid == BLS:
            proof["pi_a"] = o1(off_subgroup_g1(rng))
        elif kind == 2:
            proof["pi_a"] = o1(PR.g_mul(cid, 1, ci.g1, rng.randrange(1, ci.r)))
        elif kind == 3:
            pub = [str((int(pub[0]) + i) % ci.r)] + pub[1:]
        elif kind == 4 and cid == BLS:
            proof["pi_c"] = o1(off_subgroup_g1(rng))
        cases.append((pub, proof))
    got = groth16.verify_batch(vk, cases, curve=c)
    want = [O.groth16_verify(ovk, [int(x) for x in pub], proof) for pub, proof in cases]
    assert got == want
    assert any(want) and not all(want)


# ---- the pairing ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("cid", CURVE_IDS, ids=["bn254", "bls12381"])
def test_tower_ops(curves, cid):
    c = curves[cid]
    rng = random.Random(31 + cid)
    fl = lambda t: PR.to_flat(cid, t)
    n = 6
    A = [PR.rand_fq12(cid, rng) for _ in range(n)]
    B = [PR.rand_fq12(cid, rng) for _ in range(n)]
    A[0] = [0] * 12
    A[1] = list(PR.from_flat(cid, PR.ONE))
    A[2] = [PR.Q[cid] - 1] * 12
    cyc = [PR.from_flat(cid, PR.easy_part(cid, fl(a))) for a in A[1:]]
    unpack = lambda b, k: [PR.unpack(cid, b[i * 12 * c.n8q:(i + 1) * 12 * c.n8q]) for i in range(k)]
    got = unpack(pair_eval(c, 0, b"".join(PR.pack(cid, a + b) for a, b in zip(A, B)), 12, n), n)
    assert [fl(g) for g in got] == [PR.fmul(cid, fl(a), fl(b)) for a, b in zip(A, B)]
    got = unpack(pair_eval(c, 1, b"".join(PR.pack(cid, a) for a in A), 12, n), n)
    assert [fl(g) for g in got] == [PR.fmul(cid, fl(a), fl(a)) for a in A]
    got = unpack(pair_eval(c, 2, b"".join(PR.pack(cid, a) for a in cyc), 12, len(cyc)), len(cyc))
    assert [fl(g) for g in got] == [PR.fmul(cid, fl(a), fl(a)) for a in cyc]
    got = unpack(pair_eval(c, 3, b"".join(PR.pack(cid, a) for a in A[1:]), 12, n - 1), n - 1)
    assert all(PR.fmul(cid, fl(g), fl(a)) == PR.ONE for g, a in zip(got, A[1:]))
    got = unpack(pair_eval(c, 4, b"".join(PR.pack(cid, a) for a in A[:3]), 36, 3), 9)
    q = PR.Q[cid]
    assert [fl(g) for g in got] == [PR.fpow(cid, fl(a), q ** k) for a in A[:3] for k in (1, 2, 3)]
    got = unpack(pair_eval(c, 6, b"".join(PR.pack(cid, a) for a in A[1:3]), 12, 2), 2)
    assert [fl(g) for g in got] == [PR.final_exp_ref(cid, fl(a)) for a in A[1:3]]


def _e(c, cid, pts):
    raw = pair_eval(c, 7, b"".join(PR.pack(cid, PR.pt_vals(p, q)) for p, q in pts), 12, len(pts))
    return [PR.to_flat(cid, PR.unpack(cid, raw[i * 12 * c.n8q:(i + 1) * 12 * c.n8q])) for i in range(len(pts))]


@pytest.mark.parametrize("cid", CURVE_IDS, ids=["bn254", "bls12381"])
def test_pairing_values(curves, cid):
    """e(P, Q) is the oracle's pairing raised to c (conjugated on BLS12-381); 5 then 6 is 7; bilinearity; infinity gives 1."""
    c = curves[cid]
    ci = O.CURVES[cid]
    rng = random.Random(cid)
    a, b = rng.randrange(1, ci.r), rng.randrange(1, ci.r)
    P, Q2 = PR.g_mul(cid, 1, ci.g1, a), PR.g_mul(cid, 2, ci.g2, b)
    e = _e(c, cid, [(ci.g1, ci.g2), (P, Q2), (PR.g_mul(cid, 1, ci.g1, a * b), ci.g2), (None, ci.g2), (ci.g1, None)])
    assert e[0] == PR.pairing_ref(cid, ci.g1, ci.g2)
    assert e[1] == PR.pairing_ref(cid, P, Q2)
    assert e[1] == e[2] and e[0] != PR.ONE
    assert e[3] == PR.ONE and e[4] == PR.ONE
    ml = pair_eval(c, 5, PR.pack(cid, PR.pt_vals(P, Q2)), 12, 1)
    assert PR.to_flat(cid, PR.unpack(cid, pair_eval(c, 6, ml, 12, 1))) == e[1]


def test_keypair_kat(curves):
    """The reference's keypair known-answer test (test/keypar_test.js): e(g1_sx, g2_sp) == e(g1_s, g2_spx) on the device."""
    kat = json.load(open(os.path.join(ROOT, "tests", "golden", "keypair_kat.json")))
    c = curves[BN]
    challenge = bytes.fromhex(kat["challenge_hex"])
    for case in kat["cases"]:
        s = (int(case["g1_s"][0], 16), int(case["g1_s"][1], 16))
        sx = (int(case["g1_sx"][0], 16), int(case["g1_sx"][1], 16))
        spx = tuple((int(v[0], 16), int(v[1], 16)) for v in case["g2_spx"])
        sp = KP.get_g2sp(case["personalization"], challenge, s, sx)
        e = _e(c, BN, [(sx, sp), (s, spx)])
        assert e[0] == e[1], case["name"]
