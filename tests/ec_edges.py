"""Records and exact expected results for the device point formulas (csrc/ec.cuh: XYZZ add_affine, add_i, add, dbl and
dbl_affine) run through the test hook sb_field_eval, in Python integers only: no GPU and no oracle.

Groups are named by their base field as in sb_field_eval: 0 BN254 G1, 2 BLS12-381 G1, 4 BN254 G2, 5 BLS12-381 G2, all on
y^2 = x^3 + b with a = 0 (b = 3, b = 4; the G2 twists b' = 3/(9+u) and b' = 4(1+u) over Fq2 = Fq[u]/(u^2+1)).  On-curve
points are multiples of the standard generators, held in representatives XYZZ(P, l) = (x l^2, y l^3, l^2, l^3).

Every record has two expectations:
  (a) bytes: the formulas of ec.cuh restated on integers, with the same special cases in the same order and infinity
      written as all zeros.  Every field result is canonical, so the device must give exactly these bytes whichever multiply
      (mul, mul2_i, lazy Karatsuba) it uses; add_i and add share one expectation.
  (b) meaning, for the on-curve records only and independent of the formulas: the affine result (x/zz, y/zzz) is the
      textbook sum or double, zz == 0 exactly when that is infinity, zz^3 == zzz^2, and the result lies on the curve.

Record classes (the two-operand ones as acc + q; add_affine's q is affine and never infinity, which k_accumulate
guarantees by dropping (0, 0) bases):
  inf+inf, inf+Q, P+inf   infinity on either side (inf+q for add_affine: the result is (qx, qy, 1, 1))
  P+P same/diff rep       Pp == 0 and R == 0 through the cross-multiplied compare: the doubling branch (l = -1 included)
  P-P same/diff rep       Pp == 0, R != 0: cancellation to infinity
  P+phi(P)                phi(x, y) = (beta x, y), beta a cube root of unity in Fq: Pp != 0 with R == 0, the generic
                          formula at a zero operand, which no other class reaches
  P-phi(P), P+2P, P-2P    the generic formula at related operands
  rep                     representatives l in {1, -1, R mod p, R^-1 mod p} (and u on G2)
  random                  N_RANDOM seeded pairs (points for the doublings) in random representatives
  inf                     dbl and dbl_affine of infinity (dbl_affine's (0, 0) goes through its y == 0 guard)
  off y=0                 y = 0 with zz != 0: the doublings' y == 0 guard (directly, or from the doubling branch of an
                          addition).  No point of these groups has y = 0, so only these records see the guard.
  off const               every coordinate, representative included, from {0, 1, p-1, R mod p} as raw Montgomery words
The off-curve classes are checked against (a) only.  Every class with a target branch asserts that each of its records
takes it, so a broken generator cannot quietly weaken the tests that use it."""
from __future__ import annotations

import functools
import random

from tests.field_edges import FE_NOPS, FIELDS, _F

EC_OPS = {"add_affine": 16, "add_i": 17, "add": 18, "dbl": 19, "dbl_affine": 20}
OP_NAMES = {v: k for k, v in EC_OPS.items()}
assert max(OP_NAMES) + 1 == FE_NOPS
GROUPS = {0: "BN254 G1", 2: "BLS12-381 G1", 4: "BN254 G2", 5: "BLS12-381 G2"}
COORDS = ("x", "y", "zz", "zzz")
N_RANDOM = 1000
N_CONST = 256
N_CLASS = 8                    # records per crafted on-curve class

# standard generators (EIP-197 for BN254; the IETF pairing-friendly-curves draft for BLS12-381), affine, plain integers
_GEN = {
    0: (1, 2),
    2: (0x17f1d3a73197d7942695638c4fa9ac0fc3688c4f9774b905a14e3a3f171bac586c55e83ff97a1aeffb3af00adb22c6bb,
        0x08b3f481e3aaa0f1a09e30ed741d8ae4fcf5e095d5d00af600db18cb2c04b3edd03cc744a2888ae40caa232946c5e7e1),
    4: ((10857046999023057135944570762232829481370756359578518086990519993285655852781,
         11559732032986387107991004021392285783925812861821192530917403151452391805634),
        (8495653923123431417604973247489272438418190587263600148770280649306958101930,
         4082367875863433681332203403145435568316851327593401208105741076214120093531)),
    5: ((0x024aa2b2f08f0a91260805272dc51051c6e47ad4fa403b02b4510b647ae3d1770bac0326a805bbefd48056c8c121bdb8,
         0x13e02b6052719f607dacd3a088274f65596bd0d09920b61ab5da61bbdc7f5049334cf11213945d57e5ac7d055d042b7e),
        (0x0ce5d527727d6e118cc9cdc6da2e351aadfd9baa8cbdd3a76d429a695160d12c923ac9cc3baca289e193548608b82801,
         0x0606c4a02ea734cc32acd2b02bc28b99cb3e287e85a763af267492ab572e99ab3f370d275cec1da1aaa9075ff05f79be)),
}
_ORDER = {  # r, the order of the generators
    0: 0x30644e72e131a029b85045b68181585d2833e84879b9709143e1f593f0000001,
    2: 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001,
}
_ORDER[4], _ORDER[5] = _ORDER[0], _ORDER[2]


# ------------------------------------------------------------------------------------- fields on plain values
class _Fq:
    """Fq on plain integers; raw() / plain() convert to and from the Montgomery residues the kernels hold."""
    deg = 1

    def __init__(self, p: int, limbs: int):
        self.p, self.F = p, _F(p, limbs)
        self.zero, self.one = 0, 1

    def add(self, a, b): return (a + b) % self.p
    def sub(self, a, b): return (a - b) % self.p
    def neg(self, a): return -a % self.p
    def dbl(self, a): return 2 * a % self.p
    def mul(self, a, b): return a * b % self.p
    def sqr(self, a): return a * a % self.p
    def inv(self, a): return pow(a, -1, self.p)
    def is_zero(self, a): return a == 0
    def scale(self, a, k): return a * k % self.p           # by an Fq constant
    def embed(self, k): return k % self.p
    def rand(self, rng): return rng.randrange(self.p)
    def raw(self, a): return (a * self.F.R % self.p,)
    def plain(self, w): return w[0] * self.F.Ri % self.p
    def hex(self, a): return hex(self.raw(a)[0])


class _Fq2(_Fq):
    """Fq2 = Fq[u]/(u^2 + 1), elements (c0, c1)."""
    deg = 2

    def __init__(self, p: int, limbs: int):
        super().__init__(p, limbs)
        self.zero, self.one = (0, 0), (1, 0)

    def add(self, a, b): return ((a[0] + b[0]) % self.p, (a[1] + b[1]) % self.p)
    def sub(self, a, b): return ((a[0] - b[0]) % self.p, (a[1] - b[1]) % self.p)
    def neg(self, a): return (-a[0] % self.p, -a[1] % self.p)
    def dbl(self, a): return (2 * a[0] % self.p, 2 * a[1] % self.p)
    def mul(self, a, b): return ((a[0] * b[0] - a[1] * b[1]) % self.p, (a[0] * b[1] + a[1] * b[0]) % self.p)
    def sqr(self, a): return self.mul(a, a)

    def inv(self, a):
        n = pow((a[0] * a[0] + a[1] * a[1]) % self.p, -1, self.p)
        return (a[0] * n % self.p, -a[1] * n % self.p)

    def is_zero(self, a): return a == (0, 0)
    def scale(self, a, k): return (a[0] * k % self.p, a[1] * k % self.p)
    def embed(self, k): return (k % self.p, 0)
    def rand(self, rng): return (rng.randrange(self.p), rng.randrange(self.p))
    def raw(self, a): return (a[0] * self.F.R % self.p, a[1] * self.F.R % self.p)
    def plain(self, w): return (w[0] * self.F.Ri % self.p, w[1] * self.F.Ri % self.p)
    def hex(self, a): return "(" + ", ".join(hex(v) for v in self.raw(a)) + ")"


class _Curve:
    def __init__(self, group: int):
        _, p, limbs = FIELDS[group]
        self.K = K = (_Fq2 if group >= 4 else _Fq)(p, limbs)
        self.words = K.deg * limbs                       # 32-bit words per coordinate
        if group == 0:
            self.b = 3
        elif group == 2:
            self.b = 4
        elif group == 4:
            self.b = K.mul((3, 0), K.inv((9, 1)))        # 3 / (9 + u)
        else:
            self.b = (4, 4)                              # 4 (1 + u)
        self.g = _GEN[group]
        self.r = _ORDER[group]
        g = 2                                            # beta: a non-trivial cube root of unity in Fq (q = 1 mod 3)
        while pow(g, (p - 1) // 3, p) == 1:
            g += 1
        self.beta = pow(g, (p - 1) // 3, p)
        assert (p - 1) % 3 == 0 and self.beta != 1 and pow(self.beta, 3, p) == 1
        assert self.on_curve(self.g)

    # --- affine points: (x, y), infinity None
    def on_curve(self, P) -> bool:
        K = self.K
        return P is None or K.sqr(P[1]) == K.add(K.mul(K.sqr(P[0]), P[0]), self.b)

    def neg(self, P):
        return None if P is None else (P[0], self.K.neg(P[1]))

    def phi(self, P):
        return (self.K.scale(P[0], self.beta), P[1])

    def add(self, P, Q):
        """Textbook affine addition (chord and tangent)."""
        K = self.K
        if P is None:
            return Q
        if Q is None:
            return P
        (x1, y1), (x2, y2) = P, Q
        if x1 == x2:
            if y1 == K.neg(y2):
                return None
            lam = K.mul(K.scale(K.sqr(x1), 3), K.inv(K.dbl(y1)))
        else:
            lam = K.mul(K.sub(y2, y1), K.inv(K.sub(x2, x1)))
        x3 = K.sub(K.sub(K.sqr(lam), x1), x2)
        return (x3, K.sub(K.mul(lam, K.sub(x1, x3)), y1))

    def smul(self, k: int, P):
        acc = None
        for bit in bin(k)[2:]:
            acc = self.add(acc, acc)
            if bit == "1":
                acc = self.add(acc, P)
        return acc

    # --- XYZZ
    def inf(self):
        z = self.K.zero
        return (z, z, z, z)

    def xyzz(self, P, lam):
        K = self.K
        if P is None:
            return self.inf()
        l2 = K.sqr(lam)
        l3 = K.mul(l2, lam)
        return (K.mul(P[0], l2), K.mul(P[1], l3), l2, l3)

    def affine(self, p):
        K = self.K
        if K.is_zero(p[2]):
            return None
        return (K.mul(p[0], K.inv(p[2])), K.mul(p[1], K.inv(p[3])))


@functools.lru_cache(maxsize=None)
def curve(group: int) -> _Curve:
    return _Curve(group)


# ------------------------------------------------------------------------------------- (a): ec.cuh restated
# Each returns (result, branch); the branch names the special case the formula took.
def ref_dbl_affine(C, px, py):
    K = C.K
    if K.is_zero(py):
        return C.inf(), "y=0"
    U = K.dbl(py)
    V = K.sqr(U)
    W = K.mul(U, V)
    S = K.mul(px, V)
    M = K.sqr(px)
    M = K.add(K.dbl(M), M)
    x = K.sub(K.sqr(M), K.dbl(S))
    y = K.sub(K.mul(M, K.sub(S, x)), K.mul(W, py))
    return (x, y, V, W), "formula"


def ref_dbl(C, p):
    K = C.K
    x, y, zz, zzz = p
    if K.is_zero(zz):
        return C.inf(), "inf"
    if K.is_zero(y):
        return C.inf(), "y=0"
    U = K.dbl(y)
    V = K.sqr(U)
    W = K.mul(U, V)
    S = K.mul(x, V)
    M = K.sqr(x)
    M = K.add(K.dbl(M), M)
    X3 = K.sub(K.sqr(M), K.dbl(S))
    Y3 = K.sub(K.mul(M, K.sub(S, X3)), K.mul(W, y))
    return (X3, Y3, K.mul(V, zz), K.mul(W, zzz)), "formula"


def ref_add_affine(C, acc, qx, qy):
    K = C.K
    x, y, zz, zzz = acc
    if K.is_zero(zz):
        return (qx, qy, K.one, K.one), "acc=inf"
    U2, S2 = K.mul(qx, zz), K.mul(qy, zzz)
    Pp, R = K.sub(U2, x), K.sub(S2, y)
    if K.is_zero(Pp):
        if K.is_zero(R):
            r, b = ref_dbl_affine(C, qx, qy)
            return r, "dbl" if b == "formula" else "dbl y=0"
        return C.inf(), "cancel"
    PP = K.sqr(Pp)
    PPP = K.mul(Pp, PP)
    Q = K.mul(x, PP)
    X3 = K.sub(K.sub(K.sqr(R), PPP), K.dbl(Q))
    Y3 = K.sub(K.mul(R, K.sub(Q, X3)), K.mul(y, PPP))
    return (X3, Y3, K.mul(zz, PP), K.mul(zzz, PPP)), "generic R=0" if K.is_zero(R) else "generic"


def ref_add(C, acc, q):
    """add-2008-s as XYZZ::add and XYZZ::add_i compute it."""
    K = C.K
    if K.is_zero(q[2]):
        return acc, "q=inf"
    if K.is_zero(acc[2]):
        return q, "acc=inf"
    x, y, zz, zzz = acc
    U1, U2 = K.mul(x, q[2]), K.mul(q[0], zz)
    S1, S2 = K.mul(y, q[3]), K.mul(q[1], zzz)
    Pp, R = K.sub(U2, U1), K.sub(S2, S1)
    if K.is_zero(Pp):
        if K.is_zero(R):
            r, b = ref_dbl(C, acc)
            return r, "dbl" if b == "formula" else "dbl y=0"
        return C.inf(), "cancel"
    PP = K.sqr(Pp)
    PPP = K.mul(Pp, PP)
    Q = K.mul(U1, PP)
    X3 = K.sub(K.sub(K.sqr(R), PPP), K.dbl(Q))
    Y3 = K.sub(K.mul(R, K.sub(Q, X3)), K.mul(S1, PPP))
    return ((X3, Y3, K.mul(K.mul(zz, q[2]), PP), K.mul(K.mul(zzz, q[3]), PPP)),
            "generic R=0" if K.is_zero(R) else "generic")


def reference(C, op: int, args):
    """(a) for one record: (result XYZZ, branch)."""
    name = OP_NAMES[op]
    if name == "add_affine":
        return ref_add_affine(C, args[:4], args[4], args[5])
    if name in ("add_i", "add"):
        return ref_add(C, args[:4], args[4:])
    if name == "dbl":
        return ref_dbl(C, args)
    return ref_dbl_affine(C, args[0], args[1])


# ------------------------------------------------------------------------------------- (b): meaning
def operands(C, op: int, args) -> list:
    """The affine points a record's operands stand for (None: infinity): [acc, q] for the additions, [p] for the doublings."""
    K = C.K
    name = OP_NAMES[op]
    if name == "add_affine":
        return [C.affine(args[:4]), (args[4], args[5])]
    if name in ("add_i", "add"):
        return [C.affine(args[:4]), C.affine(args[4:])]
    if name == "dbl":
        return [C.affine(args)]
    return [None if K.is_zero(args[0]) and K.is_zero(args[1]) else (args[0], args[1])]


def meaning(C, op: int, args, res) -> str | None:
    """None if the XYZZ result `res` means what the textbook group law gives for the on-curve operands `args`, else why not."""
    K = C.K
    ins = operands(C, op, args)
    want = C.add(ins[0], ins[-1])
    x, y, zz, zzz = res
    if K.mul(K.sqr(zz), zz) != K.sqr(zzz):
        return "zz^3 != zzz^2"
    if K.is_zero(zz) != (want is None):
        return "zz == 0 but the sum is a point" if K.is_zero(zz) else "zz != 0 but the sum is infinity"
    if want is None:
        return None
    got = C.affine(res)
    if not C.on_curve(got):
        return "the affine result is not on the curve"
    if got != want:
        return f"affine result ({K.hex(got[0])}, {K.hex(got[1])}) expected ({K.hex(want[0])}, {K.hex(want[1])})"
    return None


# ------------------------------------------------------------------------------------- records
@functools.lru_cache(maxsize=None)
def _points(group: int, n: int) -> tuple:
    """n on-curve points s*G, (s+d)*G, (s+2d)*G, ... for seeded s, d."""
    C = curve(group)
    rng = random.Random(7919 * group + 1)
    P = C.smul(rng.randrange(1, C.r), C.g)
    D = C.smul(rng.randrange(1, C.r), C.g)
    out = []
    for _ in range(n):
        out.append(P)
        P = C.add(P, D)
    assert all(Q is not None for Q in out)
    return tuple(out)


def all_sets() -> list[tuple[int, int]]:
    return [(g, o) for g in GROUPS for o in EC_OPS.values()]


@functools.lru_cache(maxsize=None)
def records(group: int, op: int) -> tuple:
    """((label, operands, expected XYZZ, on_curve, branch), ...) for (group, op), deterministic; operands and results are
    plain field elements (Montgomery encoding happens in pack())."""
    if group not in GROUPS or op not in OP_NAMES:
        raise ValueError(f"op {op} is not a point op on group {group}")
    C = curve(group)
    K = C.K
    name = OP_NAMES[op]
    rng = random.Random(100 * group + op)
    pts = _points(group, 4 * N_CLASS + 2 * N_RANDOM)
    pool = pts[4 * N_CLASS:]
    recs = []
    targets = {}

    def lam():
        while True:
            v = K.rand(rng)
            if not K.is_zero(v):
                return v

    def add(label, args, on_curve=True, target=None):
        args = tuple(args)
        res, branch = reference(C, op, args)
        recs.append((label, args, res, on_curve, branch))
        if target is not None:
            targets[label] = target

    minus1 = K.neg(K.one)
    R = K.F.R % K.p
    specials = [K.one, minus1, K.embed(R), K.embed(pow(R, -1, K.p))] + ([(0, 1)] if K.deg == 2 else [])
    cls = [pts[i * N_CLASS:(i + 1) * N_CLASS] for i in range(4)]     # distinct points per class family

    if name in ("add_affine", "add_i", "add"):
        aff = name == "add_affine"

        def pair(label, P, Q, l1, l2, target=None, on_curve=True):
            # acc = XYZZ(P, l1); q = affine Q, or XYZZ(Q, l2)
            qa = (Q[0], Q[1]) if aff else C.xyzz(Q, l2)
            add(label, C.xyzz(P, l1) + tuple(qa), on_curve, target)

        if aff:
            for P in cls[0]:
                add("inf+q", C.inf() + P, target="acc=inf")
        else:
            add("inf+inf", C.inf() + C.inf(), target="q=inf")
            for P in cls[0]:
                add("inf+Q", C.inf() + C.xyzz(P, lam()), target="acc=inf")
                add("P+inf", C.xyzz(P, lam()) + C.inf(), target="q=inf")
        diff = [(minus1, K.one), (K.one, minus1), (minus1, lam()), (lam(), minus1)]     # l = -1 on either side
        for i, P in enumerate(cls[1]):
            l1 = K.one if aff else lam()            # add_affine's q is affine: representative 1
            pair("P+P same rep", P, P, l1, l1, "dbl")
            pair("P-P same rep", P, C.neg(P), l1, l1, "cancel")
            if aff:
                l1, l2 = (minus1 if i < 4 else lam()), K.one
            else:
                l1, l2 = diff[i] if i < 4 else (lam(), lam())
            pair("P+P diff rep", P, P, l1, l2, "dbl")
            pair("P-P diff rep", P, C.neg(P), l1, l2, "cancel")
        for P in cls[2]:
            pair("P+phi(P)", P, C.phi(P), lam(), lam(), "generic R=0")
            pair("P-phi(P)", P, C.neg(C.phi(P)), lam(), lam(), "generic")
            P2 = C.add(P, P)
            pair("P+2P", P, P2, lam(), lam(), "generic")
            pair("P-2P", P, C.neg(P2), lam(), lam(), "generic")
        for l1 in specials:
            for l2 in specials:
                pair("rep", rng.choice(cls[3]), rng.choice(pool), l1, l2)
        for _ in range(N_RANDOM):
            pair("random", rng.choice(pool), rng.choice(pool), lam(), lam())
        for _ in range(N_CLASS):                  # off-curve y = 0, acc and q the same: the doubling branch's y guard
            x, zz, zzz = lam(), lam(), lam()
            if aff:
                add("off y=0", (K.mul(x, zz), K.zero, zz, zzz, x, K.zero), False, "dbl y=0")
            else:
                add("off y=0", (x, K.zero, zz, zzz, x, K.zero, zz, zzz), False, "dbl y=0")
        nco = 6 if aff else 8
    elif name == "dbl":
        add("inf", C.inf(), target="inf")
        for P in cls[0]:
            add("-P", C.xyzz(P, minus1), target="formula")
        for l1 in specials:
            add("rep", C.xyzz(rng.choice(pool), l1), target="formula")
        for _ in range(N_RANDOM):
            add("random", C.xyzz(rng.choice(pool), lam()), target="formula")
        for _ in range(N_CLASS):
            add("off y=0", (lam(), K.zero, lam(), lam()), False, "y=0")
        nco = 4
    else:
        add("inf", (K.zero, K.zero), target="y=0")
        for _ in range(N_RANDOM):
            P = rng.choice(pool)
            add("random", P, target="formula")
        for _ in range(N_CLASS):
            add("off y=0", (lam(), K.zero), False, "y=0")
        nco = 2

    # off-curve: every coordinate from the raw constants {0, 1, p-1, R mod p}, exhaustively where that is at most N_CONST
    consts = [K.plain(w) for w in _const_words(K)]
    total = len(consts) ** nco
    if total <= N_CONST:
        for k in range(total):
            add("off const", tuple(consts[(k // len(consts) ** j) % len(consts)] for j in range(nco)), False)
    else:
        for _ in range(N_CONST):
            add("off const", tuple(rng.choice(consts) for _ in range(nco)), False)

    for label, target in targets.items():
        got = {b for lab, _, _, _, b in recs if lab == label}
        if got != {target}:
            raise AssertionError(f"ec_edges generator: {GROUPS[group]} {name} class '{label}' takes {sorted(got)}, "
                                 f"not only '{target}'")
    return tuple(recs)


def _const_words(K) -> list[tuple]:
    p = K.p
    vals = [0, 1, p - 1, K.F.R % p]
    if K.deg == 1:
        return [(v,) for v in vals]
    return [(a, b) for a in vals for b in vals]


def pack(group: int, recs) -> tuple[bytes, bytes]:
    """(input bytes, expected output bytes) of sb_field_eval for these records: Montgomery limbs, Fq2 as c0 || c1."""
    C = curve(group)
    w = 4 * FIELDS[group][2]

    def enc(elems):
        return b"".join(v.to_bytes(w, "little") for e in elems for v in C.K.raw(e))
    return b"".join(enc(a) for _, a, _, _, _ in recs), b"".join(enc(r) for _, _, r, _, _ in recs)


def decode(group: int, out: bytes, i: int) -> tuple:
    """The XYZZ result of record i in sb_field_eval's output, as plain field elements."""
    C = curve(group)
    w = 4 * FIELDS[group][2]
    base = i * 4 * C.words * 4
    words = [int.from_bytes(out[base + j * w:base + (j + 1) * w], "little") for j in range(4 * C.K.deg)]
    d = C.K.deg
    return tuple(C.K.plain(tuple(words[k * d:(k + 1) * d])) for k in range(4))


def describe(group: int, op: int, i: int, rec, what: str = "") -> str:
    label, args, _, _, _ = rec
    return (f"{GROUPS[group]} {OP_NAMES[op]} [{label}] record {i}{': ' + what if what else ''}; operands "
            + ", ".join(curve(group).K.hex(a) for a in args))


def mismatches(group: int, op: int, out: bytes, limit: int = 8) -> list[str]:
    """Descriptions of the records whose output in `out` differs from (a), naming the first differing coordinate, or whose
    on-curve result fails (b) (at most `limit`)."""
    C = curve(group)
    recs = records(group, op)
    _, want = pack(group, recs)
    if len(out) != len(want):
        return [f"{GROUPS[group]} {OP_NAMES[op]}: {len(out)} output bytes, expected {len(want)}"]
    size = 4 * C.words * 4
    bad = []
    for i, rec in enumerate(recs):
        got = decode(group, out, i)
        if out[i * size:(i + 1) * size] != want[i * size:(i + 1) * size]:
            j = next(k for k in range(4) if got[k] != rec[2][k])
            bad.append(describe(group, op, i, rec, f"coordinate {COORDS[j]} got {C.K.hex(got[j])} expected "
                                                   f"{C.K.hex(rec[2][j])}"))
        elif rec[3]:
            why = meaning(C, op, rec[1], got)
            if why:
                bad.append(describe(group, op, i, rec, why))
        if len(bad) >= limit:
            break
    return bad
