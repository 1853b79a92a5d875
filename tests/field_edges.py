"""Edge operands and exact expected results for the device field primitives (sb_field_eval, include/snarkb200.h), in Python
integers only: no GPU and no oracle.

For every (field, op) pair, `records(field, op)` returns labelled records (label, operands, expected results).  Every
operand and result is one N-limb element (a 2N-limb value is split into its low and high N limbs), in the raw residues the
kernels see: a "Montgomery" multiply of raw a and b is a*b*R^-1 mod p with R = 2^(32N).

Operand classes:
  const       0, 1, 2, p-1, p-2, (p+-1)/2, R mod p, R^2 mod p, 2^(32k)-1, 2^(32k), p-2^(32k) (whole-limb carry runs), and
              every pair / quadruple pattern of them
  add/sub     sums a+b of p-1, p, p+1, 2p-2; differences a-b of 0, -1, -(p-1)
  mul, mul2   operands for which the value before the final subtraction, t = (a*b [+ u*v] + M*p)/R with
              M = -(a*b [+ u*v])*p^-1 mod R, is p-1, p+1, p+2^32 or within 2^-64 of the top of its range, just under
              p + p^2/R (p + 2p^2/R for mul2)
  raw         to_mont / from_mont inputs in [p, 2^(32N)), which the conversion kernels take unchecked
  wide        products of p-1, 2p-2 and all-ones-limb values; redc_wide inputs T = t*R - M*p for t in {p-1, p, p+1},
              M in {0, 1, R-1}, and T = p*R - 1
  fp2         a0*b0 < a1*b1 and a0*b0 = a1*b1 (the borrow and the zero path of the lazy multiply), unreduced sums a0+a1 >= p,
              inversion of (0,0), (1,0), (0,1), (p-1,p-1)
  inv         0, 1, p-1, R mod p, 2^k and 2^k-1 over the whole bit range
  random      uniform background
Every crafted class is checked to have hit what it aims at: the generator recomputes the targeted quantity for its records
and raises if no record reaches it, so a broken generator cannot quietly weaken the tests that use it."""
from __future__ import annotations

import functools
import random
from fractions import Fraction

FIELDS = {  # id: (name, p, limbs); ids as sb_field_eval (4, 5: Fq2 over the base field of 0, 2)
    0: ("BN254 Fq", 0x30644e72e131a029b85045b68181585d97816a916871ca8d3c208c16d87cfd47, 8),
    1: ("BN254 Fr", 0x30644e72e131a029b85045b68181585d2833e84879b9709143e1f593f0000001, 8),
    2: ("BLS12-381 Fq", 0x1a0111ea397fe69a4b1ba7b6434bacd764774b84f38512bf6730d2a0f6b0f6241eabfffeb153ffffb9feffffffffaaab, 12),
    3: ("BLS12-381 Fr", 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001, 8),
    4: ("BN254 Fq2", 0x30644e72e131a029b85045b68181585d97816a916871ca8d3c208c16d87cfd47, 8),
    5: ("BLS12-381 Fq2", 0x1a0111ea397fe69a4b1ba7b6434bacd764774b84f38512bf6730d2a0f6b0f6241eabfffeb153ffffb9feffffffffaaab, 12),
}
FP_OPS = {"add": 0, "sub": 1, "neg": 2, "dbl": 3, "mul": 4, "mul2": 5, "mul_wide": 6, "redc_wide": 7, "to_mont": 8,
          "from_mont": 9, "inv_binary": 10, "inv": 11}
FP2_OPS = {"mul_i": 12, "mul_lazy": 13, "sqr_i": 14, "inv": 15}
OP_NAMES = {**{v: k for k, v in FP_OPS.items()}, **{v: "fp2_" + k for k, v in FP2_OPS.items()}}
FE_NOPS = 21                   # the first op sb_field_eval does not define; 16-20 are the point ops of tests/ec_edges.py
N_RANDOM = 1000


def has_mul2(p: int, limbs: int) -> bool:
    return 3 * p < 1 << (32 * limbs)          # Fp::HAS_MUL2: the dual-product running sum fits N limbs


def ops(field: int) -> list[int]:
    """The ops sb_field_eval defines on `field`."""
    _, p, n = FIELDS[field]
    if field >= 4:
        return list(FP2_OPS.values())
    return [o for o in FP_OPS.values() if o != FP_OPS["mul2"] or has_mul2(p, n)]


def all_sets() -> list[tuple[int, int]]:
    return [(f, o) for f in FIELDS for o in ops(f)]


class _F:
    """Constants of one prime field and the quantities the crafted classes aim at."""

    def __init__(self, p: int, n: int):
        self.p, self.n = p, n
        self.R = 1 << (32 * n)
        self.Ri = pow(self.R, -1, p)
        self.pinv = pow(p, -1, self.R)

    def mont(self, *prod):                      # the multiply's M for the product (sum) and its pre-subtraction value t
        M = (-sum(prod) * self.pinv) % self.R
        T = sum(prod) + M * self.p
        assert T % self.R == 0
        return M, T // self.R

    def consts(self) -> dict[str, int]:
        p, R, n = self.p, self.R, self.n
        c = {"0": 0, "1": 1, "2": 2, "p-1": p - 1, "p-2": p - 2, "(p-1)/2": (p - 1) // 2, "(p+1)/2": (p + 1) // 2,
             "R mod p": R % p, "R^2 mod p": R * R % p}
        for k in range(1, n + 1):
            c[f"2^{32 * k}-1"] = (1 << (32 * k)) - 1
            c[f"2^{32 * k}"] = 1 << (32 * k)
        for k in range(n):
            c[f"p-2^{32 * k}"] = p - (1 << (32 * k))
        out, seen = {}, set()
        for k, v in c.items():                    # canonical and distinct
            if 0 <= v < p and v not in seen:
                out[k] = v
                seen.add(v)
        return out

    def raw(self) -> dict[str, int]:
        """Inputs in [p, R): not field elements, but what an unchecked conversion can be handed."""
        p, R = self.p, self.R
        c = {"p": p, "p+1": p + 1, "2p-1": 2 * p - 1, "2p": 2 * p, "R-1": R - 1, "R-p": R - p}
        for k in range(self.n):
            c[f"p+2^{32 * k}"] = p + (1 << (32 * k))
        for k in range(1, self.n):
            c[f"R-2^{32 * k}"] = R - (1 << (32 * k))
        return {k: v for k, v in c.items() if p <= v < R}

    def near_top(self, prod_fixed: int, u: int, D: int):
        """y >= 1 for which M of prod_fixed + u*(p - y) lies in [R-D, R), found as a close vector of a 2-dimensional lattice:
        M(y) = M0 + y*alpha mod R is an arithmetic progression in y, and {(y, y*alpha - j*R)} holds every (y, M(y) - M0).
        With D about sqrt(R) both y and R - M come out near sqrt(R), so t sits about p*2^(16N)/R below its maximum."""
        R = self.R
        M0 = (-(prod_fixed + u * self.p) * self.pinv) % R
        alpha = (u * self.pinv) % R
        tau = (-M0 - D) % R                        # want y*alpha = tau + e (mod R), 0 <= e < D
        b1, b2 = _gauss((1, alpha), (0, R))
        det = b1[0] * b2[1] - b1[1] * b2[0]
        tgt = (0, tau + D // 2)
        c1 = round(Fraction(tgt[0] * b2[1] - tgt[1] * b2[0], det))
        c2 = round(Fraction(b1[0] * tgt[1] - b1[1] * tgt[0], det))
        best = None
        for i in range(-6, 7):
            for j in range(-6, 7):
                y = (c1 + i) * b1[0] + (c2 + j) * b2[0]
                e = (c1 + i) * b1[1] + (c2 + j) * b2[1] - tau
                if 1 <= y < self.p and 0 <= e < D and (best is None or y < best):
                    best = y
        return best


def _gauss(u, v):
    """Lagrange-Gauss reduction of a 2-dimensional lattice basis."""
    def dot(a, b):
        return a[0] * b[0] + a[1] * b[1]
    if dot(u, u) > dot(v, v):
        u, v = v, u
    while True:
        uu = dot(u, u)
        m = (2 * dot(u, v) + uu) // (2 * uu)
        v = (v[0] - m * u[0], v[1] - m * u[1])
        if dot(v, v) >= uu:
            return u, v
        u, v = v, u


def _hit(recs, label: str, pred, what: str):
    """The crafted class `label` must contain a record for which pred(operands) holds."""
    if not any(pred(a) for lab, a, _ in recs if lab == label):
        raise AssertionError(f"field_edges generator: no '{label}' record reaches {what}")


@functools.lru_cache(maxsize=None)
def records(field: int, op: int) -> tuple:
    """((label, operands, expected), ...) for (field, op), deterministic."""
    name, p, n = FIELDS[field]
    if op not in ops(field):
        raise ValueError(f"op {op} is not defined on {name}")
    F = _F(p, n)
    R, Ri = F.R, F.Ri
    rng = random.Random(1000 * field + op)
    C = F.consts()
    cv = list(C.items())
    recs = []

    def add(label, args, want):
        recs.append((label, tuple(args), tuple(want)))

    def rnd():
        return rng.randrange(p)

    def minv(a):                                   # R^2 * a^-1 (Montgomery inverse), 0 -> 0
        return R * R * pow(a, -1, p) % p if a % p else 0

    if field >= 4:
        return _fp2_records(F, op, cv, rng, add, recs)

    opname = OP_NAMES[op]
    if opname in ("add", "sub", "mul", "mul_wide"):
        want = {"add": lambda a, b: [(a + b) % p], "sub": lambda a, b: [(a - b) % p],
                "mul": lambda a, b: [a * b * Ri % p], "mul_wide": lambda a, b: [a * b % R, a * b // R]}[opname]
        for la, a in cv:
            for lb, b in cv:
                add(f"const {la},{lb}", (a, b), want(a, b))
        if opname == "add":
            for tgt, lab in ((p - 1, "a+b=p-1"), (p, "a+b=p"), (p + 1, "a+b=p+1"), (2 * p - 2, "a+b=2p-2")):
                for a in [v for _, v in cv] + [rnd() for _ in range(8)]:
                    if 0 <= tgt - a < p:
                        add(lab, (a, tgt - a), want(a, tgt - a))
                _hit(recs, lab, lambda x, t=tgt: x[0] + x[1] == t, f"a+b = {lab[4:]}")
        if opname == "sub":
            for d, lab in ((0, "a-b=0"), (-1, "a-b=-1"), (-(p - 1), "a-b=-(p-1)")):
                for a in [v for _, v in cv] + [rnd() for _ in range(8)]:
                    if 0 <= a - d < p:
                        add(lab, (a, a - d), want(a, a - d))
                _hit(recs, lab, lambda x, d=d: x[0] - x[1] == d, f"a-b = {lab[4:]}")
        if opname == "mul":
            for tgt, lab in ((p - 1, "t=p-1"), (p + 1, "t=p+1"), (p + (1 << 32), "t=p+2^32")):
                for _ in range(40):                  # pick a, solve b = t*R*a^-1; keep it when 0 <= M < R
                    a = rng.randrange(1, p)
                    b = tgt * R * pow(a, -1, p) % p
                    if 0 <= (tgt * R - a * b) // p < R:
                        add(lab, (a, b), want(a, b))
                _hit(recs, lab, lambda x, t=tgt: F.mont(x[0] * x[1])[1] == t, lab)
            tmax = ((p - 1) ** 2 + (R - 1) * p) // R
            for x in range(1, 9):
                a = p - x
                y = F.near_top(0, a, 1 << (16 * n + 4))          # b = p - y: a*b = a*p - a*y
                if y is not None:
                    add("t~max", (a, p - y), want(a, p - y))
            _hit(recs, "t~max", lambda x: F.mont(x[0] * x[1])[1] > tmax - ((tmax - p) >> 64),
                 "the top 2^-64 of [p, p + p^2/R)")
        if opname == "mul_wide":
            ones = [(1 << (32 * k)) - 1 for k in range(1, n + 1)]
            for a in ones + [p - 1, 2 * p - 2]:      # 2p-2: the unreduced sums the lazy Fq2 multiply feeds in
                for b in ones + [p - 1, 2 * p - 2]:
                    add("wide", (a, b), want(a, b))
            _hit(recs, "wide", lambda x: x[0] == x[1] == R - 1, "(R-1)^2")
        for _ in range(N_RANDOM):
            a, b = rnd(), rnd()
            add("random", (a, b), want(a, b))
    elif opname == "mul2":
        def want(x, y, u, v):
            return [(x * y + u * v) * Ri % p]
        for la, a in cv:
            for lb, b in cv:
                add(f"const {la},{lb},{la},{lb}", (a, b, a, b), want(a, b, a, b))
                add(f"const {la},{lb},{lb},{la}", (a, b, b, a), want(a, b, b, a))
                add(f"const {la},{la},{lb},{lb}", (a, a, b, b), want(a, a, b, b))
        for tgt, lab in ((p - 1, "t=p-1"), (p + 1, "t=p+1"), (p + (1 << 32), "t=p+2^32")):
            for _ in range(40):                      # pick x, y, u, solve v
                x, y, u = rng.randrange(1, p), rng.randrange(1, p), rng.randrange(1, p)
                v = (tgt * R - x * y) * pow(u, -1, p) % p
                if 0 <= (tgt * R - x * y - u * v) // p < R:
                    add(lab, (x, y, u, v), want(x, y, u, v))
            _hit(recs, lab, lambda q, t=tgt: F.mont(q[0] * q[1], q[2] * q[3])[1] == t, lab)
        tmax = (2 * (p - 1) ** 2 + (R - 1) * p) // R
        for s in range(1, 9):
            x, y, u = p - 1, p - 1, p - s
            w = F.near_top(x * y, u, 1 << (16 * n + 4))     # v = p - w
            if w is not None:
                add("t~max", (x, y, u, p - w), want(x, y, u, p - w))
        _hit(recs, "t~max", lambda q: F.mont(q[0] * q[1], q[2] * q[3])[1] > tmax - ((tmax - p) >> 64),
             "the top 2^-64 of [p, p + 2p^2/R)")
        for _ in range(N_RANDOM):
            q = [rnd() for _ in range(4)]
            add("random", q, want(*q))
    elif opname == "redc_wide":
        def want(T):
            return [T * Ri % p]
        targets = {}
        for t in (p - 1, p, p + 1):
            for M, lm in ((0, "0"), (1, "1"), (R - 1, "R-1")):
                T = t * R - M * p
                if 0 <= T < p * R:
                    lab = f"T=tR-Mp t={'p-1' if t == p - 1 else 'p' if t == p else 'p+1'} M={lm}"
                    add(lab, (T % R, T // R), want(T))
                    targets[lab] = t
        for lab, t in targets.items():
            _hit(recs, lab, lambda x, t=t: F.mont(x[0] + x[1] * R)[1] == t, lab)
        for t in (p - 1, p, p + 1):
            if not any(F.mont(a[0] + a[1] * R)[1] == t for lb, a, _ in recs if lb.startswith("T=tR-Mp")):
                raise AssertionError(f"field_edges generator: no redc_wide record reaches t = p{t - p:+d}")
        for T, lab in ((p * R - 1, "T=pR-1"), (0, "T=0"), ((p - 1) ** 2, "T=(p-1)^2"), (2 * (p - 1) ** 2, "T=2(p-1)^2")):
            add(lab, (T % R, T // R), want(T))
        for _ in range(N_RANDOM):
            T = rng.randrange(p * R)
            add("random", (T % R, T // R), want(T))
    else:                                           # unary
        fn = {"neg": lambda a: (-a) % p, "dbl": lambda a: 2 * a % p, "to_mont": lambda a: a * R % p,
              "from_mont": lambda a: a * Ri % p, "inv_binary": minv, "inv": minv}[opname]
        for la, a in cv:
            add(f"const {la}", (a,), [fn(a)])
        if opname in ("to_mont", "from_mont"):
            for la, a in F.raw().items():
                add(f"raw {la}", (a,), [fn(a)])
            for _ in range(64):
                a = rng.randrange(p, R)
                add("raw random", (a,), [fn(a)])
            _hit(recs, "raw R-1", lambda x: x[0] == R - 1, "R-1")
        if opname in ("inv_binary", "inv"):
            bits = p.bit_length()
            for k in sorted(set(range(1, bits, 5)) | {bits - 1}):
                for a, la in ((1 << k, f"2^{k}"), ((1 << k) - 1, f"2^{k}-1")):
                    if 0 < a < p:
                        add("inv " + la, (a,), [fn(a)])
            _hit(recs, "inv 2^" + str(bits - 1), lambda x: x[0] == 1 << (bits - 1), "2^(bits-1)")
        if opname == "dbl":
            _hit(recs, "const (p+1)/2", lambda x: 2 * x[0] == p + 1, "2a = p+1")
        n_rand = N_RANDOM // 4 if opname == "inv" else N_RANDOM
        for _ in range(n_rand):
            a = rnd()
            add("random", (a,), [fn(a)])
    return tuple(recs)


def _fp2_records(F: _F, op: int, cv, rng, add, recs) -> tuple:
    p, R, Ri = F.p, F.R, F.Ri
    opname = OP_NAMES[op][len("fp2_"):]

    def mul(x, y):
        return [(x[0] * y[0] - x[1] * y[1]) * Ri % p, (x[0] * y[1] + x[1] * y[0]) * Ri % p]

    def inv(x):
        d = (x[0] * x[0] + x[1] * x[1]) % p
        if d == 0:
            return [0, 0]
        di = pow(d, -1, p)
        return [x[0] * R * R * di % p, (-x[1]) * R * R * di % p]

    def rnd2():
        return (rng.randrange(p), rng.randrange(p))

    pairs = [((la, a), (lb, b)) for la, a in cv for lb, b in cv]
    if opname in ("mul_i", "mul_lazy"):
        ys = [(1, p - 1), (p - 1, 1), (p - 1, p - 1), ((p + 1) // 2, (p + 1) // 2), (R % p, 0), (0, R % p)]
        for (la, a), (lb, b) in pairs:
            for y in ys:
                add(f"const ({la},{lb})", (a, b, *y), mul((a, b), y))
        for _ in range(64):
            c, d = rng.randrange(1, p), rng.randrange(1, p)
            add("a0b0=a1b1", (c, d, d, c), mul((c, d), (d, c)))                    # zero path of a0b0 - a1b1
            c, d = rng.randrange(1, p // 2), rng.randrange(p // 2, p)
            add("a0b0<a1b1", (c, d, c, d), mul((c, d), (c, d)))                    # borrow path
            c, d = rng.randrange((p + 1) // 2, p), rng.randrange((p + 1) // 2, p)
            y = (rng.randrange((p + 1) // 2, p), rng.randrange((p + 1) // 2, p))
            add("a0+a1>=p", (c, d, *y), mul((c, d), y))
        _hit(recs, "a0b0=a1b1", lambda q: q[0] * q[2] == q[1] * q[3], "a0*b0 = a1*b1")
        _hit(recs, "a0b0<a1b1", lambda q: q[0] * q[2] < q[1] * q[3], "a0*b0 < a1*b1")
        _hit(recs, "a0+a1>=p", lambda q: q[0] + q[1] >= p and q[2] + q[3] >= p, "a0+a1 >= p and b0+b1 >= p")
        for _ in range(N_RANDOM):
            x, y = rnd2(), rnd2()
            add("random", (*x, *y), mul(x, y))
    else:
        fn = (lambda x: mul(x, x)) if opname == "sqr_i" else inv
        for (la, a), (lb, b) in pairs:
            add(f"const ({la},{lb})", (a, b), fn((a, b)))
        for x, lab in (((0, 0), "(0,0)"), ((1, 0), "(1,0)"), ((0, 1), "(0,1)"), ((p - 1, p - 1), "(p-1,p-1)")):
            add(lab, x, fn(x))
        for _ in range(N_RANDOM // 4 if opname == "inv" else N_RANDOM):
            x = rnd2()
            add("random", x, fn(x))
    return tuple(recs)


def pack(field: int, recs) -> tuple[bytes, bytes]:
    """(input bytes, expected output bytes) of sb_field_eval for these records."""
    w = 4 * FIELDS[field][2]
    return (b"".join(v.to_bytes(w, "little") for _, a, _ in recs for v in a),
            b"".join(v.to_bytes(w, "little") for _, _, e in recs for v in e))


def describe(field: int, op: int, rec, got: tuple | None = None) -> str:
    label, args, want = rec
    s = f"{FIELDS[field][0]} {OP_NAMES[op]} [{label}] operands " + ", ".join(hex(v) for v in args)
    s += " expected " + ", ".join(hex(v) for v in want)
    if got is not None:
        s += " got " + ", ".join(hex(v) for v in got)
    return s


def mismatches(field: int, op: int, out: bytes, limit: int = 8) -> list[str]:
    """Descriptions of the records whose output in `out` differs from the expected bytes (at most `limit`)."""
    recs = records(field, op)
    w = 4 * FIELDS[field][2]
    k = len(recs[0][2])
    _, want = pack(field, recs)
    if len(out) != len(want):
        return [f"{FIELDS[field][0]} {OP_NAMES[op]}: {len(out)} output bytes, expected {len(want)}"]
    bad = []
    for i, rec in enumerate(recs):
        lo, hi = i * k * w, (i + 1) * k * w
        if out[lo:hi] != want[lo:hi]:
            got = tuple(int.from_bytes(out[lo + j * w:lo + (j + 1) * w], "little") for j in range(k))
            bad.append(describe(field, op, rec, got))
            if len(bad) >= limit:
                break
    return bad
