"""Groth16 circuits with the shapes real circom circuits have, for the proving tests.  Every other Groth16 key the suite
proves comes from the chain x_{i+1} = x_i^2 + b: one entry per A and B row, every coefficient 1, one public signal and
nVars equal to the domain.  The classes here vary what that chain keeps fixed:

  bits    Num2Bits: one A row sums 2^i * b_i over every bit of a field element, and b_i * (b_i - 1) = 0 for each bit
  wide    one A row and one B row of 2^14 terms each (one serial loop per row in the QAP kernel)
  coeffs  coefficients 0, 1, r - 1, (r - 1)/2, 2^k and uniform; explicit zero entries; one signal twice in a linear
          combination; the constant signal 0 with large coefficients
  empty   constraints with an empty A side, an empty B side, both, or all three
  public  nPublic public signals, split between outputs and public inputs, each one used by a constraint
  fit     nConstraints + nPublic + 1 exactly 2^k (no zero rows), or 2^k + 1 (the domain doubles)
  gates   the same for PLONK and fflonk keys: exactly 2^k + extra gates, with no additions
  ratio   nVars far above or far below the domain, so that the witness MSMs and the H MSM get different geometries
  tiny    a given nVars, down to 1; nVars = nPublic + 1 leaves no private signal and an empty section 8

A circuit is a list of constraints (A, B, C), each a list of (signal, coefficient) with plain integer coefficients, and a
witness.  Every class checks in Python integers that its witness satisfies every constraint and raises if it does not.
Signals are numbered like circom's: 0 is the constant one, then the outputs, the public inputs, the private inputs and
the internal signals.

Keys come two ways:
  structured_zkey    r1cs -> oracle.zkey_new over a prepared powers of tau with known tau, alpha and beta: the proofs
                     verify.  For domains of 1024 and below.
  unstructured_zkey  the key's header and section 4 exactly as zkey_new writes them, with random valid curve points as
                     bases (the layout of snarkjs_b200.synth.groth16_zkey_image): proofs do not verify, but the bytes
                     of every proof are defined.  For any size.
shuffle() permutes the section 4 entries; the prover sums a row's entries in any order, so proofs must not change.
PLONK and fflonk keys (PLONK_CASES) come from oracle.plonk.plonk_setup / oracle.fflonk.fflonk_setup over a ptau with the
same known tau (oracle.synth_setup.plonk_ptau), or with pseudo-random points in place of its powers."""
from __future__ import annotations

import functools
import random
import struct

import numpy as np

from oracle import oracle as O
from oracle import synth_setup as SS
from oracle.plonk import wtns_bytes

KIND_ORDER = {"one": 0, "out": 1, "pub": 2, "prv": 3, "int": 4}


class Circuit:
    """Base class: subclasses add signals with new() and constraints with add() / solve() inside build()."""
    name = "circuit"

    def __init__(self, curve: int, seed: int = 1, **params):
        self.curve, self.seed, self.params = curve, seed, params
        self.r = O.CURVES[curve].r
        self.rnd = random.Random(f"{self.name}/{curve}/{seed}/{sorted(params.items())}")
        self.kind = ["one"]
        self.w = [1]
        self.cons = []
        self.build(**params)
        self._renumber()
        self.check()

    # ----------------------------------------------------------------------------------------------- construction
    def new(self, kind: str, value: int | None = None) -> int:
        self.kind.append(kind)
        self.w.append(self.rnd.randrange(self.r) if value is None else value % self.r)
        return len(self.w) - 1

    def value(self, lc) -> int:
        return sum(v * self.w[s] for s, v in lc) % self.r

    def add(self, A, B, C):
        self.cons.append((list(A), list(B), list(C)))

    def solve(self, A, B, C, kind: str = "int", coef: int = 1) -> int:
        """Adds a signal t and the constraint A * B = C + coef * t, with t's value the one that satisfies it."""
        assert coef % self.r
        t = self.new(kind, 0)
        self.w[t] = (self.value(A) * self.value(B) - self.value(C)) * pow(coef, -1, self.r) % self.r
        self.add(A, B, list(C) + [(t, coef)])
        return t

    def build(self, **params):
        raise NotImplementedError

    def _renumber(self):
        """circom order: one, outputs, public inputs, private inputs, internal signals (each kind in creation order)."""
        order = sorted(range(len(self.w)), key=lambda s: (KIND_ORDER[self.kind[s]], s))
        assert order[0] == 0
        new_id = {old: i for i, old in enumerate(order)}
        self.w = [self.w[old] for old in order]
        self.kind = [self.kind[old] for old in order]
        self.cons = [tuple([(new_id[s], v) for s, v in lc] for lc in con) for con in self.cons]

    # ----------------------------------------------------------------------------------------------- properties
    @property
    def n_vars(self):
        return len(self.w)

    @property
    def n_outputs(self):
        return self.kind.count("out")

    @property
    def n_pub_inputs(self):
        return self.kind.count("pub")

    @property
    def n_public(self):
        return self.n_outputs + self.n_pub_inputs

    @property
    def domain(self):
        """zkey_new's domain: 2^(floor(log2(nConstraints + nPublic)) + 1) (src/zkey_new.js:59)."""
        return 1 << (len(self.cons) + self.n_public).bit_length()

    def unsatisfied(self, witness=None):
        """Indices of the constraints the witness (default: the circuit's own) does not satisfy."""
        w = self.w if witness is None else witness
        val = lambda lc: sum(v * w[s] for s, v in lc) % self.r
        return [i for i, (a, b, c) in enumerate(self.cons) if (val(a) * val(b) - val(c)) % self.r]

    def check(self):
        bad = self.unsatisfied()
        if bad:
            raise ValueError(f"{self.name}: witness does not satisfy constraints {bad[:8]}")
        for con in self.cons:
            for lc in con:
                for s, v in lc:
                    if not (0 <= s < self.n_vars and 0 <= v < self.r):
                        raise ValueError(f"{self.name}: entry ({s}, {v}) out of range")

    def broken_witness(self):
        """The witness with one signal outside the public ones changed, so that some constraint fails."""
        w = list(self.w)
        for s in range(self.n_vars - 1, self.n_public, -1):
            w[s] = (w[s] + 1) % self.r
            if self.unsatisfied(w):
                return w
            w[s] = self.w[s]
        raise ValueError(f"{self.name}: no private signal changes a constraint")

    # ----------------------------------------------------------------------------------------------- containers
    def r1cs_bytes(self) -> bytes:
        """.r1cs container (r1csfile layout: header, constraints, wire-to-label map)."""
        n8 = 32
        body = bytearray()
        for con in self.cons:
            for lc in con:
                body += struct.pack("<I", len(lc))
                for s, v in lc:
                    body += struct.pack("<I", s) + v.to_bytes(n8, "little")
        n_prv = self.kind.count("prv")
        hdr = struct.pack("<I", n8) + self.r.to_bytes(n8, "little")
        hdr += struct.pack("<IIII", self.n_vars, self.n_outputs, self.n_pub_inputs, n_prv)
        hdr += struct.pack("<Q", self.n_vars) + struct.pack("<I", len(self.cons))
        labels = b"".join(struct.pack("<Q", i) for i in range(self.n_vars))
        return O.write_binfile("r1cs", 1, [(1, hdr), (2, bytes(body)), (3, labels)])

    def wtns(self, witness=None) -> bytes:
        return wtns_bytes(self.w if witness is None else witness, self.r)

    def witness_array(self, witness=None) -> np.ndarray:
        w = self.w if witness is None else witness
        return np.frombuffer(b"".join(int(x).to_bytes(32, "little") for x in w), np.uint8)

    def public(self):
        return self.w[1:self.n_public + 1]

    def __repr__(self):
        return f"{self.name}(curve={self.curve}, nVars={self.n_vars}, nPublic={self.n_public}, rows={len(self.cons)}, domain={self.domain})"


# --------------------------------------------------------------------------------------------------- the shapes
class Bits(Circuit):
    """Num2Bits of a public input x: bits b_i with b_i * (b_i - 1) = 0, and (sum 2^i b_i) * 1 = x."""
    name = "bits"

    def build(self):
        nbits = 254 if self.curve == O.BN254 else 255
        x = self.new("pub")
        bits = [self.new("int", (self.w[x] >> i) & 1) for i in range(nbits)]
        for b in bits:
            self.add([(b, 1)], [(b, 1), (0, self.r - 1)], [])
        self.add([(b, 1 << i) for i, b in enumerate(bits)], [(0, 1)], [(x, 1)])


class Wide(Circuit):
    """out = (sum c_j u_j) * (sum d_j v_j) with `terms` entries on each side, plus a short row that uses the output."""
    name = "wide"

    def build(self, terms=1 << 14):
        u = [self.new("prv") for _ in range(terms)]
        v = [self.new("prv") for _ in range(terms)]
        A = [(s, self.rnd.randrange(1, self.r)) for s in u]
        B = [(s, self.rnd.randrange(1, self.r)) for s in v]
        out = self.solve(A, B, [], "out")
        self.solve([(out, 1)], [(u[0], 1), (v[-1], 1)], [])


class Coeffs(Circuit):
    """Coefficients at the edges of Fr, explicit zero entries, a signal twice in one linear combination, and the
    constant signal with large coefficients.  repeat=False keeps every signal to one entry per linear combination: PLONK
    and fflonk keys key a linear combination by signal, so a repeated signal's last entry overwrites the others and the
    key no longer encodes the circuit (src/plonk_setup.js, src/r1cs_constraint_processor.js)."""
    name = "coeffs"

    def coef(self):
        r = self.r
        return self.rnd.choice([0, 1, r - 1, (r - 1) // 2, (r + 1) // 2, 1 << self.rnd.randrange(r.bit_length() - 1),
                                r - (1 << self.rnd.randrange(64)), self.rnd.randrange(r), self.rnd.randrange(r)])

    def lc(self, pool, k):
        out = [(self.rnd.choice(pool), self.coef()) for _ in range(k)]
        if out and self.rnd.random() < 0.5:                 # the same signal twice: the entries must add up
            s, v = out[0][0], self.coef()
            if self.repeat:
                out.append((s, v))
        if self.rnd.random() < 0.3:                         # the constant signal with a large coefficient
            out.append((0, self.r - 1 - self.rnd.randrange(1 << 32)))
        if self.rnd.random() < 0.3:                         # an explicit zero entry
            out.append((self.rnd.choice(pool), 0))
        if not self.repeat:                                 # the first entry of each signal
            first = {}
            for s, v in out:
                first.setdefault(s, v)
            out = list(first.items())
        self.rnd.shuffle(out)
        return out

    def build(self, rows=96, repeat=True):
        self.repeat = repeat
        x = self.new("pub")
        pool = [x] + [self.new("prv") for _ in range(12)]
        specials = [0, 1, self.r - 1, (self.r - 1) // 2, 1 << 200]
        for i in range(rows):
            A, B, C = self.lc(pool, self.rnd.randrange(1, 5)), self.lc(pool, self.rnd.randrange(1, 5)), self.lc(pool, self.rnd.randrange(0, 3))
            if i < len(specials):                           # every special coefficient on a lone entry of A and of B
                A, B = [(pool[i + 1], specials[i])], [(pool[i + 2], specials[-1 - i])]
            kind = "out" if i == rows - 1 else "int"
            c = self.coef() or self.r - 1
            pool.append(self.solve(A, B, C, kind, c))
        # a row whose A and B entries all carry the coefficient 0, next to ones that cancel to zero
        z = pool[3]
        self.add([(z, 0), (pool[4], 0)], [(z, 1)], [(z, 5), (z, self.r - 5)] if repeat else [(z, 0), (pool[5], 0)])


class Empty(Circuit):
    """Constraints whose A side, B side, or both are empty (0 = C.w), an all-empty row, and an empty C side."""
    name = "empty"

    def build(self, rows=40):
        pool = [self.new("prv") for _ in range(6)]
        zero = self.solve([], [(pool[0], 1)], [])           # A empty: the solved signal is 0
        pool.append(self.solve([(pool[1], 1)], [(pool[2], 3)], [], "out"))
        for i in range(rows):
            kind = i % 4
            other = [(self.rnd.choice(pool), self.rnd.randrange(self.r)) for _ in range(self.rnd.randrange(0, 3))]
            side = [(self.rnd.choice(pool), self.rnd.randrange(1, self.r)) for _ in range(self.rnd.randrange(1, 4))]
            if kind == 0:
                pool.append(self.solve([], side, other))
            elif kind == 1:
                pool.append(self.solve(side, [], other))
            elif kind == 2:
                pool.append(self.solve([], [], other, coef=self.rnd.randrange(1, self.r)))
            else:
                self.add([], [], [])
        self.add([(zero, 1)], side, [])                        # C empty: A.w = 0
        self.add([], [], [])


class Public(Circuit):
    """n_public public signals, a third of them outputs and the rest public inputs; each takes part in a constraint."""
    name = "public"

    def build(self, n_public=17, n_private=8):
        n_out = (n_public + 2) // 3
        ins = [self.new("pub") for _ in range(n_public - n_out)]
        prv = [self.new("prv") for _ in range(n_private)]
        k = 0
        for j in range(n_out):                               # out_j = (in + prv) * prv'
            a = [(ins[k % len(ins)], 1), (prv[j % n_private], 2)] if ins else [(prv[j % n_private], 2)]
            k += 1
            self.solve(a, [(prv[(j + 1) % n_private], 1)], [], "out")
        while k < len(ins):                                  # the remaining public inputs, two per row
            pair = ins[k:k + 2]
            k += 2
            self.solve([(pair[0], 1)], [(pair[-1], 3), (0, 1)], [(prv[k % n_private], 7)])
        if n_public == 0:
            self.solve([(prv[0], 1)], [(prv[1], 1)], [])


class Fit(Circuit):
    """nConstraints + nPublic + 1 = 2^k + extra (k >= 4) with two public signals: extra = 0 fills the domain to its
    last row, extra = 1 doubles it."""
    name = "fit"

    def build(self, k=8, extra=0):
        x = self.new("pub")
        prev = [x, self.new("prv")]
        rows = (1 << k) + extra - 3
        for i in range(rows - 1):
            prev.append(self.solve([(prev[-1], 1), (prev[-2], 2)], [(prev[-2], 1)], [(0, i)]))
        self.solve([(prev[-1], 1)], [(0, 1)], [], "out")


class Gates(Circuit):
    """Two public inputs and 2^k + extra - 2 rows of one entry per side (no PLONK additions): 2^k + extra PLONK / fflonk
    gates.  PLONK's domain is 2^bitlen(gates - 1) and fflonk's 2^bitlen(gates + 1), as fflonk keeps two rows for its
    blinding: extra = 0 / 1 fills / doubles the PLONK domain, extra = -2 / -1 the fflonk domain."""
    name = "gates"

    def build(self, k=8, extra=0):
        prev = [self.new("pub"), self.new("pub")]
        for i in range((1 << k) + extra - 2):
            a, b = self.rnd.randrange(1, self.r), self.rnd.randrange(1, self.r)
            prev.append(self.solve([(prev[-1], a)], [(prev[-2], b)], [], coef=(i % 7) + 1))


class Ratio(Circuit):
    """mode 'vars': n_vars signals in rows + 1 wide linear constraints (nVars far above the domain when rows is small);
    mode 'rows': four signals in `rows` repeated constraints (nVars far below the domain)."""
    name = "ratio"

    def build(self, mode="vars", n_vars=1 << 15, rows=1 << 9):
        if mode == "rows":
            a, b = self.new("prv"), self.new("prv")
            out = self.solve([(a, 1)], [(b, 1)], [], "out")
            for i in range(rows - 1):
                self.add([(a, 1)], [(b, 1)], [(out, 1)])
            return
        out = self.new("out", 0)
        n_in = n_vars - 2 - rows
        ins = [self.new("prv") for _ in range(n_in)]
        per = -(-n_in // rows)
        acc = []
        for i in range(rows):
            chunk = ins[i * per:(i + 1) * per] or ins[-2:]
            acc.append(self.solve([(s, 1 + (j & 7)) for j, s in enumerate(chunk)], [(0, 1)], []))
        self.w[out] = self.value([(t, 1) for t in acc])
        self.add([(t, 1) for t in acc], [(0, 1)], [(out, 1)])


class Tiny(Circuit):
    """Exactly n_vars signals: nVars = 1 is the constant alone, nVars = 2 and 4 have no private signal (section 8 is
    empty), larger ones have an output, a public input and private inputs."""
    name = "tiny"

    def build(self, n_vars=4):
        if n_vars == 1:
            self.add([(0, 1)], [(0, 1)], [(0, 1)])
            return
        if n_vars == 2:
            self.solve([(0, 3)], [(0, 5)], [], "out")
            return
        if n_vars == 4:
            a, b = self.new("pub"), self.new("pub")
            self.solve([(a, 1)], [(b, 1), (0, 1)], [], "out")
            return
        x = self.new("pub")
        prv = [self.new("prv") for _ in range(n_vars - 3)]
        self.solve([(x, 1), (prv[0], 1)], [(prv[-1], 1)], [], "out")
        for i in range(0, len(prv) - 2, 3):                  # every private signal in some row
            p = prv[i:i + 3]
            c = self.value([(p[0], 1)]) * self.value([(p[1], 1)]) - self.value([(p[-1], 1)])
            self.add([(p[0], 1)], [(p[1], 1)], [(p[-1], 1), (0, c % self.r)])
        if len(prv) % 3:
            p = prv[-2:]
            self.add([(p[0], 1)], [(0, 1)], [(p[0], 1), (p[-1], 0)])


SHAPES = {cls.name: cls for cls in (Bits, Wide, Coeffs, Empty, Public, Fit, Gates, Ratio, Tiny)}

BN, BLS = O.BN254, O.BLS12_381

# label -> (shape, curve, params, structured).  The window tables of the MSMs are built for sets of 2^12 points or more,
# and only when both the witness side (nVars) and the H side (domain) have that many: ratio_vars and wide have only
# the first, ratio_rows only the second, ratio_both both with different window sizes.  On BN254 a plain MSM over 49
# points or fewer uses 3-bit windows (86 of them); tiny covers both sides of that and of BLS12-381's bounds.
CASES = {
    "bits": ("bits", BN, {}, True),
    "coeffs": ("coeffs", BN, {}, True),
    "empty": ("empty", BN, {}, True),
    **{f"public{n}": ("public", BN, {"n_public": n}, True) for n in (0, 2, 17, 300)},
    "fit_exact": ("fit", BN, {"k": 8, "extra": 0}, True),
    "fit_double": ("fit", BN, {"k": 8, "extra": 1}, True),
    **{f"tiny{n}": ("tiny", BN, {"n_vars": n}, True) for n in (1, 2, 4, 7, 48, 49, 50, 64)},
    "wide": ("wide", BN, {"terms": 1 << 14}, False),
    "ratio_vars": ("ratio", BN, {"mode": "vars", "n_vars": 1 << 15, "rows": 1 << 9}, False),
    "ratio_rows": ("ratio", BN, {"mode": "rows", "rows": 1 << 15}, False),
    "ratio_both": ("ratio", BN, {"mode": "vars", "n_vars": 1 << 15, "rows": 3000}, False),
    "bls_bits": ("bits", BLS, {}, True),
    "bls_coeffs": ("coeffs", BLS, {}, True),
    "bls_public17": ("public", BLS, {"n_public": 17}, True),
    **{f"bls_tiny{n}": ("tiny", BLS, {"n_vars": n}, True) for n in (49, 200, 362, 363, 400)},
    "bls_ratio_vars": ("ratio", BLS, {"mode": "vars", "n_vars": 1 << 14, "rows": 1 << 8}, False),
    "bls_ratio_rows": ("ratio", BLS, {"mode": "rows", "rows": 1 << 13}, False),
    "bls_ratio_both": ("ratio", BLS, {"mode": "vars", "n_vars": 1 << 14, "rows": 3000}, False),
}


# The same format for PLONK and fflonk keys (plonk_zkey / fflonk_zkey), with CASES' labels where the circuit is the same.
# Structured keys are for domains of 1024 and below.  The tiny circuits give the minimum domain of 8 and domain 32 (a
# commitment of n + 3 ... n + 6 <= 49 points takes 3-bit windows on BN254); public17 / public300 put 17 / 300 Lagrange
# terms into PI(X); bits has a 254-term linear combination, 252 additions in a chain; coeffs_distinct takes edge
# coefficients to the selectors (coeffs, with a repeated signal, gives a key that does not encode its circuit: "Polynomial is
# not divisible"); gates*+0 / +1 fill / overflow the PLONK domain and gates*-2 / -1 the fflonk domain.  gates12* commit
# over 4102 and 8198 points, the first sizes with window tables; wide4096 (8191 additions) and ratio_rows8192 have domain
# 2^14.  fflonk is BN254 only, as the reference's setup constants.
PLONK_CASES = {
    **{label: CASES[label] for label in ("tiny1", "tiny2", "tiny4", "tiny7", "tiny48", "tiny64", "public0", "public2",
                                         "public17", "public300", "empty", "bits", "coeffs")},
    "coeffs_distinct": ("coeffs", BN, {"repeat": False}, True),
    **{f"gates8{e:+d}": ("gates", BN, {"k": 8, "extra": e}, True) for e in (-2, -1, 0, 1)},
    **{f"gates12{e:+d}": ("gates", BN, {"k": 12, "extra": e}, False) for e in (0, 1)},
    "wide4096": ("wide", BN, {"terms": 1 << 12}, False),
    "ratio_rows8192": ("ratio", BN, {"mode": "rows", "rows": 1 << 13}, False),
    **{label: CASES[label] for label in ("bls_bits", "bls_public17", "bls_tiny362", "bls_tiny363", "bls_ratio_rows")},
}
# keys that no witness proves: the reference's prover throws this text in round 3 (fflonk proves the nPublic = 0 keys)
PLONK_ERRORS = {"coeffs": "Polynomial is not divisible", **{label: "Evaluations.getEvaluation() out of bounds" for label in ("public0", "tiny1")}}
FFLONK_ERRORS = {"coeffs": "Polynomial is not divisible"}


@functools.lru_cache(maxsize=None)
def case(label: str) -> Circuit:
    shape, curve, params, _ = CASES[label] if label in CASES else PLONK_CASES[label]
    return SHAPES[shape](curve, 1, **params)


@functools.lru_cache(maxsize=None)
def case_zkey(label: str) -> bytes:
    circ = case(label)
    return structured_zkey(circ) if CASES[label][3] else unstructured_zkey(circ)


# --------------------------------------------------------------------------------------------------- keys
TOXIC = dict(tau=0x1234567890ABCDEF1234, alpha=0xA1FA5555, beta=0xBE7A7777)


@functools.lru_cache(maxsize=None)
def prepared_ptau(curve: int, domain: int) -> bytes:
    """A prepared powers of tau for one (curve, domain), with known toxic waste; cached for the session."""
    return SS.prepared_ptau(curve, domain, **TOXIC)


@functools.lru_cache(maxsize=None)
def plonk_zkey(label: str) -> bytes:
    """oracle.plonk.plonk_setup of the case's r1cs over plonk_ptau (structured or not, as PLONK_CASES says)."""
    from oracle import plonk as OP
    circ = case(label)
    gates, _adds, _nv, _np = OP.plonk_gates_from_r1cs(O.read_r1cs(circ.r1cs_bytes()), circ.r)
    power = max(3, (len(gates) - 1).bit_length())
    return OP.plonk_setup(circ.r1cs_bytes(), _plonk_ptau(label, power, (1 << power) + 6))


@functools.lru_cache(maxsize=None)
def fflonk_zkey(label: str) -> bytes:
    """oracle.fflonk.fflonk_setup of the case's r1cs over plonk_ptau (BN254 cases only)."""
    from oracle import fflonk as OF
    circ = case(label)
    assert circ.curve == BN, "fflonk keys are BN254 only"
    gates, _adds, _nv, _np = OF.fflonk_gates_from_r1cs(O.read_r1cs(circ.r1cs_bytes()), circ.r)
    power = max(3, (len(gates) + 1).bit_length())
    return OF.fflonk_setup(circ.r1cs_bytes(), _plonk_ptau(label, power, 9 * (1 << power) + 18))


def _plonk_ptau(label: str, power: int, n_g1: int) -> bytes:
    structured = PLONK_CASES[label][3]
    assert not structured or power <= 10, "structured keys are for domains of 1024 and below"
    return SS.plonk_ptau(case(label).curve, power, TOXIC["tau"], n_g1, structured)


def structured_zkey(circ: Circuit) -> bytes:
    assert circ.domain <= 1024, "structured keys are for domains of 1024 and below"
    return O.zkey_new(circ.r1cs_bytes(), prepared_ptau(circ.curve, circ.domain))


def section4(circ: Circuit) -> bytes:
    """zkey section 4 as zkey_new writes it: A then B entries per constraint, then one A entry per public signal, each
    coefficient times R^2 mod r (src/zkey_new.js:213-330)."""
    r = circ.r
    R2 = pow(1 << 256, 2, r)
    out = []
    for c, (la, lb, _lc) in enumerate(circ.cons):
        out += [struct.pack("<III", 0, c, s) + (v * R2 % r).to_bytes(32, "little") for s, v in la]
        out += [struct.pack("<III", 1, c, s) + (v * R2 % r).to_bytes(32, "little") for s, v in lb]
    nc = len(circ.cons)
    out += [struct.pack("<III", 0, nc + s, s) + R2.to_bytes(32, "little") for s in range(circ.n_public + 1)]
    return struct.pack("<I", len(out)) + b"".join(out)


def unstructured_zkey(circ: Circuit, seed: int = 1) -> bytes:
    """The zkey of `circ` with zkey_new's header and section 4, and pseudo-random valid points as bases and vk points."""
    ci = O.CURVES[circ.curve]
    n, nv, npub = circ.domain, circ.n_vars, circ.n_public
    g1 = lambda s, k: bytes(O.gen_points(ci.id, 1, seed * 1000003 + s, k)) if k else b""
    g2 = lambda s, k: bytes(O.gen_points(ci.id, 2, seed * 1000003 + s, k)) if k else b""
    hdr = struct.pack("<I", ci.n8q) + ci.q.to_bytes(ci.n8q, "little") + struct.pack("<I", 32) + ci.r.to_bytes(32, "little")
    hdr += struct.pack("<III", nv, npub, n)
    hdr += g1(11, 1) + g1(12, 1) + g2(13, 1) + g2(14, 1) + g1(15, 1) + g2(16, 1)
    return O.write_binfile("zkey", 1, [
        (1, struct.pack("<I", 1)), (2, hdr), (3, g1(20, npub + 1)), (4, section4(circ)),
        (5, g1(1 << 32, nv)), (6, g1(2 << 32, nv)), (7, g2(3 << 32, nv)), (8, g1(4 << 32, nv - npub - 1)),
        (9, g1(5 << 32, n)), (10, bytes(64) + struct.pack("<I", 0))])


def shuffle(zkey: bytes, seed: int) -> bytes:
    """The same key with the entries of section 4 in a seeded random order."""
    data, secs = O.read_binfile(zkey, "zkey", 2)
    p, ln = secs[4][0]
    body = np.frombuffer(data[p + 4:p + ln], np.uint8).reshape(-1, 44)
    perm = np.random.default_rng(seed).permutation(body.shape[0])
    return data[:p + 4] + body[perm].tobytes() + data[p + ln:]


def expected_abc(circ: Circuit, witness=None):
    """A.w, B.w and their product per row over the whole domain (zero rows past the constraints, and 1 * w[s] for the
    public-signal rows zkey_new appends), as Python integers."""
    w = circ.w if witness is None else witness
    r, n = circ.r, circ.domain
    A, B = [0] * n, [0] * n
    for i, (la, lb, _lc) in enumerate(circ.cons):
        A[i] = sum(v * w[s] for s, v in la) % r
        B[i] = sum(v * w[s] for s, v in lb) % r
    for s in range(circ.n_public + 1):
        A[len(circ.cons) + s] = w[s] % r
    return A, B, [a * b % r for a, b in zip(A, B)]
