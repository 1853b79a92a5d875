"""oracle/plonk.py — CPU restatement of snarkjs' PLONK prover and verifier.  TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import this module.

What it restates (reference file:line):
  * Keccak256Transcript          src/Keccak256Transcript.js:25-71 (keccak_256 = @noble/hashes sha3, FIPS-202 Keccak
                                 with the 0x01 domain byte, rate 136)
  * plonkVerify                  src/plonk_verify.js:29-421
  * plonk16Prove                 src/plonk_prove.js:47-889 with Polynomial (src/polynomial/polynomial.js:31-35, 68-93,
                                 163-184, 218-296, 592-660, 970-977), Evaluations (src/polynomial/evaluations.js:29-36)
                                 and MulZ (src/mul_z.js:20-148)
  * the PLONK zkey layout        src/zkey_utils.js:261-299, src/plonk_constants.js:1-15, src/plonk_setup.js:99-480
  * plonkSetup                   src/plonk_setup.js:36-510 (plonk_setup: from an r1cs and a prepared ptau)
  * a *synthetic* structured setup (plonk_setup_synth): same sections as plonk_setup.js writes, from directly-given
    gates and a known tau (the reference derives the gates from an r1cs and the points from a ptau file)

Pins (tests/test_oracle_plonk.py), and what is NOT pinned:
  * Keccak-256 against the published known answers ("" and "abc").
  * plonk_setup(r1cs, prepared ptau) reproduces BYTE FOR BYTE the two PLONK zkeys the reference ships — test/plonk_circuit/
    circuit.zkey (14 748 bytes) and test/circuit2/circuit.zkey (4 160 728 bytes: domain 2048, 1001 additions, 4 public
    signals): gate derivation, additions, wire maps, selector / sigma / Lagrange sections, commitments, header.  This pins the
    key layout the prover reads and everything plonk_setup_synth shares with it.
  * plonk_vk(test/plonk_circuit/circuit.zkey) == the reference's verification_key.json (header layout, Fr.w[power]).
  * a proof made here from the reference's own circuit.zkey + witness.wtns verifies with the reference's
    verification key, and stops verifying when any proof field or public signal is perturbed; the same holds for keys
    from plonk_setup_synth.  Prover and verifier restate two different reference files (plonk_prove.js /
    plonk_verify.js), so algebra slips show up as a failed verification.
  * the NTT / MSM primitives underneath are pinned byte-for-byte by the zkey sections (tests/test_oracle_golden.py).
  * the BN254 pairing the verifier ends in is pinned to the reference's hard-coded known-answer vectors
    (test/keypar_test.js via oracle/keypair.py, tests/test_oracle_keypair_kat.py).
  * the transcript's byte layout (32-byte big-endian words: Qm.x, Qm.y, ..., S3.y, the public signals, A, B, C; then
    beta -> gamma; beta, gamma, Z -> alpha; alpha, T1..T3 -> xi; xi, 6 evaluations -> v; Wxi, Wxiw -> u; keccak256
    reduced mod r) is stated a third time, independently, by the reference's current Solidity template
    templates/verifier_plonk.sol.ejs:256-360, and agrees with Transcript / _challenges below.
  * NOT pinned: the prover's bytes (the reference draws the blinders b1..b11 with Fr.random(), plonk_prove.js:246-249;
    here they are inputs) and the transcript's byte layout beyond what prover and verifier share.  The stored
    test/plonk_circuit/proof.json cannot serve: it is a stale development artifact — it is rejected by this restatement
    of the current src/plonk_verify.js, and its sibling verifier.sol differs from the current template (it hashes
    S1x twice instead of S1x,S1y and accumulates T3 twice).  PLONK prover parity is therefore "partially pinned".

Field elements are plain Python ints in [0, r) inside this file; bulk NTT / MSM go through the C++ restatement
(oracle.fr_fft, oracle.multiexp_affine), whose own pins are the zkey/ptau fixtures.  Prover: both curves; verifier: BN254
through oracle.py's pairing, BLS12-381 through oracle/pairing_bls.py.
"""
from __future__ import annotations

import struct
from typing import Dict, List, Sequence, Tuple

import numpy as np

from . import oracle as orc

# ----------------------------------------------------------------------------- Keccak-256
_RC = [0x0000000000000001, 0x0000000000008082, 0x800000000000808A, 0x8000000080008000, 0x000000000000808B,
       0x0000000080000001, 0x8000000080008081, 0x8000000000008009, 0x000000000000008A, 0x0000000000000088,
       0x0000000080008009, 0x000000008000000A, 0x000000008000808B, 0x800000000000008B, 0x8000000000008089,
       0x8000000000008003, 0x8000000000008002, 0x8000000000000080, 0x000000000000800A, 0x800000008000000A,
       0x8000000080008081, 0x8000000000008080, 0x0000000080000001, 0x8000000080008008]
_ROT = [[0, 36, 3, 41, 18], [1, 44, 10, 45, 2], [62, 6, 43, 15, 61], [28, 55, 25, 21, 56], [27, 20, 39, 8, 14]]
_M64 = (1 << 64) - 1


def _rol(x, n):
    n %= 64
    return ((x << n) | (x >> (64 - n))) & _M64 if n else x


def _keccak_f(a):
    for rc in _RC:
        c = [a[x][0] ^ a[x][1] ^ a[x][2] ^ a[x][3] ^ a[x][4] for x in range(5)]
        d = [c[(x - 1) % 5] ^ _rol(c[(x + 1) % 5], 1) for x in range(5)]
        a = [[a[x][y] ^ d[x] for y in range(5)] for x in range(5)]
        b = [[0] * 5 for _ in range(5)]
        for x in range(5):
            for y in range(5):
                b[y][(2 * x + 3 * y) % 5] = _rol(a[x][y], _ROT[x][y])
        a = [[b[x][y] ^ ((~b[(x + 1) % 5][y]) & b[(x + 2) % 5][y]) for y in range(5)] for x in range(5)]
        a[0][0] ^= rc
    return a


def keccak256(data: bytes) -> bytes:
    rate = 136
    msg = bytearray(data)
    msg.append(0x01)
    while len(msg) % rate:
        msg.append(0)
    msg[-1] |= 0x80
    a = [[0] * 5 for _ in range(5)]
    for off in range(0, len(msg), rate):
        for i in range(rate // 8):
            a[i % 5][i // 5] ^= int.from_bytes(msg[off + 8 * i:off + 8 * i + 8], "little")
        a = _keccak_f(a)
    out = b"".join(a[i % 5][i // 5].to_bytes(8, "little") for i in range(4))
    return out


# ----------------------------------------------------------------------------- transcript
class Transcript:
    """src/Keccak256Transcript.js:25-71.  Points are affine int pairs (None = infinity, written as zeros:
    build/snarkjs.js:7122-7148), scalars plain ints; both big-endian, in insertion order."""

    def __init__(self, ci: orc.CurveInfo):
        self.ci = ci
        self.data: List[bytes] = []

    def reset(self):
        self.data = []

    def add_pol(self, pt):
        n = self.ci.n8q
        self.data.append(bytes(2 * n) if pt is None else pt[0].to_bytes(n, "big") + pt[1].to_bytes(n, "big"))

    def add_scalar(self, x: int):
        self.data.append((x % self.ci.r).to_bytes(self.ci.n8r, "big"))

    def challenge(self) -> int:
        if not self.data:
            raise ValueError("Keccak256Transcript: No data to generate a transcript")
        return int.from_bytes(keccak256(b"".join(self.data)), "big") % self.ci.r


# ----------------------------------------------------------------------------- small helpers
def _g1(obj):
    """G1.fromObject of a JSON point [x, y, z] (decimal strings); z == 0 -> infinity."""
    x, y, z = (int(v) for v in obj)
    return None if z == 0 else (x, y)


def _g1_obj(pt) -> List[str]:
    """G1.toObject + stringifyBigInts: affine [x, y, 1]; infinity is [0, 1, 0]."""
    return ["0", "1", "0"] if pt is None else [str(pt[0]), str(pt[1]), "1"]


def _g1_valid(pt) -> bool:
    return pt is None or (pt[1] * pt[1] - pt[0] ** 3 - 3) % orc.P_BN_Q == 0


def _neg(pt):
    return None if pt is None else (pt[0], (-pt[1]) % orc.P_BN_Q)


_add = orc._g1_add_int
_mul = orc._g1_mul_int


def _fr_w(ci: orc.CurveInfo, k: int) -> int:
    """Fr.w[k]: the primitive 2^k-th root of unity the reference uses (build/snarkjs.js:12866-12893)."""
    return ci.fr_from_mont(orc.fr_root(ci.id, k))


def _ints_from_mont(ci, buf) -> List[int]:
    plain = bytes(orc.batch_convert(ci.fr, False, buf))
    return [int.from_bytes(plain[i:i + 32], "little") for i in range(0, len(plain), 32)]


def _mont_from_ints(ci, xs: Sequence[int]) -> bytes:
    return bytes(orc.batch_convert(ci.fr, True, b"".join(int(x).to_bytes(32, "little") for x in xs)))


def _ifft(ci, evals: Sequence[int]) -> List[int]:
    return _ints_from_mont(ci, orc.fr_fft(ci.id, _mont_from_ints(ci, evals), True))


def _fft(ci, coefs: Sequence[int]) -> List[int]:
    return _ints_from_mont(ci, orc.fr_fft(ci.id, _mont_from_ints(ci, coefs), False))


def _commit(ci, ptau: bytes, coefs: Sequence[int]):
    """Polynomial.multiExponentiation (polynomial.js:970-977): MSM over the first len(coefs) PTau points."""
    n = len(coefs)
    sc = b"".join(int(c).to_bytes(32, "little") for c in coefs)
    jac = orc.multiexp_affine(ci.id, 1, ptau[:n * 2 * ci.n8q], sc)
    return ci.g1_from_affine_bytes(orc.g_to_affine(ci.id, 1, jac)[:2 * ci.n8q])


def _degree(c: Sequence[int]) -> int:
    for i in range(len(c) - 1, 0, -1):
        if c[i]:
            return i
    return 0


def _evaluate(c: Sequence[int], x: int, r: int) -> int:
    res = 0
    for i in range(_degree(c), -1, -1):          # polynomial.js:174-184
        res = (c[i] + res * x) % r
    return res


def _blind(c: List[int], bf: Sequence[int], r: int) -> List[int]:
    """polynomial.js:68-93: append len(bf) coefficients; c[len+i] += bf[i], c[i] -= bf[i]."""
    n = len(c)
    out = list(c) + [0] * len(bf)
    for i, b in enumerate(bf):
        out[n + i] = (out[n + i] + b) % r
        out[i] = (out[i] - b) % r
    return out


def _poly_acc(dst: List[int], src: Sequence[int], k: int, r: int, sign: int = 1):
    """dst += sign * k * src, growing dst if src is longer (polynomial.js:218-276)."""
    if len(src) > len(dst):
        dst.extend([0] * (len(src) - len(dst)))
    for i, s in enumerate(src):
        dst[i] = (dst[i] + sign * k * s) % r


def _div_zerofier1(c: List[int], beta: int, r: int) -> List[int]:
    """polynomial.js:617-660 with n = 1: divide by (X - beta) in place; the top coefficient must come out zero."""
    inv = pow(beta, -1, r)
    out = list(c)
    out[0] = (-inv * out[0]) % r
    for i in range(1, len(out)):
        out[i] = (out[i - 1] - out[i]) * inv % r
        if i > len(out) - 2 and out[i]:
            raise ValueError("Polynomial is not divisible")
    return out


# ----------------------------------------------------------------------------- zkey reader (plonk)
def read_plonk_zkey(zkey) -> Dict:
    data, secs = orc.read_binfile(zkey, "zkey", 2)
    zk = orc.read_zkey_header(data, secs)
    if zk["protocol"] != "plonk":
        raise ValueError("zkey file is not plonk")                                   # plonk_prove.js:58-60
    ci = orc.curve_from_q(zk["q"])
    zk["ci"] = ci
    zk["data"], zk["secs"] = data, secs
    return zk


def plonk_vk(zkey) -> Dict:
    """src/zkey_export_verificationkey.js (plonk branch): the verification key as the JSON-shaped dict."""
    zk = read_plonk_zkey(zkey)
    ci = zk["ci"]
    vk = {"protocol": "plonk", "curve": ci.name, "nPublic": zk["nPublic"], "power": zk["power"],
          "k1": str(ci.fr_from_mont(zk["k1"])), "k2": str(ci.fr_from_mont(zk["k2"]))}
    for name in ("Qm", "Ql", "Qr", "Qo", "Qc", "S1", "S2", "S3"):
        vk[name] = _g1_obj(ci.g1_from_affine_bytes(zk[name]))
    x2 = ci.g2_from_affine_bytes(zk["X_2"])
    vk["X_2"] = [[str(x2[0][0]), str(x2[0][1])], [str(x2[1][0]), str(x2[1][1])], ["1", "0"]]
    vk["w"] = str(_fr_w(ci, zk["power"]))
    return vk


# ----------------------------------------------------------------------------- verifier
def _challenges(ci, vk, pub: Sequence[int], pr) -> Dict:
    """plonk_verify.js:208-272"""
    t = Transcript(ci)
    for name in ("Qm", "Ql", "Qr", "Qo", "Qc", "S1", "S2", "S3"):
        t.add_pol(vk[name])
    for s in pub:
        t.add_scalar(s)
    for name in ("A", "B", "C"):
        t.add_pol(pr[name])
    ch = {"beta": t.challenge()}
    t.reset(); t.add_scalar(ch["beta"])
    ch["gamma"] = t.challenge()
    t.reset(); t.add_scalar(ch["beta"]); t.add_scalar(ch["gamma"]); t.add_pol(pr["Z"])
    ch["alpha"] = t.challenge()
    t.reset(); t.add_scalar(ch["alpha"]); t.add_pol(pr["T1"]); t.add_pol(pr["T2"]); t.add_pol(pr["T3"])
    ch["xi"] = t.challenge()
    t.reset(); t.add_scalar(ch["xi"])
    for name in ("eval_a", "eval_b", "eval_c", "eval_s1", "eval_s2", "eval_zw"):
        t.add_scalar(pr[name])
    v1 = t.challenge()
    ch["v"] = [None, v1] + [pow(v1, i, ci.r) for i in range(2, 6)]
    t.reset(); t.add_pol(pr["Wxi"]); t.add_pol(pr["Wxiw"])
    ch["u"] = t.challenge()
    return ch


def plonk_verify(vk_json: Dict, public_signals: Sequence, proof_json: Dict) -> bool:
    """src/plonk_verify.js:29-124 on JSON-shaped inputs (decimal strings)."""
    if vk_json.get("curve", "bn128") == "bn128":
        ci = orc.CURVES[orc.BN254]
        _add, _mul, _neg, _g1_valid, pairing = orc._g1_add_int, orc._g1_mul_int, globals()["_neg"], globals()["_g1_valid"], orc.pairing_product_is_one
    else:                                   # bls12381: same verifier, its own G1 arithmetic and pairing
        from . import pairing_bls as pb
        ci = orc.CURVES[orc.BLS12_381]
        _add, _mul, _neg, _g1_valid, pairing = pb.g1_add, pb.g1_mul, pb.g1_neg, pb.g1_valid, pb.pairing_product_is_one
    r = ci.r
    pr = {k: _g1(proof_json[k]) for k in ("A", "B", "C", "Z", "T1", "T2", "T3", "Wxi", "Wxiw")}
    evals_raw = {k: int(proof_json[k]) for k in ("eval_a", "eval_b", "eval_c", "eval_s1", "eval_s2", "eval_zw")}
    vk = {k: _g1(vk_json[k]) for k in ("Qm", "Ql", "Qr", "Qo", "Qc", "S1", "S2", "S3")}
    k1, k2, power, n_public = int(vk_json["k1"]), int(vk_json["k2"]), int(vk_json["power"]), int(vk_json["nPublic"])
    x2 = vk_json["X_2"]
    X_2 = ((int(x2[0][0]), int(x2[0][1])), (int(x2[1][0]), int(x2[1][1])))
    pub = [int(s) for s in public_signals]

    if not all(_g1_valid(p) for p in pr.values()):                                      # :45-48, 175-187
        return False
    if len(pub) != n_public:                                                            # :50-53
        return False
    if not all(0 <= v < r for v in evals_raw.values()):                                 # :55-58
        return False
    if not all(0 <= s < r for s in pub):                                                # :60-63
        return False
    pr.update(evals_raw)

    ch = _challenges(ci, vk, pub, pr)
    beta, gamma, alpha, xi, v, u = ch["beta"], ch["gamma"], ch["alpha"], ch["xi"], ch["v"], ch["u"]
    # Lagrange evaluations :274-297
    xin = pow(xi, 1 << power, r)
    n = 1 << power
    zh = (xin - 1) % r
    wroot = _fr_w(ci, power)
    L = [None]
    w = 1
    for _ in range(max(1, n_public)):
        L.append(w * zh % r * pow(n * (xi - w) % r, -1, r) % r)
        w = w * wroot % r
    pi = 0
    for i, s in enumerate(pub):                                                         # :299-308
        pi = (pi - s * L[i + 1]) % r
    ea, eb, ec, es1, es2, ezw = (pr[k] for k in ("eval_a", "eval_b", "eval_c", "eval_s1", "eval_s2", "eval_zw"))
    # r0 :310-333
    e3 = (ea + beta * es1 + gamma) * (eb + beta * es2 + gamma) % r * (ec + gamma) % r * ezw % r * alpha % r
    r0 = (pi - L[1] * alpha * alpha - e3) % r
    # D :335-375
    d1 = _mul(vk["Qm"], ea * eb % r)
    d1 = _add(d1, _mul(vk["Ql"], ea)); d1 = _add(d1, _mul(vk["Qr"], eb)); d1 = _add(d1, _mul(vk["Qo"], ec))
    d1 = _add(d1, vk["Qc"])
    betaxi = beta * xi % r
    d2a = (ea + betaxi + gamma) * (eb + betaxi * k1 + gamma) % r * (ec + betaxi * k2 + gamma) % r * alpha % r
    d2b = L[1] * alpha * alpha % r
    d2 = _mul(pr["Z"], (d2a + d2b + u) % r)
    d3 = _mul(vk["S3"], (ea + beta * es1 + gamma) * (eb + beta * es2 + gamma) % r * (alpha * beta % r * ezw % r) % r)
    d4 = _add(pr["T1"], _add(_mul(pr["T2"], xin), _mul(pr["T3"], xin * xin % r)))
    d4 = _mul(d4, zh)
    D = _add(_add(_add(d1, d2), _neg(d3)), _neg(d4))
    # F :377-387
    F = D
    for pt, k in ((pr["A"], v[1]), (pr["B"], v[2]), (pr["C"], v[3]), (vk["S1"], v[4]), (vk["S2"], v[5])):
        F = _add(F, _mul(pt, k))
    # E :389-403
    e = (-r0 + v[1] * ea + v[2] * eb + v[3] * ec + v[4] * es1 + v[5] * es2 + u * ezw) % r
    E = _mul(ci.g1, e)
    # pairing :405-421
    A1 = _add(pr["Wxi"], _mul(pr["Wxiw"], u))
    B1 = _mul(pr["Wxi"], xi)
    B1 = _add(B1, _mul(pr["Wxiw"], u * xi % r * wroot % r))
    B1 = _add(_add(B1, F), _neg(E))
    if A1 is None or B1 is None:
        return A1 is None and B1 is None
    return pairing([(_neg(A1), X_2), (B1, ci.g2)])


# ----------------------------------------------------------------------------- prover
def _mulz_consts(ci):
    """src/mul_z.js:21-47 (Z1, Z2, Z3 for the four cosets of the 4n domain)."""
    r = ci.r
    w2 = _fr_w(ci, 2)
    Z1 = [0, (-1 + w2) % r, (-2) % r, (-1 - w2) % r]
    Z2 = [0, (-2 * w2) % r, 4, (2 * w2) % r]
    Z3 = [0, (2 + 2 * w2) % r, (-8) % r, (2 - 2 * w2) % r]
    return Z1, Z2, Z3


def plonk_prove(zkey, wtns, blinders: Sequence[int], return_parts: bool = False):
    """src/plonk_prove.js:47-889 with b[1..11] = blinders[0..10] (the reference draws them with Fr.random(), :246-249).
    Returns (proof dict, public signals as decimal strings) — the JSON the reference writes."""
    zk = read_plonk_zkey(zkey)
    ci: orc.CurveInfo = zk["ci"]
    r = ci.r
    data, secs = zk["data"], zk["secs"]
    wh, wbytes = orc.read_wtns(wtns)
    if wh["q"] != zk["r"]:
        raise ValueError("Curve of the witness does not match the curve of the proving key")          # :62-64
    n_vars, n_add, n_pub, n, n_cons = zk["nVars"], zk["nAdditions"], zk["nPublic"], zk["domainSize"], zk["nConstraints"]
    if wh["nWitness"] != n_vars - n_add:
        raise ValueError(f"Invalid witness length. Circuit: {n_vars}, witness: {wh['nWitness']}, {n_add}")  # :66-68
    power = zk["power"]
    b = [None] + [int(x) % r for x in blinders]
    assert len(b) == 12
    k1, k2 = ci.fr_from_mont(zk["k1"]), ci.fr_from_mont(zk["k2"])

    wit = [int.from_bytes(wbytes[i:i + 32], "little") for i in range(0, len(wbytes), 32)]
    wit[0] = 0                                                                                    # :97-99
    # additions :166-195 (factors are Montgomery, so factor * witness is plain)
    add_sec = bytes(orc.section(data, secs, 3))
    internal: List[int] = []
    n_wit = n_vars - n_add

    def get_witness(idx):                                                                         # :203-211
        if idx < n_wit:
            return wit[idx]
        if idx < n_vars:
            return internal[idx - n_wit]
        return 0

    s_sum = 8 + 64
    for i in range(n_add):
        s1, s2 = struct.unpack_from("<II", add_sec, i * s_sum)
        f1 = ci.fr_from_mont(add_sec[i * s_sum + 8:i * s_sum + 40])
        f2 = ci.fr_from_mont(add_sec[i * s_sum + 40:i * s_sum + 72])
        internal.append((f1 * get_witness(s1) + f2 * get_witness(s2)) % r)

    def sec_ints(sid, first_fe, count):
        s = orc.section(data, secs, sid)
        return _ints_from_mont(ci, bytes(s[first_fe * 32:(first_fe + count) * 32]))

    sigma_coef = [sec_ints(12, 5 * k * n, n) for k in range(3)]                                   # :115-121
    sigma_ev = [sec_ints(12, 5 * k * n + n, 4 * n) for k in range(3)]                             # :124-130
    ptau = bytes(orc.section(data, secs, 14))
    public = [wit[i] for i in range(1, n_pub + 1)]                                                # :137-140

    proof_pts: Dict[str, object] = {}
    proof_ev: Dict[str, int] = {}
    header_pts = {k: ci.g1_from_affine_bytes(zk[k]) for k in ("Qm", "Ql", "Qr", "Qo", "Qc", "S1", "S2", "S3")}

    # ---- round 1 :244-313
    maps = [np.frombuffer(bytes(orc.section(data, secs, sid)), dtype="<u4") for sid in (4, 5, 6)]
    bufA, bufB, bufC = ([get_witness(int(m[i])) for i in range(n_cons)] + [0] * (n - n_cons) for m in maps)
    cA, cB, cC = _ifft(ci, bufA), _ifft(ci, bufB), _ifft(ci, bufC)
    evA, evB, evC = (_fft(ci, c + [0] * (3 * n)) for c in (cA, cB, cC))
    pA, pB, pC = _blind(cA, [b[2], b[1]], r), _blind(cB, [b[4], b[3]], r), _blind(cC, [b[6], b[5]], r)
    for name, p in (("A", pA), ("B", pB), ("C", pC)):
        if _degree(p) >= n + 2:
            raise ValueError(f"{name} Polynomial is not well calculated")
        proof_pts[name] = _commit(ci, ptau, p)

    # ---- round 2 :315-458
    t = Transcript(ci)
    for k in ("Qm", "Ql", "Qr", "Qo", "Qc", "S1", "S2", "S3"):
        t.add_pol(header_pts[k])
    for i in range(n_pub):
        t.add_scalar(bufA[i])
    for k in ("A", "B", "C"):
        t.add_pol(proof_pts[k])
    beta = t.challenge()
    t.reset(); t.add_scalar(beta)
    gamma = t.challenge()

    wn = _fr_w(ci, power)
    num = [0] * n
    den = [0] * n
    num[0] = den[0] = 1
    w = 1
    for i in range(n):
        a_, b_, c_ = bufA[i], bufB[i], bufC[i]
        betaw = beta * w % r
        nn = (a_ + betaw + gamma) * ((b_ + k1 * betaw + gamma) * (c_ + k2 * betaw + gamma) % r) % r
        dd = (a_ + sigma_ev[0][4 * i] * beta + gamma) * ((b_ + sigma_ev[1][4 * i] * beta + gamma)
                                                         * (c_ + sigma_ev[2][4 * i] * beta + gamma) % r) % r
        num[(i + 1) % n] = num[i] * nn % r
        den[(i + 1) % n] = den[i] * dd % r
        w = w * wn % r
    bufZ = [num[i] * pow(den[i], -1, r) % r for i in range(n)]
    if bufZ[0] != 1:
        raise ValueError("Copy constraints does not match")                                       # :436-438
    cZ = _ifft(ci, bufZ)
    evZ = _fft(ci, cZ + [0] * (3 * n))
    pZ = _blind(cZ, [b[9], b[8], b[7]], r)
    if _degree(pZ) >= n + 3:
        raise ValueError("Z Polynomial is not well calculated")
    proof_pts["Z"] = _commit(ci, ptau, pZ)

    # ---- round 3 :460-684
    t.reset(); t.add_scalar(beta); t.add_scalar(gamma); t.add_pol(proof_pts["Z"])
    alpha = t.challenge()
    alpha2 = alpha * alpha % r
    if n_pub == 0:              # e4 reads L1 from a buffer of nPublic Lagrange polynomials (:503-509, 613-617; evaluations.js:39-44)
        raise ValueError("Evaluations.getEvaluation() out of bounds")
    q_ev ={name: sec_ints(sid, n, 4 * n) for name, sid in (("QM", 7), ("QL", 8), ("QR", 9), ("QO", 10), ("QC", 11))}
    lag_ev = [sec_ints(13, 5 * j * n + n, 4 * n) for j in range(n_pub)]                           # :503-509
    Z1, Z2, Z3 = _mulz_consts(ci)
    w4n = _fr_w(ci, power + 2)
    T = [0] * (4 * n)
    Tz = [0] * (4 * n)
    def mul4(a, bb, c, d, ap, bp, cp, dp, p):                                                    # mul_z.js:104-147
        a_b, a_bp, ap_b, ap_bp = a * bb % r, a * bp % r, ap * bb % r, ap * bp % r
        c_d, c_dp, cp_d, cp_dp = c * d % r, c * dp % r, cp * d % r, cp * dp % r
        rr = a_b * c_d % r
        rz = (ap_b * c_d + a_bp * c_d + a_b * cp_d + a_b * c_dp) % r
        if p:
            a1 = (ap_bp * c_d + ap_b * cp_d + ap_b * c_dp + a_bp * cp_d + a_bp * c_dp + a_b * cp_dp) % r
            a2 = (a_bp * cp_dp + ap_b * cp_dp + ap_bp * c_dp + ap_bp * cp_d) % r
            a3 = ap_bp * cp_dp % r
            rz = (rz + Z1[p] * a1 + Z2[p] * a2 + Z3[p] * a3) % r
        return rr, rz

    w = 1
    for i in range(4 * n):
        a_, b_, c_, z_ = evA[i], evB[i], evC[i], evZ[i]
        zw_ = evZ[(4 * n + 4 + i) % (4 * n)]
        qm, ql, qr_, qo, qc = q_ev["QM"][i], q_ev["QL"][i], q_ev["QR"][i], q_ev["QO"][i], q_ev["QC"][i]
        s1, s2, s3 = sigma_ev[0][i], sigma_ev[1][i], sigma_ev[2][i]
        ap = (b[2] + b[1] * w) % r
        bp = (b[4] + b[3] * w) % r
        cp = (b[6] + b[5] * w) % r
        w2 = w * w % r
        zp = (b[7] * w2 + b[8] * w + b[9]) % r
        wW = w * wn % r
        zWp = (b[7] * (wW * wW % r) + b[8] * wW + b[9]) % r
        pi = 0
        for j in range(n_pub):
            pi = (pi - lag_ev[j][i] * bufA[j]) % r
        p = i % 4
        # e1 (MulZ.mul2, mul_z.js:49-70)
        e1 = a_ * b_ % r
        e1z = (a_ * bp + ap * b_) % r
        if p:
            e1z = (e1z + Z1[p] * (ap * bp % r)) % r
        e1 = (e1 * qm + a_ * ql + b_ * qr_ + c_ * qo + pi + qc) % r
        e1z = (e1z * qm + ap * ql + bp * qr_ + cp * qo) % r
        betaw = beta * w % r
        e2, e2z = mul4((a_ + betaw + gamma) % r, (b_ + betaw * k1 + gamma) % r, (c_ + betaw * k2 + gamma) % r, z_, ap, bp, cp, zp, p)
        e3, e3z = mul4((a_ + beta * s1 + gamma) % r, (b_ + beta * s2 + gamma) % r, (c_ + beta * s3 + gamma) % r, zw_, ap, bp, cp, zWp, p)
        l1 = lag_ev[0][i]
        e4 = (z_ - 1) * l1 % r * alpha2 % r
        e4z = zp * l1 % r * alpha2 % r
        T[i] = (e1 + e2 * alpha - e3 * alpha + e4) % r
        Tz[i] = (e1z + e2z * alpha - e3z * alpha + e4z) % r
        w = w * w4n % r
    cT = _ifft(ci, T)
    # divZh :592-614
    for i in range(n):
        cT[i] = (-cT[i]) % r
    for i in range(n, 4 * n):
        cT[i] = (cT[i - n] - cT[i]) % r
        if i > 3 * n - 4 and cT[i]:
            raise ValueError("Polynomial is not divisible")
    cTz = _ifft(ci, Tz)
    cT = [(x + y) % r for x, y in zip(cT, cTz)]
    if _degree(cT) >= 3 * n + 6:
        raise ValueError("T Polynomial is not well calculated")
    T1 = cT[0:n] + [b[10]]
    T2 = cT[n:2 * n] + [b[11]]
    T2[0] = (T2[0] - b[10]) % r
    T3 = cT[2 * n:3 * n + 6]
    T3[0] = (T3[0] - b[11]) % r
    proof_pts["T1"], proof_pts["T2"], proof_pts["T3"] = _commit(ci, ptau, T1), _commit(ci, ptau, T2), _commit(ci, ptau, T3)

    # ---- round 4 :686-708
    t.reset(); t.add_scalar(alpha); t.add_pol(proof_pts["T1"]); t.add_pol(proof_pts["T2"]); t.add_pol(proof_pts["T3"])
    xi = t.challenge()
    xiw = xi * wn % r
    proof_ev["eval_a"] = _evaluate(pA, xi, r)
    proof_ev["eval_b"] = _evaluate(pB, xi, r)
    proof_ev["eval_c"] = _evaluate(pC, xi, r)
    proof_ev["eval_s1"] = _evaluate(sigma_coef[0], xi, r)
    proof_ev["eval_s2"] = _evaluate(sigma_coef[1], xi, r)
    proof_ev["eval_zw"] = _evaluate(pZ, xiw, r)

    # ---- round 5 :710-888
    t.reset(); t.add_scalar(xi)
    for k in ("eval_a", "eval_b", "eval_c", "eval_s1", "eval_s2", "eval_zw"):
        t.add_scalar(proof_ev[k])
    v1 = t.challenge()
    v = [None, v1] + [pow(v1, i, r) for i in range(2, 6)]
    q_coef = {name: sec_ints(sid, 0, n) for name, sid in (("QM", 7), ("QL", 8), ("QR", 9), ("QO", 10), ("QC", 11))}
    xin = pow(xi, n, r)
    zh = (xin - 1) % r
    L = [None]
    w = 1
    for _ in range(max(1, n_pub)):
        L.append(w * zh % r * pow(n * (xi - w) % r, -1, r) % r)
        w = w * wn % r
    eval_l1 = (xin - 1) * pow(n * (xi - 1) % r, -1, r) % r
    eval_pi = 0
    for i, s in enumerate(public):
        eval_pi = (eval_pi - s * L[i + 1]) % r
    ea, eb, ec, es1, es2, ezw = (proof_ev[k] for k in ("eval_a", "eval_b", "eval_c", "eval_s1", "eval_s2", "eval_zw"))
    betaxi = beta * xi % r
    e2 = (ea + betaxi + gamma) * (eb + betaxi * k1 + gamma) % r * (ec + betaxi * k2 + gamma) % r * alpha % r
    e3 = (ea + beta * es1 + gamma) * (eb + beta * es2 + gamma) % r * ezw % r * alpha % r
    e4 = eval_l1 * alpha2 % r
    R = [0] * (n + 6)
    _poly_acc(R, q_coef["QM"], ea * eb % r, r)
    _poly_acc(R, q_coef["QL"], ea, r)
    _poly_acc(R, q_coef["QR"], eb, r)
    _poly_acc(R, q_coef["QO"], ec, r)
    _poly_acc(R, q_coef["QC"], 1, r)
    _poly_acc(R, pZ, e2, r)
    _poly_acc(R, sigma_coef[2], e3 * beta % r, r, -1)
    _poly_acc(R, pZ, e4, r)
    tmp = [x * (xin * xin % r) % r for x in T3]
    _poly_acc(tmp, T2, xin, r)
    _poly_acc(tmp, T1, 1, r)
    tmp = [x * zh % r for x in tmp]
    _poly_acc(R, tmp, 1, r, -1)
    r0 = (eval_pi - e3 * (ec + gamma) - e4) % r
    R[0] = (R[0] + r0) % r
    Wxi = [0] * (n + 6)
    _poly_acc(Wxi, R, 1, r)
    for p_, k_ in ((pA, v[1]), (pB, v[2]), (pC, v[3]), (sigma_coef[0], v[4]), (sigma_coef[1], v[5])):
        _poly_acc(Wxi, p_, k_, r)
    Wxi[0] = (Wxi[0] - v[1] * ea - v[2] * eb - v[3] * ec - v[4] * es1 - v[5] * es2) % r
    Wxi = _div_zerofier1(Wxi, xi, r)
    Wxiw = list(pZ)
    Wxiw[0] = (Wxiw[0] - ezw) % r
    Wxiw = _div_zerofier1(Wxiw, xiw, r)
    proof_pts["Wxi"], proof_pts["Wxiw"] = _commit(ci, ptau, Wxi), _commit(ci, ptau, Wxiw)

    proof = {k: _g1_obj(proof_pts[k]) for k in ("A", "B", "C", "Z", "T1", "T2", "T3", "Wxi", "Wxiw")}
    for k in ("eval_a", "eval_b", "eval_c", "eval_s1", "eval_s2", "eval_zw"):
        proof[k] = str(proof_ev[k])
    proof["protocol"] = "plonk"
    proof["curve"] = ci.name
    pub_out = [str(s) for s in public]
    if return_parts:
        parts = {"beta": beta, "gamma": gamma, "alpha": alpha, "xi": xi, "v": v1, "bufA": bufA, "bufB": bufB, "bufC": bufC,
                 "Z": bufZ, "T": T, "Tz": Tz, "cT": cT, "pA": pA, "pB": pB, "pC": pC, "pZ": pZ, "T1": T1, "T2": T2, "T3": T3,
                 "R": R, "Wxi": Wxi, "Wxiw": Wxiw, "internal": internal}
        return proof, pub_out, parts
    return proof, pub_out


# ----------------------------------------------------------------------------- synthetic structured setup
def chain_gates(n_gates: int, seed: int = 7, r: int = orc.P_BN_R, n_pub: int = 1, with_additions: bool = True,
                deep_additions: bool = False):
    """A PLONK circuit given directly as gates (the reference derives them from an r1cs, plonk_setup.js:142-299):
    the chain x_{i+1} = x_i^2 + c with public output x_m (and, for n_pub > 1, x_0, x_1, ... as further public signals),
    plus linear 'addition' wires y_j = 3 x_j + 7 x_{j+1} and z_j = y_j + 2 y_{j+1} (the shape reduceCoefs emits,
    plonk_setup.js:176-215), so calculateAdditions is exercised with two dependency levels; deep_additions=True makes
    y_j = 3 x_j + 7 y_{j-1} instead, a dependency chain as long as the number of additions.
    Returns (gates, additions, n_vars, n_public, witness ints for the wtns file).
    gate = (sl, sr, so, qm, ql, qr, qo, qc) with plain ints; the first n_pub gates are the public-input gates
    (plonk_setup.js:285-297)."""
    n_y = max(2, n_gates // 8) if with_additions else 0
    n_z = n_y - 1 if with_additions else 0
    m = n_gates - n_pub - n_y - n_z           # chain multiplications
    assert m >= max(n_y + 1, n_pub)
    cst = (seed * 0x9E3779B97F4A7C15 + 12345) % r
    x = [(seed * 1000003 + 17) % r]
    for _ in range(m):
        x.append((x[-1] * x[-1] + cst) % r)
    # witness wires: 0 = one, 1 = x_m (public), 2..n_pub = x_0.. (public), then the remaining x_i
    wire_x = [2 + i for i in range(m)] + [1]
    wit = [1, x[m]] + x[:m]
    n_wit = len(wit)
    gates = [(s, 0, 0, 0, 1, 0, 0, 0) for s in range(1, n_pub + 1)]
    for i in range(m):
        gates.append((wire_x[i], wire_x[i], wire_x[i + 1], 1, 0, 0, (-1) % r, cst))
    additions = []
    wire_y = []
    for j in range(n_y):
        so = n_wit + len(additions)
        other = wire_y[j - 1] if (deep_additions and j) else wire_x[j + 1]
        additions.append((wire_x[j], other, 3, 7))
        gates.append((wire_x[j], other, so, 0, (-3) % r, (-7) % r, 1, 0))
        wire_y.append(so)
    for j in range(n_z):
        so = n_wit + len(additions)
        additions.append((wire_y[j], wire_y[j + 1], 1, 2))
        gates.append((wire_y[j], wire_y[j + 1], so, 0, (-1) % r, (-2) % r, 1, 0))
    assert len(gates) == n_gates
    return gates, additions, n_wit + len(additions), n_pub, wit


def plonk_setup_synth(gates, additions, n_vars: int, n_public: int, tau: int, structured: bool = True,
                      curve: int = orc.BN254) -> bytes:
    """Writes the sections plonk_setup.js:99-480 writes (3 additions, 4-6 wire maps, 7-11 selectors [coef n | evals 4n],
    12 sigmas, 13 Lagrange, 14 PTau, 2 header) for directly-given gates and a KNOWN tau, so that proofs verify.
    structured=False fills PTau with pseudo-random curve points instead (throughput / parity only)."""
    ci = orc.CURVES[curve]
    r = ci.r
    ng = len(gates)
    power = max(3, (ng - 1).bit_length())                                           # plonk_setup.js:74-76
    n = 1 << power
    wn = _fr_w(ci, power)
    k1 = 2
    while pow(k1, n, r) == 1:                                                       # getK1K2, plonk_setup.js:482-510
        k1 += 1
    k2 = k1 + 1
    while pow(k2, n, r) == 1 or pow(k2 * pow(k1, -1, r) % r, n, r) == 1:
        k2 += 1
    secs = []
    secs.append((3, b"".join(struct.pack("<II", a[0], a[1]) + ci.fr_to_mont(a[2]) + ci.fr_to_mont(a[3]) for a in additions)))
    for pos in range(3):
        secs.append((4 + pos, np.array([g[pos] for g in gates], dtype="<u4").tobytes()))

    def p4(evals: List[int]) -> Tuple[bytes, bytes]:                               # writeP4, plonk_setup.js:331-338
        coef = bytes(orc.fr_fft(ci.id, _mont_from_ints(ci, evals), True))          # Montgomery bytes throughout
        ev4 = orc.fr_fft(ci.id, coef + bytes(3 * n * 32), False)
        return coef + bytes(ev4), coef

    if structured:
        pts = _tau_powers(ci, tau, n + 6)
    else:
        pts = bytes(orc.gen_points(ci.id, 1, tau & 0xFFFFFFFF, n + 6))
    sG1 = 2 * ci.n8q
    cheap = [ci.g1_from_affine_bytes(pts[i * sG1:(i + 1) * sG1]) for i in range(8)]

    def commit_coef(coef: bytes):
        """[q(tau)]_1 for structured keys; for unstructured ones any valid point serves (the transcript only hashes it)."""
        if not structured:
            return cheap.pop()
        jac = orc.multiexp_affine(ci.id, 1, pts[:n * sG1], bytes(orc.batch_convert(ci.fr, False, coef)))
        return ci.g1_from_affine_bytes(orc.g_to_affine(ci.id, 1, jac)[:sG1])

    header_pts = {}
    for pos, (sid, name) in enumerate(((7, "Qm"), (8, "Ql"), (9, "Qr"), (10, "Qo"), (11, "Qc"))):
        payload, coef = p4([g[3 + pos] for g in gates] + [0] * (n - ng))
        secs.append((sid, payload))
        header_pts[name] = commit_coef(coef)
    # sigma, plonk_setup.js:362-438
    sigma = [0] * (3 * n)
    last: Dict[int, int] = {}
    first: Dict[int, int] = {}
    w = 1
    for i in range(n):
        for col in range(3):
            s = gates[i][col] if i < ng else 0
            p = col * n + i
            if s not in last:
                first[s] = p
            else:
                sigma[p] = last[s]
            last[s] = w if col == 0 else (w * k1 % r if col == 1 else w * k2 % r)
        w = w * wn % r
    for s, p in first.items():
        sigma[p] = last[s]
    payload = b""
    for col, name in enumerate(("S1", "S2", "S3")):
        pl, coef = p4(sigma[col * n:(col + 1) * n])
        payload += pl
        header_pts[name] = commit_coef(coef)
    secs.append((12, payload))
    # writeLs, plonk_setup.js:440-450 (joined once: appending to one bytes object is quadratic in n_public)
    secs.append((13, b"".join(p4([1 if j == i else 0 for j in range(n)])[0] for i in range(max(n_public, 1)))))
    secs.append((14, pts))
    x2 = _g2_times_gen(ci, tau) if structured else ci.g2_affine_bytes(ci.g2)
    hdr = struct.pack("<I", ci.n8q) + ci.q.to_bytes(ci.n8q, "little") + struct.pack("<I", 32) + r.to_bytes(32, "little")
    hdr += struct.pack("<IIIII", n_vars, n_public, n, len(additions), ng)
    hdr += ci.fr_to_mont(k1) + ci.fr_to_mont(k2)
    for name in ("Qm", "Ql", "Qr", "Qo", "Qc", "S1", "S2", "S3"):
        hdr += ci.g1_affine_bytes(header_pts[name])
    hdr += x2
    secs = [(1, struct.pack("<I", 2)), (2, hdr)] + secs
    return orc.write_binfile("zkey", 1, secs)


def _tau_powers(ci, tau: int, count: int) -> bytes:
    """tau^i * G1 for i < count as affine Montgomery bytes."""
    g = orc.g_from_affine(ci.id, 1, ci.g1_affine_bytes(ci.g1))
    out = bytearray()
    t = 1
    jac = []
    for _ in range(count):
        jac.append(orc.g_times(ci.id, 1, g, t.to_bytes(32, "little")))
        t = t * tau % ci.r
    aff = orc.batch_to_affine(ci.id, 1, b"".join(jac))
    out += bytes(aff)
    return bytes(out)


def _g2_times_gen(ci, k: int) -> bytes:
    g = orc.g_from_affine(ci.id, 2, ci.g2_affine_bytes(ci.g2))
    jac = orc.g_times(ci.id, 2, g, (k % ci.r).to_bytes(32, "little"))
    return bytes(orc.g_to_affine(ci.id, 2, jac))[:4 * ci.n8q]


def wtns_bytes(wit: Sequence[int], r: int = orc.P_BN_R) -> bytes:
    """wtns container (src/wtns_utils.js:24-60)."""
    hdr = struct.pack("<I", 32) + r.to_bytes(32, "little") + struct.pack("<I", len(wit))
    return orc.write_binfile("wtns", 2, [(1, hdr), (2, b"".join(int(x).to_bytes(32, "little") for x in wit))])


# ----------------------------------------------------------------------------- plonk setup from an r1cs and a prepared ptau
def plonk_gates_from_r1cs(r1: Dict, r: int):
    """processConstraints (src/plonk_setup.js:142-299): r1cs constraints -> PLONK gates (sl, sr, so, qm, ql, qr, qo, qc) and
    additions, including the reference's behaviour on JavaScript objects: linear combinations are keyed by signal (a repeated
    signal overwrites), iterate in ascending signal order, and a zero coefficient is never dropped (`x == 0n` is false for the
    byte-array field elements, :147-149, 189-191)."""
    n_pub = r1["nOutputs"] + r1["nPubInputs"]
    state = {"nvars": r1["nVars"]}
    gates, additions = [], []

    def as_lc(terms):
        return {int(s): int(v) % r for s, v in terms}

    def lc_type(lc):                                                                 # :258-274
        n = sum(1 for s in lc if s != 0)
        if n > 0:
            return str(n)
        return "k" if 0 in lc else "0"

    def join(lc1, k, lc2):                                                          # :151-173
        res = {}
        for s in sorted(lc1):
            res[s] = (res.get(s, 0) + k * lc1[s]) % r
        for s in sorted(lc2):
            res[s] = (res.get(s, 0) - lc2[s]) % r
        return res

    def reduce_coefs(lc, max_c):                                                    # :175-220
        k = 0
        cs = []
        for s in sorted(lc):
            if s == 0:
                k = (k + lc[s]) % r
            else:
                cs.append([s, lc[s]])
        while len(cs) > max_c:
            c1, c2 = cs.pop(0), cs.pop(0)
            so = state["nvars"]
            state["nvars"] += 1
            gates.append((c1[0], c2[0], so, 0, (-c1[1]) % r, (-c2[1]) % r, 1, 0))
            additions.append((c1[0], c2[0], c1[1], c2[1]))
            cs.append([so, 1])
        ss = [c[0] for c in cs] + [0] * (max_c - len(cs))
        cf = [c[1] for c in cs] + [0] * (max_c - len(cs))
        return k, ss, cf

    def add_sum(lc):                                                                # :222-233
        k, ss, cf = reduce_coefs(lc, 3)
        gates.append((ss[0], ss[1], ss[2], 0, cf[0], cf[1], cf[2], k))

    def add_mul(la, lb, lc):                                                        # :235-256
        ka, sa, ca = reduce_coefs(la, 1)
        kb, sb_, cb = reduce_coefs(lb, 1)
        kc, sc, cc = reduce_coefs(lc, 1)
        gates.append((sa[0], sb_[0], sc[0], ca[0] * cb[0] % r, ca[0] * kb % r, ka * cb[0] % r, (-cc[0]) % r, (ka * kb - kc) % r))

    for s in range(1, n_pub + 1):                                                   # :285-297
        gates.append((s, 0, 0, 0, 1, 0, 0, 0))
    for la, lb, lc in r1["constraints"]:                                            # :276-283, 299-302
        la, lb, lc = as_lc(la), as_lc(lb), as_lc(lc)
        ta, tb = lc_type(la), lc_type(lb)
        if ta == "0" or tb == "0":
            add_sum(lc)
        elif ta == "k":
            add_sum(join(lb, la[0], lc))
        elif tb == "k":
            add_sum(join(la, lb[0], lc))
        else:
            add_mul(la, lb, lc)
    return gates, additions, state["nvars"], n_pub


def plonk_setup(r1cs, ptau) -> bytes:
    """src/plonk_setup.js:36-480 from an r1cs and a prepared ptau: the zkey the reference writes, byte for byte (sections in the
    reference's order 3..14, 1, 2).  Pinned by tests/test_oracle_plonk.py against test/plonk_circuit/circuit.zkey."""
    r1 = orc.read_r1cs(r1cs)
    pdata, psecs = orc.read_binfile(ptau, "ptau", 1)
    ph = orc.read_ptau_header(pdata, psecs)
    ci = orc.curve_from_q(ph["q"])
    r = ci.r
    if r1["prime"] != r:
        raise ValueError("r1cs curve does not match powers of tau ceremony curve")
    gates, additions, n_vars, n_public = plonk_gates_from_r1cs(r1, r)
    ng = len(gates)
    power = max(3, (ng - 1).bit_length())                                           # :74-76
    if power > ph["power"]:
        raise ValueError("circuit too big for this power of tau ceremony")
    if 12 not in psecs:
        raise ValueError("Powers of tau is not prepared.")
    n = 1 << power
    sG1, sG2 = 2 * ci.n8q, 4 * ci.n8q

    def psec(sid, lo, hi):
        p, _ = psecs[sid][0]
        return bytes(pdata[p + lo:p + hi])

    lpoints = psec(12, (n - 1) * sG1, (2 * n - 1) * sG1)                            # :86-88
    wn = _fr_w(ci, power)
    k1 = 2
    while pow(k1, n, r) == 1:                                                       # getK1K2 :482-503 (membership of <w> is k^n == 1)
        k1 += 1
    k2 = k1 + 1
    while pow(k2, n, r) == 1 or pow(k2 * pow(k1, -1, r) % r, n, r) == 1:
        k2 += 1
    secs = [(3, b"".join(struct.pack("<II", a[0], a[1]) + ci.fr_to_mont(a[2]) + ci.fr_to_mont(a[3]) for a in additions))]
    for pos in range(3):
        secs.append((4 + pos, np.array([g[pos] for g in gates], dtype="<u4").tobytes()))

    def p4(evals_mont: bytes) -> bytes:                                             # writeP4 :331-338
        coef = bytes(orc.fr_fft(ci.id, evals_mont, True))
        return coef + bytes(orc.fr_fft(ci.id, coef + bytes(3 * n * 32), False))

    def commit_evals(evals_mont: bytes):                                            # multiExpAffine(LPoints, fromMontgomery(Q)) :326-329
        jac = orc.multiexp_affine(ci.id, 1, lpoints, bytes(orc.batch_convert(ci.fr, False, evals_mont)))
        return bytes(orc.g_to_affine(ci.id, 1, jac))[:sG1]

    vk = {}
    for pos, (sid, name) in enumerate(((7, "Qm"), (8, "Ql"), (9, "Qr"), (10, "Qo"), (11, "Qc"))):
        ev = _mont_from_ints(ci, [g[3 + pos] for g in gates] + [0] * (n - ng))
        secs.append((sid, p4(ev)))
        vk[name] = commit_evals(ev)
    sigma = [0] * (3 * n)                                                           # writeSigma :362-438
    last: Dict[int, int] = {}
    first: Dict[int, int] = {}
    w = 1
    for i in range(n):
        for col in range(3):
            s = gates[i][col] if i < ng else 0
            p = col * n + i
            if s not in last:
                first[s] = p
            else:
                sigma[p] = last[s]
            last[s] = w if col == 0 else (w * k1 % r if col == 1 else w * k2 % r)
        w = w * wn % r
    for s, p in first.items():
        sigma[p] = last[s]
    payload = b""
    for col, name in enumerate(("S1", "S2", "S3")):
        ev = _mont_from_ints(ci, sigma[col * n:(col + 1) * n])
        payload += p4(ev)
        vk[name] = commit_evals(ev)
    secs.append((12, payload))
    secs.append((13, b"".join(p4(_mont_from_ints(ci, [1 if j == i else 0 for j in range(n)])) for i in range(max(n_public, 1)))))
    secs.append((14, psec(2, 0, (n + 6) * sG1)))                                    # :122-127
    hdr = struct.pack("<I", ci.n8q) + ci.q.to_bytes(ci.n8q, "little") + struct.pack("<I", 32) + r.to_bytes(32, "little")
    hdr += struct.pack("<IIIII", n_vars, n_public, n, len(additions), ng)
    hdr += ci.fr_to_mont(k1) + ci.fr_to_mont(k2)
    for name in ("Qm", "Ql", "Qr", "Qo", "Qc", "S1", "S2", "S3"):
        hdr += vk[name]
    hdr += psec(3, sG2, 2 * sG2)                                                    # X_2 = tau * G2 (:477-479)
    return orc.write_binfile("zkey", 1, secs + [(1, struct.pack("<I", 2)), (2, hdr)])
