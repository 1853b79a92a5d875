"""oracle/fflonk.py — CPU restatement of snarkjs' fflonk prover and verifier.  TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import this module.

What it restates (reference file:line):
  * fflonkProve                  src/fflonk_prove.js:51-1286 (rounds 1-5, getMontgomeryBatchedInverse :1182-1285)
  * CPolynomial                  src/polynomial/cpolynomial.js:29-82
  * Polynomial helpers           src/polynomial/polynomial.js: divByZerofier :617-660, divBy :341-360,
                                 lagrangePolynomialInterpolation :896-930, zerofierPolynomial :932-948
  * fflonkVerify                 src/fflonk_verify.js:29-597
  * the fflonk zkey layout       src/zkey_utils.js:301-339, src/fflonk_constants.js:27-44
  * fflonkSetup                  src/fflonk_setup.js:59-559, src/r1cs_constraint_processor.js:24-200 (fflonk_setup)

Pins (tests/test_oracle_fflonk.py): fflonk_setup(r1cs, ptau) reproduces test/fflonk/circuit.zkey BYTE FOR BYTE (593 092 bytes:
gate derivation with 100 additions, selectors, sigmas, Lagrange, PTau, C0, header), which pins the key layout the prover
reads; fflonk_vk(test/fflonk/circuit.zkey) equals the reference's circuit_vk.json; a proof
made here from the reference's circuit.zkey + witness.wtns verifies against that verification key and public.json, and
stops verifying when a commitment, an evaluation or the public signal is perturbed.  Prover and verifier restate two
different reference files.  The reference ships no fflonk proof and draws its blinders at random (:321-324), so the
prover's bytes are not pinned directly: "partially pinned", as oracle/plonk.py.

Field elements are plain ints in [0, r); bulk NTT / MSM go through the C++ restatement.  BN254 only (pairing: oracle.py's,
pinned to the reference's known-answer vectors by tests/test_oracle_keypair_kat.py).
"""
from __future__ import annotations

import struct
from typing import Dict, List, Sequence

import numpy as np

from . import oracle as orc
from .plonk import (Transcript, _add, _blind, _commit, _degree, _evaluate, _fft, _fr_w, _g1, _g1_obj, _g1_valid, _ifft,
                    _ints_from_mont, _mul, _neg)

EVAL_NAMES = ("ql", "qr", "qm", "qo", "qc", "s1", "s2", "s3", "a", "b", "c", "z", "zw", "t1w", "t2w")


# ----------------------------------------------------------------------------- polynomial helpers (int lists)
def _div_zerofier(c: List[int], n: int, beta: int, r: int) -> List[int]:
    """polynomial.js:617-660: in-place division by (X^n - beta); the top n coefficients must come out zero."""
    inv = pow(beta, -1, r)
    out = list(c)
    for i in range(min(n, len(out))):
        out[i] = (-inv * out[i]) % r
    for i in range(n, len(out)):
        out[i] = (out[i - n] - out[i]) * inv % r
        if i > len(out) - n - 1 and out[i]:
            raise ValueError("Polynomial is not divisible")
    return out


def _padd(a: List[int], b: Sequence[int], r: int, k: int = 1) -> List[int]:
    """Polynomial.add / sub (k = -1) with the reference's length rule: the result has the longer length."""
    out = list(a) + [0] * max(0, len(b) - len(a))
    for i, x in enumerate(b):
        out[i] = (out[i] + k * x) % r
    return out


def _cpoly(polys: Sequence[Sequence[int]]) -> List[int]:
    """CPolynomial.getPolynomial (cpolynomial.js:52-72): P_0(X^n) + X P_1(X^n) + ...; power-of-two buffer length."""
    n = len(polys)
    degs = [_degree(p) for p in polys]
    max_degree = max(d * n + j for j, d in enumerate(degs))
    length = 1 << ((max_degree - 1).bit_length())          # 2 ** (log2(maxDegree - 1) + 1)
    out = [0] * length
    for j, p in enumerate(polys):
        for i in range(min(degs[j] + 1, max_degree)):
            if i * n + j < length:
                out[i * n + j] = p[i]
    return out


def _interpolate(xs: Sequence[int], ys: Sequence[int], r: int) -> List[int]:
    """Polynomial.lagrangePolynomialInterpolation (:896-930); result has len(xs) coefficients."""
    m = len(xs)
    res = [0] * m
    for i in range(m):
        basis = [1]
        for j in range(m):
            if j == i:
                continue
            nxt = [0] * (len(basis) + 1)                   # basis * (X - xs[j])
            for k, c in enumerate(basis):
                nxt[k] = (nxt[k] - c * xs[j]) % r
                nxt[k + 1] = (nxt[k + 1] + c) % r
            basis = nxt
        den = _evaluate(basis, xs[i], r)
        f = ys[i] * pow(den, -1, r) % r
        for k, c in enumerate(basis):
            res[k] = (res[k] + c * f) % r
    return res


def _zerofier(xs: Sequence[int], r: int) -> List[int]:
    p = [1]
    for x in xs:
        nxt = [0] * (len(p) + 1)
        for k, c in enumerate(p):
            nxt[k] = (nxt[k] - c * x) % r
            nxt[k + 1] = (nxt[k + 1] + c) % r
        p = nxt
    return p


# ----------------------------------------------------------------------------- zkey
def read_fflonk_zkey(zkey) -> Dict:
    data, secs = orc.read_binfile(zkey, "zkey", 2)
    zk = orc.read_zkey_header(data, secs)
    if zk["protocol"] != "fflonk":
        raise ValueError("zkey file is not fflonk")                                  # fflonk_prove.js:71-73
    zk["ci"] = orc.curve_from_q(zk["q"])
    zk["data"], zk["secs"] = data, secs
    return zk


def fflonk_vk(zkey) -> Dict:
    """src/zkey_export_verificationkey.js (fflonk branch)."""
    zk = read_fflonk_zkey(zkey)
    ci = zk["ci"]
    x2 = ci.g2_from_affine_bytes(zk["X_2"])
    vk = {"protocol": "fflonk", "curve": ci.name, "nPublic": zk["nPublic"], "power": zk["power"],
          "k1": str(ci.fr_from_mont(zk["k1"])), "k2": str(ci.fr_from_mont(zk["k2"])),
          "w": str(_fr_w(ci, zk["power"]))}
    for name in ("w3", "w4", "w8", "wr"):
        vk[name] = str(ci.fr_from_mont(zk[name]))
    vk["X_2"] = [[str(x2[0][0]), str(x2[0][1])], [str(x2[1][0]), str(x2[1][1])], ["1", "0"]]
    vk["C0"] = _g1_obj(ci.g1_from_affine_bytes(zk["C0"]))
    return vk


# ----------------------------------------------------------------------------- shared: roots of the opening sets
def _roots(r: int, xi_seed: int, w3: int, w4: int, w8: int, wr: int):
    """fflonk_prove.js:843-897 / fflonk_verify.js:246-300"""
    seed2 = xi_seed * xi_seed % r
    h0 = seed2 * xi_seed % r
    S0 = [h0 * pow(w8, i, r) % r for i in range(8)]
    h1 = h0 * h0 % r
    S1 = [h1 * pow(w4, i, r) % r for i in range(4)]
    h2 = h1 * seed2 % r
    S2 = [h2, h2 * w3 % r, h2 * w3 % r * w3 % r]
    h3 = h2 * wr % r
    S2p = [h3, h3 * w3 % r, h3 * w3 % r * w3 % r]
    xi = h2 * h2 % r * h2 % r
    return S0, S1, S2, S2p, xi


# ----------------------------------------------------------------------------- prover
def fflonk_prove(zkey, wtns, blinders: Sequence[int], return_parts: bool = False):
    """src/fflonk_prove.js:51-267 with b[1..9] = blinders[0..8] as field values (the reference draws Fr.random(), :321-324).
    b1..b6 enter as *raw Montgomery bytes written into the plain evaluation buffers* (:375-380), i.e. the evaluation is
    b*R mod r; b7..b9 are used as field elements."""
    zk = read_fflonk_zkey(zkey)
    ci: orc.CurveInfo = zk["ci"]
    r = ci.r
    data, secs = zk["data"], zk["secs"]
    wh, wbytes = orc.read_wtns(wtns)
    if wh["q"] != zk["r"]:
        raise ValueError("Curve of the witness does not match the curve of the proving key")
    n_vars, n_add, n_pub, n, n_cons, power = zk["nVars"], zk["nAdditions"], zk["nPublic"], zk["domainSize"], zk["nConstraints"], zk["power"]
    if wh["nWitness"] != n_vars - n_add:
        raise ValueError(f"Invalid witness length. Circuit: {n_vars}, witness: {wh['nWitness']}, {n_add}")
    b = [None] + [int(x) % r for x in blinders]
    assert len(b) == 10
    k1, k2 = ci.fr_from_mont(zk["k1"]), ci.fr_from_mont(zk["k2"])
    w3, w4, w8, wr = (ci.fr_from_mont(zk[k]) for k in ("w3", "w4", "w8", "wr"))
    wn = _fr_w(ci, power)

    wit = [int.from_bytes(wbytes[i:i + 32], "little") for i in range(0, len(wbytes), 32)]
    wit[0] = 0
    add_sec = bytes(orc.section(data, secs, 3))
    internal: List[int] = []
    n_wit = n_vars - n_add

    def get_witness(idx):
        if idx < n_wit:
            return wit[idx]
        if idx < n_vars:
            return internal[idx - n_wit]
        return 0

    for i in range(n_add):
        s1, s2 = struct.unpack_from("<II", add_sec, i * 72)
        f1 = ci.fr_from_mont(add_sec[i * 72 + 8:i * 72 + 40])
        f2 = ci.fr_from_mont(add_sec[i * 72 + 40:i * 72 + 72])
        internal.append((f1 * get_witness(s1) + f2 * get_witness(s2)) % r)

    def sec_ints(sid, first_fe, count):
        s = orc.section(data, secs, sid)
        return _ints_from_mont(ci, bytes(s[first_fe * 32:(first_fe + count) * 32]))

    sigma_coef = [sec_ints(12 + k, 0, n) for k in range(3)]
    sigma_ev = [sec_ints(12 + k, n, 4 * n) for k in range(3)]
    ptau = bytes(orc.section(data, secs, 16))
    ptau += bytes(16 * n * 2 * ci.n8q - len(ptau))        # the reference reserves 16n points, zeros past 9n + 18 (:164-169)
    c0_point = ci.g1_from_affine_bytes(zk["C0"])

    # ---- round 1 (:319-520)
    maps = [np.frombuffer(bytes(orc.section(data, secs, sid)), dtype="<u4") for sid in (4, 5, 6)]
    bufs = [[get_witness(int(m[i])) for i in range(n_cons)] + [0] * (n - n_cons) for m in maps]
    for j in range(3):                                                               # :375-380
        bufs[j][n - 2] = b[2 * j + 1] * ci.Rr % r
        bufs[j][n - 1] = b[2 * j + 2] * ci.Rr % r
    bufA, bufB, bufC = bufs
    pA, pB, pC = _ifft(ci, bufA), _ifft(ci, bufB), _ifft(ci, bufC)
    evA, evB, evC = (_fft(ci, c + [0] * (3 * n)) for c in (pA, pB, pC))
    q_ev = {name: sec_ints(sid, n, 4 * n) for name, sid in (("QL", 7), ("QR", 8), ("QM", 9), ("QO", 10), ("QC", 11))}
    lag_ev = [sec_ints(15, 5 * j * n + n, 4 * n) for j in range(max(n_pub, 1))]
    T0 = [0] * (4 * n)
    for i in range(4 * n):
        a_, b_, c_ = evA[i], evB[i], evC[i]
        pi = 0
        for j in range(n_pub):
            pi = (pi - lag_ev[j][i] * bufA[j]) % r
        T0[i] = (a_ * q_ev["QL"][i] + b_ * q_ev["QR"][i] + a_ * b_ % r * q_ev["QM"][i] + c_ * q_ev["QO"][i] + q_ev["QC"][i] + pi) % r
    pT0 = _div_zerofier(_ifft(ci, T0), n, 1, r)
    if _degree(pT0) >= 2 * n - 2:
        raise ValueError("T0 Polynomial is not well calculated")
    C1 = _cpoly([pA, pB, pC, pT0])
    if _degree(C1) >= 8 * n - 8:
        raise ValueError("C1 Polynomial is not well calculated")
    pts = {"C1": _commit(ci, ptau, C1)}

    # ---- round 2 (:522-830)
    t = Transcript(ci)
    t.add_pol(c0_point)
    for i in range(n_pub):
        t.add_scalar(bufA[i])
    t.add_pol(pts["C1"])
    beta = t.challenge()
    t.reset(); t.add_scalar(beta)
    gamma = t.challenge()
    num = [0] * n
    den = [0] * n
    num[0] = den[0] = 1
    w = 1
    for i in range(n):
        betaw = beta * w % r
        nn = (bufA[i] + betaw + gamma) * ((bufB[i] + k1 * betaw + gamma) * (bufC[i] + k2 * betaw + gamma) % r) % r
        dd = (bufA[i] + beta * sigma_ev[0][4 * i] + gamma) * ((bufB[i] + beta * sigma_ev[1][4 * i] + gamma)
                                                              * (bufC[i] + beta * sigma_ev[2][4 * i] + gamma) % r) % r
        num[(i + 1) % n] = num[i] * nn % r
        den[(i + 1) % n] = den[i] * dd % r
        w = w * wn % r
    bufZ = [num[i] * pow(den[i], -1, r) % r for i in range(n)]
    if bufZ[0] != 1:
        raise ValueError("Copy constraints does not match")
    cZ = _ifft(ci, bufZ)
    evZ = _fft(ci, cZ + [0] * (3 * n))
    pZ = _blind(cZ, [b[9], b[8], b[7]], r)
    if _degree(pZ) >= n + 3:
        raise ValueError("Z Polynomial is not well calculated")
    # T1 (:667-718) on the 2n domain
    w2n = _fr_w(ci, power + 1)
    T1 = [0] * (2 * n)
    T1z = [0] * (2 * n)
    om = 1
    for i in range(2 * n):
        zp = (b[7] * om % r * om + b[8] * om + b[9]) % r
        l1 = lag_ev[0][2 * i]
        T1[i] = (evZ[2 * i] - 1) * l1 % r
        T1z[i] = zp * l1 % r
        om = om * w2n % r
    pT1 = _padd(_div_zerofier(_ifft(ci, T1), n, 1, r), _ifft(ci, T1z), r)
    if _degree(pT1) >= n + 2:
        raise ValueError("T1 Polynomial is not well calculated")
    # T2 (:720-815) on the 4n domain
    w4n = _fr_w(ci, power + 2)
    T2 = [0] * (4 * n)
    T2z = [0] * (4 * n)
    om = 1
    for i in range(4 * n):
        omW = om * wn % r
        zp = (b[7] * om % r * om + b[8] * om + b[9]) % r
        zWp = (b[7] * omW % r * omW + b[8] * omW + b[9]) % r
        a_, b_, c_ = evA[i], evB[i], evC[i]
        betaX = beta * om % r
        e1c = (a_ + betaX + gamma) * (b_ + betaX * k1 + gamma) % r * (c_ + betaX * k2 + gamma) % r
        e2c = (a_ + beta * sigma_ev[0][i] + gamma) * (b_ + beta * sigma_ev[1][i] + gamma) % r * (c_ + beta * sigma_ev[2][i] + gamma) % r
        T2[i] = (e1c * evZ[i] - e2c * evZ[(i + 4) % (4 * n)]) % r
        T2z[i] = (e1c * zp - e2c * zWp) % r
        om = om * w4n % r
    pT2 = _padd(_div_zerofier(_ifft(ci, T2), n, 1, r), _ifft(ci, T2z), r)
    if _degree(pT2) >= 3 * n:
        raise ValueError("T2 Polynomial is not well calculated")
    C2 = _cpoly([pZ, pT1, pT2])
    if _degree(C2) >= 9 * n:
        raise ValueError("C2 Polynomial is not well calculated")
    pts["C2"] = _commit(ci, ptau, C2)

    # ---- round 3 (:832-931)
    t.reset(); t.add_scalar(gamma); t.add_pol(pts["C2"])
    xi_seed = t.challenge()
    S0, S1, S2, S2p, xi = _roots(r, xi_seed, w3, w4, w8, wr)
    q_coef = {name: sec_ints(sid, 0, n) for name, sid in (("ql", 7), ("qr", 8), ("qm", 9), ("qo", 10), ("qc", 11))}
    ev: Dict[str, int] = {k: _evaluate(q_coef[k], xi, r) for k in ("ql", "qr", "qm", "qo", "qc")}
    ev["s1"], ev["s2"], ev["s3"] = (_evaluate(sigma_coef[k], xi, r) for k in range(3))
    ev["a"], ev["b"], ev["c"] = _evaluate(pA, xi, r), _evaluate(pB, xi, r), _evaluate(pC, xi, r)
    ev["z"] = _evaluate(pZ, xi, r)
    xiw = xi * wn % r
    ev["zw"], ev["t1w"], ev["t2w"] = _evaluate(pZ, xiw, r), _evaluate(pT1, xiw, r), _evaluate(pT2, xiw, r)

    # ---- round 4 (:933-1057)
    t.reset(); t.add_scalar(xi_seed)
    for k in EVAL_NAMES:
        t.add_scalar(ev[k])
    alpha = t.challenge()
    C0 = sec_ints(17, 0, 8 * n)
    R0 = _interpolate(S0, [_evaluate(C0, x, r) for x in S0], r)
    R1 = _interpolate(S1, [_evaluate(C1, x, r) for x in S1], r)
    R2 = _interpolate(S2 + S2p, [_evaluate(C2, x, r) for x in S2 + S2p], r)
    F = _div_zerofier(_padd(C0, R0, r, -1), 8, xi, r)
    f2 = _div_zerofier([x * alpha % r for x in _padd(C1, R1, r, -1)], 4, xi, r)
    f3 = [x * alpha % r * alpha % r for x in _padd(C2, R2, r, -1)]
    f3 = _div_zerofier(_div_zerofier(f3, 3, xi, r), 3, xiw, r)
    F = _padd(_padd(F, f2, r), f3, r)
    if _degree(F) >= 9 * n - 6:
        raise ValueError("F Polynomial is not well calculated")
    pts["W1"] = _commit(ci, ptau, F)

    # ---- round 5 (:1059-1180)
    t.reset(); t.add_scalar(alpha); t.add_pol(pts["W1"])
    y = t.challenge()
    mulL0 = 1
    for x in S0:
        mulL0 = mulL0 * (y - x) % r
    mulL1 = 1
    for x in S1:
        mulL1 = mulL1 * (y - x) % r
    mulL2 = 1
    for x in S2 + S2p:
        mulL2 = mulL2 * (y - x) % r
    preL0 = mulL1 * mulL2 % r
    preL1 = alpha * mulL0 % r * mulL2 % r
    preL2 = alpha * alpha % r * mulL0 % r * mulL1 % r
    to_inverse: Dict[str, int] = {"denH1": mulL1, "denH2": mulL2}                   # insertion order matters only for the product
    L = list(C0)
    L[0] = (L[0] - _evaluate(R0, y, r)) % r
    L = [x * preL0 % r for x in L]
    l2 = list(C1)
    l2[0] = (l2[0] - _evaluate(R1, y, r)) % r
    l3 = list(C2)
    l3[0] = (l3[0] - _evaluate(R2, y, r)) % r
    L = _padd(L, [x * preL1 % r for x in l2], r)
    L = _padd(L, [x * preL2 % r for x in l3], r)
    ZT = _zerofier(S0 + S1 + S2 + S2p, r)
    zty = _evaluate(ZT, y, r)
    L = _padd(L, [x * zty % r for x in F], r, -1)
    if _degree(L) >= 9 * n:
        raise ValueError("L Polynomial is not well calculated")
    zts2y = pow(_evaluate(_zerofier(S1 + S2 + S2p, r), y, r), -1, r)
    L = [x * zts2y % r for x in L]
    # divBy (X - y) (:341-360): synthetic division from the top; the remainder must vanish
    dA = _degree(L)
    quo = [0] * len(L)
    rem = list(L)
    for i in range(dA - 1, -1, -1):
        quo[i] = rem[i + 1]
        rem[i] = (rem[i] + quo[i] * y) % r                 # rem[i+j] -= q_i * divisor[j]; divisor = (-y, 1)
        rem[i + 1] = 0
    if _degree(rem) > 0:
        raise ValueError("Degree of L(X)/(ZTS2(y)(X-y)) remainder should be 0")
    if _degree(quo) >= 9 * n - 1:
        raise ValueError("Degree of L(X)/(ZTS2(y)(X-y)) is not correct")
    pts["W2"] = _commit(ci, ptau, quo)

    # ---- the batched inverse (:1182-1285)
    to_inverse["zh"] = (pow(xi, n, r) - 1) % r
    for name, roots in (("LiS0_", S0), ("LiS1_", S1)):
        ln = len(roots)
        den1 = ln * pow(roots[0], ln - 2, r) % r
        for i in range(ln):
            to_inverse[name + str(i + 1)] = den1 * roots[((ln - 1) * i) % ln] % r * ((y - roots[i]) % r) % r
    den1 = 3 * S2[0] % r * ((xi - xiw) % r) % r
    for i in range(3):
        to_inverse["LiS2_" + str(i + 1)] = den1 * S2[2 * i % 3] % r * ((y - S2[i]) % r) % r
    den1 = 3 * S2p[0] % r * ((xiw - xi) % r) % r
    for i in range(3):
        to_inverse["LiS2_" + str(i + 4)] = den1 * S2p[2 * i % 3] % r * ((y - S2p[i]) % r) % r
    w = 1
    for i in range(max(1, n_pub)):
        to_inverse["Li_" + str(i + 1)] = n * ((xi - w) % r) % r
        w = w * wn % r
    acc = 1
    for v in to_inverse.values():
        acc = acc * v % r
    ev["inv"] = pow(acc, -1, r)

    proof = {"polynomials": {k: _g1_obj(pts[k]) for k in ("C1", "C2", "W1", "W2")},
             "evaluations": {k: str(ev[k]) for k in EVAL_NAMES + ("inv",)},
             "protocol": "fflonk", "curve": ci.name}
    public = [str(wit[i]) for i in range(1, n_pub + 1)]
    if return_parts:
        return proof, public, {"C1": C1, "C2": C2, "F": F, "W2": quo, "beta": beta, "gamma": gamma, "xi_seed": xi_seed, "alpha": alpha, "y": y}
    return proof, public


# ----------------------------------------------------------------------------- verifier
def _li_si(roots: Sequence[int], x: int, xi: int, r: int) -> List[int]:
    """computeLagrangeLiSi, fflonk_verify.js:546-563"""
    ln = len(roots)
    num = (pow(x, ln, r) - xi) % r
    den1 = ln * pow(roots[0], ln - 2, r) % r
    return [num * pow(den1 * roots[((ln - 1) * i) % ln] % r * ((x - roots[i]) % r) % r, -1, r) % r for i in range(ln)]


def _li_s2(S2: Sequence[int], S2p: Sequence[int], x: int, xi0: int, xi1: int, r: int) -> List[int]:
    """computeLagrangeLiS2, fflonk_verify.js:565-597"""
    ln = 3
    num = (pow(x, 6, r) - (xi0 + xi1) * pow(x, ln, r) + xi0 * xi1) % r
    out = []
    for roots, d in ((S2, (xi0 - xi1) % r), (S2p, (xi1 - xi0) % r)):
        den1 = ln * roots[0] % r * d % r
        for i in range(ln):
            den = den1 * roots[(ln - 1) * i % ln] % r * ((x - roots[i]) % r) % r
            out.append(num * pow(den, -1, r) % r)
    return out


def fflonk_verify(vk_json: Dict, public_signals: Sequence, proof_json: Dict) -> bool:
    """src/fflonk_verify.js:29-137 on JSON-shaped inputs."""
    ci = orc.CURVES[orc.BN254]
    if vk_json.get("curve", "bn128") != "bn128":
        raise NotImplementedError("python pairing is BN254-only")
    r = ci.r
    pol = {k: _g1(proof_json["polynomials"][k]) for k in ("C1", "C2", "W1", "W2")}
    ev = {k: int(proof_json["evaluations"][k]) for k in EVAL_NAMES + ("inv",)}
    k1, k2, power, n_pub = int(vk_json["k1"]), int(vk_json["k2"]), int(vk_json["power"]), int(vk_json["nPublic"])
    w, w3, w4, w8, wr = (int(vk_json[k]) for k in ("w", "w3", "w4", "w8", "wr"))
    x2 = vk_json["X_2"]
    X_2 = ((int(x2[0][0]), int(x2[0][1])), (int(x2[1][0]), int(x2[1][1])))
    C0 = _g1(vk_json["C0"])
    pub = [int(s) for s in public_signals]
    if len(pub) != n_pub:
        return False
    if not all(_g1_valid(p) for p in list(pol.values()) + [C0]):
        return False
    if not all(0 <= ev[k] < r for k in EVAL_NAMES) or not all(0 <= s < r for s in pub):
        return False
    # challenges (:221-338)
    t = Transcript(ci)
    t.add_pol(C0)
    for s in pub:
        t.add_scalar(s)
    t.add_pol(pol["C1"])
    beta = t.challenge()
    t.reset(); t.add_scalar(beta)
    gamma = t.challenge()
    t.reset(); t.add_scalar(gamma); t.add_pol(pol["C2"])
    xi_seed = t.challenge()
    S0, S1, S2, S2p, xi = _roots(r, xi_seed, w3, w4, w8, wr)
    xiw = xi * w % r
    n = 1 << power
    xin = pow(xi, n, r)
    t.reset(); t.add_scalar(xi_seed)
    for k in EVAL_NAMES:
        t.add_scalar(ev[k])
    alpha = t.challenge()
    t.reset(); t.add_scalar(alpha); t.add_pol(pol["W1"])
    y = t.challenge()
    zh = (xin - 1) % r
    invzh = pow(zh, -1, r)
    L = [None]
    wq = 1
    for _ in range(max(1, n_pub)):
        L.append(wq * zh % r * pow(n * (xi - wq) % r, -1, r) % r)
        wq = wq * w % r
    pi = 0
    for i, s in enumerate(pub):
        pi = (pi - s * L[i + 1]) % r
    # r0 (:383-410)
    li = _li_si(S0, y, xi, r)
    r0 = 0
    for i in range(8):
        h = S0[i]
        c0 = 0
        for k, name in enumerate(("ql", "qr", "qo", "qm", "qc", "s1", "s2", "s3")):
            c0 = (c0 + ev[name] * pow(h, k, r)) % r
        r0 = (r0 + c0 * li[i]) % r
    # r1 (:412-447)
    t0 = (ev["ql"] * ev["a"] + ev["qr"] * ev["b"] + ev["qm"] * ev["a"] % r * ev["b"] + ev["qo"] * ev["c"] + ev["qc"] + pi) % r * invzh % r
    li = _li_si(S1, y, xi, r)
    r1 = 0
    for i in range(4):
        h = S1[i]
        c1 = (ev["a"] + h * ev["b"] + h * h % r * ev["c"] + h * h % r * h % r * t0) % r
        r1 = (r1 + c1 * li[i]) % r
    # r2 (:449-503)
    t1 = (ev["z"] - 1) * L[1] % r * invzh % r
    betaxi = beta * xi % r
    t21 = (ev["a"] + betaxi + gamma) * (ev["b"] + betaxi * k1 + gamma) % r * (ev["c"] + betaxi * k2 + gamma) % r * ev["z"] % r
    t22 = (ev["a"] + beta * ev["s1"] + gamma) * (ev["b"] + beta * ev["s2"] + gamma) % r * (ev["c"] + beta * ev["s3"] + gamma) % r * ev["zw"] % r
    t2 = (t21 - t22) * invzh % r
    li2 = _li_s2(S2, S2p, y, xi, xiw, r)
    r2 = 0
    for i in range(3):
        r2 = (r2 + (ev["z"] + S2[i] * t1 + S2[i] * S2[i] % r * t2) % r * li2[i]) % r
    for i in range(3):
        r2 = (r2 + (ev["zw"] + S2p[i] * ev["t1w"] + S2p[i] * S2p[i] % r * ev["t2w"]) % r * li2[i + 3]) % r
    # F, E, J (:505-544)
    mulH0 = 1
    for x in S0:
        mulH0 = mulH0 * (y - x) % r
    mulH1 = 1
    for x in S1:
        mulH1 = mulH1 * (y - x) % r
    mulH2 = 1
    for x in S2 + S2p:
        mulH2 = mulH2 * (y - x) % r
    q1 = alpha * mulH0 % r * pow(mulH1, -1, r) % r
    q2 = alpha * alpha % r * mulH0 % r * pow(mulH2, -1, r) % r
    Fp = _add(C0, _add(_mul(pol["C1"], q1), _mul(pol["C2"], q2)))
    E = _mul(ci.g1, (r0 + r1 * q1 + r2 * q2) % r)
    J = _mul(pol["W1"], mulH0)
    A1 = _add(_add(_add(Fp, _neg(E)), _neg(J)), _mul(pol["W2"], y))
    if A1 is None or pol["W2"] is None:
        return A1 is None and pol["W2"] is None
    return orc.pairing_product_is_one([(_neg(A1), ci.g2), (pol["W2"], X_2)])


# ----------------------------------------------------------------------------- synthetic structured setup
def fflonk_setup_synth(gates, additions, n_vars: int, n_public: int, tau: int, structured: bool = True) -> bytes:
    """The sections src/fflonk_setup.js:211-503 writes (3 additions, 4-6 wire maps, 7-11 QL QR QM QO QC, 12-14 sigmas,
    15 Lagrange, 16 PTau with 9n + 18 points, 17 C0, 2 header with w3 w4 w8 wr X_2 [C0]_1) for directly-given gates
    (oracle.plonk.chain_gates) and a KNOWN tau, so that proofs verify.  BN254 only, like the reference's constants
    (computeW3 :534-542, getOmegaCubicRoot :552-557).  structured=False: pseudo-random PTau points (parity / throughput)."""
    from .plonk import _g2_times_gen, _mont_from_ints, _tau_powers
    ci = orc.CURVES[orc.BN254]
    r = ci.r
    ng = len(gates)
    power = max(3, (ng + 2 - 1).bit_length())                                       # fflonk_setup.js:112 (two rows stay free for blinding)
    n = 1 << power
    wn = _fr_w(ci, power)
    k1 = 2
    while pow(k1, n, r) == 1:
        k1 += 1
    k2 = k1 + 1
    while pow(k2, n, r) == 1 or pow(k2 * pow(k1, -1, r) % r, n, r) == 1:
        k2 += 1
    w3 = pow(31624, 3648040478639879203707734290876212514758060733402672390616367364429301415936 // 3, r)   # computeW3 :534-542
    w4, w8 = _fr_w(ci, 2), _fr_w(ci, 3)
    wr = pow(467799165886069610036046866799264026481344299079011762026774533774345988080, 1 << (28 - power), r)
    assert pow(w3, 3, r) == 1 and w3 != 1 and pow(wr, 3, r) == wn
    secs = [(3, b"".join(struct.pack("<II", a[0], a[1]) + ci.fr_to_mont(a[2]) + ci.fr_to_mont(a[3]) for a in additions))]
    for pos in range(3):
        secs.append((4 + pos, np.array([g[pos] for g in gates], dtype="<u4").tobytes()))

    def p4(evals):
        coef = bytes(orc.fr_fft(ci.id, _mont_from_ints(ci, evals), True))          # Montgomery bytes throughout
        ev4 = orc.fr_fft(ci.id, coef + bytes(3 * n * 32), False)
        return coef + bytes(ev4), coef

    polys = {}
    # gate tuple = (sl, sr, so, qm, ql, qr, qo, qc); sections 7..11 hold QL QR QM QO QC
    for sid, name, pos in ((7, "QL", 4), (8, "QR", 5), (9, "QM", 3), (10, "QO", 6), (11, "QC", 7)):
        payload, polys[name] = p4([g[pos] for g in gates] + [0] * (n - ng))
        secs.append((sid, payload))
    sigma = [0] * (3 * n)
    last: Dict[int, int] = {}
    first: Dict[int, int] = {}
    w = 1
    for i in range(n):
        for col in range(3):
            p = col * n + i
            v = w if col == 0 else (w * k1 % r if col == 1 else w * k2 % r)
            if i >= n - 2:                      # the two blinding rows map to themselves (fflonk_setup.js:356-360)
                sigma[p] = v
                continue
            s = gates[i][col] if i < ng else 0
            if s not in last:
                first[s] = p
            else:
                sigma[p] = last[s]
            last[s] = v
        w = w * wn % r
    for s, p in first.items():
        sigma[p] = last[s]
    for col, name in enumerate(("S1", "S2", "S3")):
        payload, polys[name] = p4(sigma[col * n:(col + 1) * n])
        secs.append((12 + col, payload))
    # joined once: appending to one bytes object is quadratic in n_public
    secs.append((15, b"".join(p4([1 if j == i else 0 for j in range(n)])[0] for i in range(max(n_public, 1)))))
    npts = 9 * n + 18
    pts = _tau_powers(ci, tau, npts) if structured else bytes(orc.gen_points(ci.id, 1, tau & 0xFFFFFFFF, npts))
    secs.append((16, pts))
    # writeC0 :441-464: C0[8 i + j] = P_j[i] (all eight have n coefficients, so interleaving the byte rows is the CPolynomial)
    rows = np.stack([np.frombuffer(polys[k], dtype=np.uint8).reshape(n, 32) for k in ("QL", "QR", "QO", "QM", "QC", "S1", "S2", "S3")], axis=1)
    c0_bytes = rows.reshape(8 * n * 32).tobytes()
    secs.append((17, c0_bytes))
    if structured:
        jac = orc.multiexp_affine(ci.id, 1, pts[:8 * n * 2 * ci.n8q], bytes(orc.batch_convert(ci.fr, False, c0_bytes)))
        c0_point = ci.g1_from_affine_bytes(orc.g_to_affine(ci.id, 1, jac)[:2 * ci.n8q])
    else:
        c0_point = ci.g1_from_affine_bytes(pts[:2 * ci.n8q])       # any valid point: the transcript only hashes it
    hdr = struct.pack("<I", ci.n8q) + ci.q.to_bytes(ci.n8q, "little") + struct.pack("<I", 32) + r.to_bytes(32, "little")
    hdr += struct.pack("<IIIII", n_vars, n_public, n, len(additions), ng)
    for v in (k1, k2, w3, w4, w8, wr):
        hdr += ci.fr_to_mont(v)
    hdr += _g2_times_gen(ci, tau) if structured else ci.g2_affine_bytes(ci.g2)
    hdr += ci.g1_affine_bytes(c0_point)
    return orc.write_binfile("zkey", 1, [(1, struct.pack("<I", 10)), (2, hdr)] + secs)


# ----------------------------------------------------------------------------- fflonk setup from an r1cs and a ptau
def fflonk_gates_from_r1cs(r1: Dict, r: int):
    """computeFFConstraints (src/fflonk_setup.js:160-209) with src/r1cs_constraint_processor.js:24-200: gates are
    (s1, s2, so, ql, qr, qm, qo, qc).  Unlike plonk_setup.js, zero coefficients ARE dropped (normalizeLinearCombination uses
    Fr.isZero, :85-92); linear combinations are keyed by signal and iterate in ascending signal order."""
    n_pub = r1["nOutputs"] + r1["nPubInputs"]
    state = {"nvars": r1["nVars"]}
    gates, additions = [], []

    def norm(lc):
        return {s: v for s, v in lc.items() if v % r}

    def lc_type(lc):                                                                 # :54-83
        if any(s != 0 for s in lc):
            return 2
        return 1 if lc.get(0, 0) % r else 0

    def join(lc1, lc2, k):                                                          # :94-115
        res = {}
        for s in sorted(lc1):
            res[s] = (res.get(s, 0) + k * lc1[s]) % r
        for s in sorted(lc2):
            res[s] = (res.get(s, 0) - lc2[s]) % r
        return norm(res)

    def reduce_coefs(lc, max_c):                                                    # :117-160
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
            gates.append((c1[0], c2[0], so, (-c1[1]) % r, (-c2[1]) % r, 0, 1, 0))
            additions.append((c1[0], c2[0], c1[1], c2[1]))
            cs.append([so, 1])
        return k, [c[0] for c in cs] + [0] * (max_c - len(cs)), [c[1] for c in cs] + [0] * (max_c - len(cs))

    for s in range(1, n_pub + 1):                                                   # getFFlonkConstantConstraint
        gates.append((s, 0, 0, 1, 0, 0, 0, 0))
    for la, lb, lc in r1["constraints"]:
        la, lb, lc = (norm({int(s): int(v) % r for s, v in t}) for t in (la, lb, lc))
        ta, tb = lc_type(la), lc_type(lb)
        if ta == 0 or tb == 0:
            lin = lc
        elif ta == 1:
            lin = join(lb, lc, la[0])
        elif tb == 1:
            lin = join(la, lc, lb[0])
        else:
            lin = None
        if lin is not None:                                                         # processR1csAdditionConstraint :162-176
            k, ss, cf = reduce_coefs(lin, 3)
            gates.append((ss[0], ss[1], ss[2], cf[0], cf[1], 0, cf[2], k))
        else:                                                                       # processR1csMultiplicationConstraint :178-199
            ka, sa, ca = reduce_coefs(la, 1)
            kb, sb_, cb = reduce_coefs(lb, 1)
            kc, sc, cc = reduce_coefs(lc, 1)
            gates.append((sa[0], sb_[0], sc[0], ca[0] * kb % r, ka * cb[0] % r, ca[0] * cb[0] % r, (-cc[0]) % r, (ka * kb - kc) % r))
    return gates, additions, state["nvars"], n_pub


def fflonk_setup(r1cs, ptau) -> bytes:
    """src/fflonk_setup.js:59-559 from an r1cs and a ptau: the zkey the reference writes, byte for byte (section order 1, 3..17,
    2).  Pinned by tests/test_oracle_fflonk.py against test/fflonk/circuit.zkey."""
    from .plonk import _mont_from_ints
    r1 = orc.read_r1cs(r1cs)
    pdata, psecs = orc.read_binfile(ptau, "ptau", 1)
    ph = orc.read_ptau_header(pdata, psecs)
    ci = orc.curve_from_q(ph["q"])
    r = ci.r
    if r1["prime"] != r:
        raise ValueError("r1cs curve does not match powers of tau ceremony curve")
    if 12 not in psecs:
        raise ValueError("Powers of Tau is not well prepared. Section 12 missing.")
    gates, additions, n_vars, n_public = fflonk_gates_from_r1cs(r1, r)
    ng = len(gates)
    power = max(3, (ng + 2 - 1).bit_length())                                       # :112
    n = 1 << power
    sG1, sG2 = 2 * ci.n8q, 4 * ci.n8q
    p2, l2 = psecs[2][0]
    if l2 < (9 * n + 18) * sG1:
        raise ValueError("Powers of Tau is not big enough for this circuit size. Section 2 too small.")
    pts = bytes(pdata[p2:p2 + (9 * n + 18) * sG1])
    wn = _fr_w(ci, power)
    k1 = 2
    while pow(k1, n, r) == 1:
        k1 += 1
    k2 = k1 + 1
    while pow(k2, n, r) == 1 or pow(k2 * pow(k1, -1, r) % r, n, r) == 1:
        k2 += 1
    w3 = pow(31624, 3648040478639879203707734290876212514758060733402672390616367364429301415936 // 3, r)
    w4, w8 = _fr_w(ci, 2), _fr_w(ci, 3)
    wr = pow(467799165886069610036046866799264026481344299079011762026774533774345988080, 1 << (28 - power), r)
    secs = [(1, struct.pack("<I", 10)),
            (3, b"".join(struct.pack("<II", a[0], a[1]) + ci.fr_to_mont(a[2]) + ci.fr_to_mont(a[3]) for a in additions))]
    for pos in range(3):
        secs.append((4 + pos, np.array([g[pos] for g in gates], dtype="<u4").tobytes()))

    def p4(evals_mont: bytes):
        coef = bytes(orc.fr_fft(ci.id, evals_mont, True))
        return coef + bytes(orc.fr_fft(ci.id, coef + bytes(3 * n * 32), False)), coef

    polys = {}
    for sid, name, pos in ((7, "QL", 3), (8, "QR", 4), (9, "QM", 5), (10, "QO", 6), (11, "QC", 7)):
        payload, polys[name] = p4(_mont_from_ints(ci, [g[pos] for g in gates] + [0] * (n - ng)))
        secs.append((sid, payload))
    sigma = [0] * (3 * n)                                                           # writeSigma :340-415
    last: Dict[int, int] = {}
    first: Dict[int, int] = {}
    w = 1
    for i in range(n):
        for col in range(3):
            p = col * n + i
            v = w if col == 0 else (w * k1 % r if col == 1 else w * k2 % r)
            if i >= n - 2:
                sigma[p] = v
                continue
            s = gates[i][col] if i < ng else 0
            if s not in last:
                first[s] = p
            else:
                sigma[p] = last[s]
            last[s] = v
        w = w * wn % r
    for s, p in first.items():
        sigma[p] = last[s]
    for col, name in enumerate(("S1", "S2", "S3")):
        payload, polys[name] = p4(_mont_from_ints(ci, sigma[col * n:(col + 1) * n]))
        secs.append((12 + col, payload))
    secs.append((15, b"".join(p4(_mont_from_ints(ci, [1 if j == i else 0 for j in range(n)]))[0] for i in range(max(n_public, 1)))))
    secs.append((16, pts))
    rows = np.stack([np.frombuffer(polys[k], dtype=np.uint8).reshape(n, 32) for k in ("QL", "QR", "QO", "QM", "QC", "S1", "S2", "S3")], axis=1)
    c0_bytes = rows.reshape(8 * n * 32).tobytes()                                   # writeC0 :441-464
    secs.append((17, c0_bytes))
    jac = orc.multiexp_affine(ci.id, 1, pts[:8 * n * sG1], bytes(orc.batch_convert(ci.fr, False, c0_bytes)))
    hdr = struct.pack("<I", ci.n8q) + ci.q.to_bytes(ci.n8q, "little") + struct.pack("<I", 32) + r.to_bytes(32, "little")
    hdr += struct.pack("<IIIII", n_vars, n_public, n, len(additions), ng)
    for v in (k1, k2, w3, w4, w8, wr):
        hdr += ci.fr_to_mont(v)
    p3, _ = psecs[3][0]
    hdr += bytes(pdata[p3 + sG2:p3 + 2 * sG2])                                      # X_2 (:498-500)
    hdr += bytes(orc.g_to_affine(ci.id, 1, jac))[:sG1]
    return orc.write_binfile("zkey", 1, secs + [(2, hdr)])
