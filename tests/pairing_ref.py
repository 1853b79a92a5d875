"""Python big-integer restatement of what the device pairing (snarkjs_b200/csrc/pairing.cuh) computes, on top of the oracle's
flat Fq12 arithmetic, for the pairing tests and the Groth16 verify tests.

The device keeps Fq12 as a tower, Fq12 = Fq6[w]/(w^2 - v), Fq6 = Fq2[v]/(v^3 - xi), with 12 Fq coefficients in ffjavascript's
order (the Fq2 coefficient of w^(2j + k) at c_k.c_j).  The oracle works in the flat basis 1, w, ..., w^11 with
u = w^6 - 9 on BN254 and u = w^6 - 1 on BLS12-381 (w^6 = xi on both).  to_flat / from_flat convert between the two."""
from __future__ import annotations

import random

from oracle import oracle as O
from oracle import pairing_bls as PB

CURVES = (O.BN254, O.BLS12_381)
Q = {O.BN254: O.P_BN_Q, O.BLS12_381: O.P_BLS_Q}
R = {O.BN254: O.P_BN_R, O.BLS12_381: O.P_BLS_R}
N8 = {O.BN254: 32, O.BLS12_381: 48}
BETA = {O.BN254: 9, O.BLS12_381: 1}                  # u = w^6 - BETA
X_BN = 4965661367192848881
# the final exponentiation computes f^(C (q^12 - 1) / r) (pairing.cuh header)
C_EXP = {O.BN254: 2 * X_BN * (6 * X_BN * X_BN + 3 * X_BN + 1), O.BLS12_381: 3}
def twist_b(curve):
    """The G2 twist's b as an Fq2 pair."""
    q = Q[curve]
    if curve == O.BN254:                            # 3 / (9 + u)
        n = pow(82, -1, q)
        return (3 * 9 * n % q, -3 * n % q)
    return (4, 4)                                    # 4 (1 + u)


# ---- tower <-> flat ----------------------------------------------------------------------------------------------------
def to_flat(curve, t):
    """12 tower coefficients (device order) -> 12 flat coefficients."""
    q, beta = Q[curve], BETA[curve]
    f = [0] * 12
    for k in range(2):
        for j in range(3):
            a, b = t[(3 * k + j) * 2], t[(3 * k + j) * 2 + 1]
            i = 2 * j + k
            f[i] = (f[i] + a - beta * b) % q
            f[i + 6] = (f[i + 6] + b) % q
    return f


def from_flat(curve, f):
    q, beta = Q[curve], BETA[curve]
    t = [0] * 12
    for k in range(2):
        for j in range(3):
            i = 2 * j + k
            b = f[i + 6] % q
            t[(3 * k + j) * 2] = (f[i] + beta * b) % q
            t[(3 * k + j) * 2 + 1] = b
    return t


# ---- flat arithmetic ---------------------------------------------------------------------------------------------------
def fmul(curve, a, b):
    if curve == O.BN254:
        return (O._FQ12(a) * O._FQ12(b)).c
    return PB._mul(a, b)


def fpow(curve, a, e):
    if curve == O.BN254:
        return (O._FQ12(a) ** e).c
    return PB._pow(a, e)


def finv(curve, a):
    if curve == O.BN254:
        return O._FQ12(a).inv().c
    return PB._inv(a)


def fconj(curve, a):
    """a^(q^6): w -> -w."""
    q = Q[curve]
    return [x if i % 2 == 0 else (-x) % q for i, x in enumerate(a)]


ONE = [1] + [0] * 11


def easy_part(curve, f):
    q = Q[curve]
    t = fmul(curve, fconj(curve, f), finv(curve, f))
    return fmul(curve, fpow(curve, t, q * q), t)


def final_exp_ref(curve, f):
    """f^(C (q^12 - 1) / r): what the device's final exponentiation computes."""
    q, r = Q[curve], R[curve]
    return fpow(curve, easy_part(curve, f), C_EXP[curve] * ((q ** 4 - q ** 2 + 1) // r))


def miller_ref(curve, p1, q2):
    """The oracle's Miller loop (flat, no final exponentiation); None = infinity."""
    if curve == O.BN254:
        return O._miller(q2, p1).c
    return PB._miller(q2, p1)


def pairing_ref(curve, p1, q2):
    """The device's e(P, Q): the oracle's f^((q^12 - 1)/r) raised to C, conjugated on BLS12-381 (where the oracle's loop runs
    over |x| and the device's over x < 0)."""
    e = final_exp_ref(curve, miller_ref(curve, p1, q2))
    return fconj(curve, e) if curve == O.BLS12_381 else e


# ---- points ------------------------------------------------------------------------------------------------------------
def g_mul(curve, group, pt, k):
    """k * pt for affine int points (None = infinity) through the oracle's group arithmetic."""
    ci = O.CURVES[curve]
    enc = ci.g1_affine_bytes if group == 1 else ci.g2_affine_bytes
    dec = ci.g1_from_affine_bytes if group == 1 else ci.g2_from_affine_bytes
    if pt is None or k % ci.r == 0:
        return None
    j = O.g_times(curve, group, O.g_from_affine(curve, group, enc(pt)), (k % ci.r).to_bytes(32, "little"))
    return dec(O.g_to_affine(curve, group, j))


def rand_fq12(curve, rng: random.Random):
    return [rng.randrange(Q[curve]) for _ in range(12)]


def mont(curve, x):
    return (x % Q[curve]) * (1 << (8 * N8[curve])) % Q[curve]


def unmont(curve, x):
    return x * pow(1 << (8 * N8[curve]), -1, Q[curve]) % Q[curve]


def pack(curve, vals) -> bytes:
    """Fq values (plain ints) -> Montgomery little-endian bytes."""
    n8 = N8[curve]
    return b"".join(mont(curve, v).to_bytes(n8, "little") for v in vals)


def unpack(curve, data: bytes):
    n8 = N8[curve]
    return [unmont(curve, int.from_bytes(data[i:i + n8], "little")) for i in range(0, len(data), n8)]


def pt_vals(p1, q2):
    """(G1 affine ints | None, G2 affine ints | None) -> the 6 Fq values of an op-5/7 record."""
    a = [0, 0] if p1 is None else [p1[0], p1[1]]
    b = [0, 0, 0, 0] if q2 is None else [q2[0][0], q2[0][1], q2[1][0], q2[1][1]]
    return a + b
