"""oracle/oracle.py — Python face of the CPU oracle (TEST INFRASTRUCTURE, not product code).

ctypes wrapper over oracle/liboracle.so (snark_oracle.cpp) plus CPU restatements of the
reference's host-side logic that sits either side of the hot path:

  * binfile container reader/writer      (@iden3/binfileutils, build/snarkjs.js:17468-17598)
  * wtns / r1cs / zkey / ptau readers    (src/wtns_utils.js:62-72, src/zkey_utils.js:229-339,
                                          src/powersoftau_utils.js:52-71)
  * Groth16 phase-2 setup `zkey new`     (src/zkey_new.js:36-586)   -- needed because the
    reference ships no Groth16 .zkey fixture (SURVEY.md fact 5)
  * Groth16 prover with injectable (r,s) (src/groth16_prove.js:28-374)
  * Groth16 verifier + BN254 optimal-ate pairing in pure Python ints
                                         (src/groth16_verify.js:25-85)

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
import this module.  Parity status: pinned against reference-produced bytes in tests/golden/
(see snark_oracle.cpp header).
"""
from __future__ import annotations

import ctypes
import os
import struct
import subprocess
from typing import Dict, List, Tuple

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

BN254, BLS12_381 = 0, 1
F_BN_FQ, F_BN_FR, F_BLS_FQ, F_BLS_FR = 0, 1, 2, 3

P_BN_Q = 0x30644e72e131a029b85045b68181585d97816a916871ca8d3c208c16d87cfd47
P_BN_R = 0x30644e72e131a029b85045b68181585d2833e84879b9709143e1f593f0000001
P_BLS_Q = 0x1a0111ea397fe69a4b1ba7b6434bacd764774b84f38512bf6730d2a0f6b0f6241eabfffeb153ffffb9feffffffffaaab
P_BLS_R = 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001


def build(force: bool = False) -> str:
    so = os.path.join(_HERE, "liboracle.so")
    src = os.path.join(_HERE, "snark_oracle.cpp")
    if force or not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "-B" if force else "-s"], stdout=subprocess.DEVNULL)
    return so


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "liboracle.so")
        if not os.path.exists(so):
            build()
        _LIB = ctypes.CDLL(so)
        _LIB.or_init()
    return _LIB


def _p(b):
    """bytes/bytearray/ndarray -> c pointer (zero-copy for ndarray/bytearray)."""
    if b is None:
        return None
    if isinstance(b, np.ndarray):
        return b.ctypes.data_as(ctypes.c_char_p)
    if isinstance(b, (bytes, bytearray, memoryview)):
        return (ctypes.c_char * len(b)).from_buffer_copy(b) if isinstance(b, (bytes, memoryview)) else (ctypes.c_char * len(b)).from_buffer(b)
    raise TypeError(type(b))


def _chk(rc, what):
    if rc != 0:
        raise RuntimeError(f"oracle {what} failed rc={rc}")


# ----------------------------------------------------------------------------- curve info
class CurveInfo:
    def __init__(self, cid):
        self.id = cid
        self.name = "bn128" if cid == BN254 else "bls12381"
        self.q = P_BN_Q if cid == BN254 else P_BLS_Q
        self.r = P_BN_R if cid == BN254 else P_BLS_R
        self.n8q = 32 if cid == BN254 else 48
        self.n8r = 32
        self.fq = F_BN_FQ if cid == BN254 else F_BLS_FQ
        self.fr = F_BN_FR if cid == BN254 else F_BLS_FR
        self.Rq = (1 << (8 * self.n8q)) % self.q
        self.Rr = (1 << 256) % self.r
        if cid == BN254:
            self.g1 = (1, 2)                                                # build/snarkjs.js:9468-9472
            self.g2 = ((10857046999023057135944570762232829481370756359578518086990519993285655852781,
                        11559732032986387107991004021392285783925812861821192530917403151452391805634),
                       (8495653923123431417604973247489272438418190587263600148770280649306958101930,
                        4082367875863433681332203403145435568316851327593401208105741076214120093531))
        else:
            self.g1 = (0x17f1d3a73197d7942695638c4fa9ac0fc3688c4f9774b905a14e3a3f171bac586c55e83ff97a1aeffb3af00adb22c6bb,
                       0x08b3f481e3aaa0f1a09e30ed741d8ae4fcf5e095d5d00af600db18cb2c04b3edd03cc744a2888ae40caa232946c5e7e1)
            self.g2 = ((0x024aa2b2f08f0a91260805272dc51051c6e47ad4fa403b02b4510b647ae3d1770bac0326a805bbefd48056c8c121bdb8,
                        0x13e02b6052719f607dacd3a088274f65596bd0d09920b61ab5da61bbdc7f5049334cf11213945d57e5ac7d055d042b7e),
                       (0x0ce5d527727d6e118cc9cdc6da2e351aadfd9baa8cbdd3a76d429a695160d12c923ac9cc3baca289e193548608b82801,
                        0x0606c4a02ea734cc32acd2b02bc28b99cb3e287e85a763af267492ab572e99ab3f370d275cec1da1aaa9075ff05f79be))

    # integer <-> Montgomery LE bytes
    def fq_to_mont(self, x: int) -> bytes:
        return ((x % self.q) * self.Rq % self.q).to_bytes(self.n8q, "little")

    def fq_from_mont(self, b: bytes) -> int:
        return int.from_bytes(b, "little") * pow(self.Rq, -1, self.q) % self.q

    def fr_to_mont(self, x: int) -> bytes:
        return ((x % self.r) * self.Rr % self.r).to_bytes(32, "little")

    def fr_from_mont(self, b: bytes) -> int:
        return int.from_bytes(b, "little") * pow(self.Rr, -1, self.r) % self.r

    def g1_affine_bytes(self, pt) -> bytes:
        if pt is None:
            return bytes(2 * self.n8q)
        return self.fq_to_mont(pt[0]) + self.fq_to_mont(pt[1])

    def g2_affine_bytes(self, pt) -> bytes:
        if pt is None:
            return bytes(4 * self.n8q)
        (x0, x1), (y0, y1) = pt
        return self.fq_to_mont(x0) + self.fq_to_mont(x1) + self.fq_to_mont(y0) + self.fq_to_mont(y1)

    def g1_from_affine_bytes(self, b: bytes):
        n = self.n8q
        if b == bytes(2 * n):
            return None
        return (self.fq_from_mont(b[:n]), self.fq_from_mont(b[n:2 * n]))

    def g2_from_affine_bytes(self, b: bytes):
        n = self.n8q
        if b == bytes(4 * n):
            return None
        return ((self.fq_from_mont(b[:n]), self.fq_from_mont(b[n:2 * n])),
                (self.fq_from_mont(b[2 * n:3 * n]), self.fq_from_mont(b[3 * n:4 * n])))


CURVES = {BN254: CurveInfo(BN254), BLS12_381: CurveInfo(BLS12_381)}


def curve_from_q(q: int) -> CurveInfo:
    """src/curves.js:23-34 getCurveFromQ"""
    for c in CURVES.values():
        if c.q == q:
            return c
    raise ValueError(f"Curve not supported: {q}")


def curve_from_r(r: int) -> CurveInfo:
    for c in CURVES.values():
        if c.r == r:
            return c
    raise ValueError(f"Curve not supported: {r}")


# ----------------------------------------------------------------------------- field / group wrappers
def field_op(fid, op, a: bytes, b: bytes | None = None) -> bytes:
    n8 = lib().or_field_n8(fid)
    out = ctypes.create_string_buffer(n8)
    _chk(lib().or_field_op(fid, op, a, b, out), "field_op")
    return out.raw


def fr_root(curve: int, idx: int) -> bytes:
    out = ctypes.create_string_buffer(32)
    lib().or_fr_root(curve, idx, out)
    return out.raw


def fr_s(curve: int) -> int:
    out = ctypes.create_string_buffer(32)
    return lib().or_fr_root(curve, 0, out)


def _buf(n):
    return np.empty(n, dtype=np.uint8)


def _in(b):
    if isinstance(b, np.ndarray):
        return np.ascontiguousarray(b.view(np.uint8).reshape(-1))
    return np.frombuffer(bytes(b), dtype=np.uint8)


def batch_convert(fid, to_mont: bool, data) -> np.ndarray:
    a = _in(data)
    n8 = lib().or_field_n8(fid)
    if a.size % n8:
        raise ValueError("Invalid buffer size")          # build/snarkjs.js:12780-12830
    out = _buf(a.size)
    _chk(lib().or_batch_convert(fid, int(to_mont), _p(a), ctypes.c_uint64(a.size // n8), _p(out)), "batch_convert")
    return out


def fr_fft(curve: int, data, inverse: bool = False) -> np.ndarray:
    a = _in(data)
    n = a.size // 32
    if n == 0 or n & (n - 1):
        raise ValueError("fft must be multiple of 2")     # build/snarkjs.js:14745-14747
    out = _buf(a.size)
    _chk(lib().or_fr_fft(curve, _p(a), ctypes.c_uint64(n), int(inverse), _p(out)), "fr_fft")
    return out


def fr_batch_apply_key(curve: int, data, first: bytes, inc: bytes) -> np.ndarray:
    a = _in(data)
    out = _buf(a.size)
    _chk(lib().or_fr_batch_apply_key(curve, _p(a), ctypes.c_uint64(a.size // 32), first, inc, _p(out)), "apply_key")
    return out


def qap_join_abc(curve: int, a, b, c) -> np.ndarray:
    a, b, c = _in(a), _in(b), _in(c)
    out = _buf(a.size)
    _chk(lib().or_qap_join_abc(curve, _p(a), _p(b), _p(c), ctypes.c_uint64(a.size // 32), _p(out)), "join_abc")
    return out


def build_abc(curve: int, coeffs, witness, domain_size: int):
    """coeffs = zkey section 4 payload (including the leading u32 count)."""
    cf = _in(coeffs)
    w = _in(witness)
    ncoef = (cf.size - 4) // 44
    A, B, C = _buf(domain_size * 32), _buf(domain_size * 32), _buf(domain_size * 32)
    body = np.ascontiguousarray(cf[4:])
    _chk(lib().or_build_abc(curve, _p(body), ctypes.c_uint64(ncoef), _p(w), ctypes.c_uint64(w.size // 32),
                            ctypes.c_uint64(domain_size), _p(A), _p(B), _p(C)), "build_abc")
    return A, B, C


def multiexp_affine(curve: int, group: int, bases, scalars, concurrency: int = 8) -> bytes:
    """G.multiExpAffine (build/snarkjs.js:14666-14668) -> Jacobian Montgomery bytes."""
    ci = CURVES[curve]
    sG = ci.n8q * 2 * group
    b, s = _in(bases), _in(scalars)
    n = b.size // sG
    out = ctypes.create_string_buffer(ci.n8q * 3 * group)
    if n == 0:
        return group_zero(curve, group)
    ss = s.size // n
    if ss * n != s.size:
        raise ValueError("Scalar size does not match")    # build/snarkjs.js:14562-14565
    _chk(lib().or_multiexp_affine(curve, group, _p(b), _p(s), ss, ctypes.c_uint64(n), concurrency, out), "multiexp")
    return out.raw


def multiexp_naive(curve: int, group: int, bases, scalars) -> bytes:
    ci = CURVES[curve]
    sG = ci.n8q * 2 * group
    b, s = _in(bases), _in(scalars)
    n = b.size // sG
    out = ctypes.create_string_buffer(ci.n8q * 3 * group)
    _chk(lib().or_multiexp_naive(curve, group, _p(b), _p(s), s.size // max(n, 1), ctypes.c_uint64(n), out), "naive")
    return out.raw


def group_zero(curve, group) -> bytes:
    ci = CURVES[curve]
    one = ci.fq_to_mont(1)
    z = bytes(ci.n8q)
    if group == 1:
        return z + one + z
    return z + z + one + z + z + z


def group_op(curve, group, op, a: bytes, b: bytes | None = None) -> bytes:
    ci = CURVES[curve]
    out_len = {2: ci.n8q * 2 * group, 6: 1}.get(op, ci.n8q * 3 * group)
    out = ctypes.create_string_buffer(out_len)
    _chk(lib().or_group_op(curve, group, op, a, b, out), "group_op")
    return out.raw


def g_add(curve, group, a, b): return group_op(curve, group, 0, a, b)
def g_double(curve, group, a): return group_op(curve, group, 1, a)
def g_to_affine(curve, group, a): return group_op(curve, group, 2, a)
def g_neg(curve, group, a): return group_op(curve, group, 3, a)
def g_from_affine(curve, group, a): return group_op(curve, group, 5, a)
def g_eq(curve, group, a, b): return group_op(curve, group, 6, a, b)[0] == 1


def g_times(curve, group, a: bytes, scalar_le: bytes) -> bytes:
    ci = CURVES[curve]
    out = ctypes.create_string_buffer(ci.n8q * 3 * group)
    _chk(lib().or_group_times(curve, group, a, scalar_le, len(scalar_le), out), "times")
    return out.raw


def g_times_fr(curve, group, a: bytes, fr_mont: bytes) -> bytes:
    """g?m_timesFr = frm_fromMontgomery then timesScalar (build/snarkjs.js:9426-9456)"""
    plain = field_op(CURVES[curve].fr, 6, fr_mont)
    return g_times(curve, group, a, plain)


def batch_to_affine(curve, group, data) -> np.ndarray:
    ci = CURVES[curve]
    a = _in(data)
    n = a.size // (ci.n8q * 3 * group)
    out = _buf(n * ci.n8q * 2 * group)
    _chk(lib().or_batch_to_affine(curve, group, _p(a), ctypes.c_uint64(n), _p(out)), "batch_to_affine")
    return out


def gen_points(curve, group, seed: int, n: int) -> np.ndarray:
    """Deterministic synthetic affine bases (valid curve points), Montgomery LE."""
    ci = CURVES[curve]
    g = ci.g1_affine_bytes(ci.g1) if group == 1 else ci.g2_affine_bytes(ci.g2)
    out = _buf(n * ci.n8q * 2 * group)
    _chk(lib().or_gen_points(curve, group, g, ctypes.c_uint64(seed), ctypes.c_uint64(n), _p(out)), "gen_points")
    return out


# ----------------------------------------------------------------------------- deterministic RNG (SURVEY §8d)
def splitmix64_stream(seed: int, n_words: int) -> np.ndarray:
    """n_words uint64 of SplitMix64(seed) — vectorised."""
    with np.errstate(over="ignore"):
        idx = np.arange(1, n_words + 1, dtype=np.uint64)
        z = np.uint64(seed) + idx * np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
    return z


def random_scalars(seed: int, n: int, modulus: int, bits: int | None = None) -> np.ndarray:
    """n plain LE 32-byte scalars, uniform-ish below `modulus` (top bits masked then conditional subtract)."""
    w = splitmix64_stream(seed, 4 * n).reshape(n, 4).copy()
    nb = modulus.bit_length() if bits is None else bits
    top_bits = nb - 192
    if top_bits < 64:
        w[:, 3] &= np.uint64((1 << max(top_bits, 0)) - 1)
    if nb <= 192:
        w[:, 3] = 0
    # conditional subtract of modulus where value >= modulus (vectorised 256-bit compare)
    m = [(modulus >> (64 * i)) & 0xFFFFFFFFFFFFFFFF for i in range(4)]
    ge = np.zeros(n, dtype=bool)
    eq = np.ones(n, dtype=bool)
    for i in (3, 2, 1, 0):
        ge |= eq & (w[:, i] > np.uint64(m[i]))
        eq &= (w[:, i] == np.uint64(m[i]))
    ge |= eq
    if ge.any():
        idxs = np.nonzero(ge)[0]
        for k in idxs:
            v = sum(int(w[k, i]) << (64 * i) for i in range(4)) - modulus
            for i in range(4):
                w[k, i] = np.uint64((v >> (64 * i)) & 0xFFFFFFFFFFFFFFFF)
    return w.view(np.uint8).reshape(-1)


# ----------------------------------------------------------------------------- binfile container
def read_binfile(path_or_bytes, magic: str, max_version: int = 2) -> Tuple[bytes, Dict[int, List[Tuple[int, int]]]]:
    """@iden3/binfileutils readBinFile (build/snarkjs.js:17468-17498): returns (data, {id: [(pos,len)]})."""
    data = path_or_bytes if isinstance(path_or_bytes, (bytes, bytearray)) else open(path_or_bytes, "rb").read()
    if data[:4] != magic.encode():
        raise ValueError(f"{magic}: Invalid File format")
    ver, nsec = struct.unpack_from("<II", data, 4)
    if ver > max_version:
        raise ValueError("Version not supported")
    pos = 12
    sections: Dict[int, List[Tuple[int, int]]] = {}
    for _ in range(nsec):
        sid, ln = struct.unpack_from("<IQ", data, pos)
        pos += 12
        sections.setdefault(sid, []).append((pos, ln))
        pos += ln
    if pos != len(data):
        raise ValueError("Invalid file size")
    return data, sections


def section(data, sections, sid) -> memoryview:
    if sid not in sections:
        raise KeyError(f"Missing section {sid}")
    if len(sections[sid]) > 1:
        raise ValueError(f"Section Duplicated {sid}")
    p, ln = sections[sid][0]
    return memoryview(data)[p:p + ln]


def write_binfile(magic: str, version: int, secs: List[Tuple[int, bytes]]) -> bytes:
    out = bytearray(magic.encode() + struct.pack("<II", version, len(secs)))
    for sid, payload in secs:
        out += struct.pack("<IQ", sid, len(payload)) + bytes(payload)
    return bytes(out)


def read_wtns(path_or_bytes):
    """src/wtns_utils.js:62-72 — returns (header dict, witness bytes plain LE)."""
    data, secs = read_binfile(path_or_bytes, "wtns", 2)
    h = section(data, secs, 1)
    n8 = struct.unpack_from("<I", h, 0)[0]
    q = int.from_bytes(h[4:4 + n8], "little")
    nw = struct.unpack_from("<I", h, 4 + n8)[0]
    w = bytes(section(data, secs, 2))
    return {"n8": n8, "q": q, "nWitness": nw}, w


def read_r1cs(path_or_bytes):
    """r1csfile header + constraints (SURVEY Appendix A)."""
    data, secs = read_binfile(path_or_bytes, "r1cs", 1)
    h = section(data, secs, 1)
    n8 = struct.unpack_from("<I", h, 0)[0]
    prime = int.from_bytes(h[4:4 + n8], "little")
    nVars, nOutputs, nPubInputs, nPrvInputs = struct.unpack_from("<IIII", h, 4 + n8)
    nLabels = struct.unpack_from("<Q", h, 20 + n8)[0]
    nConstraints = struct.unpack_from("<I", h, 28 + n8)[0]
    body = bytes(section(data, secs, 2))
    cons = []
    pos = 0
    for _ in range(nConstraints):
        lc3 = []
        for _k in range(3):
            k = struct.unpack_from("<I", body, pos)[0]
            pos += 4
            lc = []
            for _j in range(k):
                wire = struct.unpack_from("<I", body, pos)[0]
                pos += 4
                lc.append((wire, int.from_bytes(body[pos:pos + n8], "little")))
                pos += n8
            lc3.append(lc)
        cons.append(lc3)
    return {"n8": n8, "prime": prime, "nVars": nVars, "nOutputs": nOutputs, "nPubInputs": nPubInputs,
            "nPrvInputs": nPrvInputs, "nLabels": nLabels, "nConstraints": nConstraints, "constraints": cons}


def read_ptau_header(data, secs):
    """src/powersoftau_utils.js:52-71"""
    h = section(data, secs, 1)
    n8 = struct.unpack_from("<I", h, 0)[0]
    q = int.from_bytes(h[4:4 + n8], "little")
    power, ceremony_power = struct.unpack_from("<II", h, 4 + n8)
    return {"n8": n8, "q": q, "power": power, "ceremonyPower": ceremony_power}


def read_zkey_header(data, secs):
    """src/zkey_utils.js:208-339"""
    proto = struct.unpack_from("<I", section(data, secs, 1), 0)[0]
    h = section(data, secs, 2)
    n8q = struct.unpack_from("<I", h, 0)[0]
    q = int.from_bytes(h[4:4 + n8q], "little")
    n8r = struct.unpack_from("<I", h, 4 + n8q)[0]
    r = int.from_bytes(h[8 + n8q:8 + n8q + n8r], "little")
    o = 8 + n8q + n8r
    z = {"protocolId": proto, "n8q": n8q, "q": q, "n8r": n8r, "r": r}
    if proto == 1:      # groth16  zkey_utils.js:229-259
        z["protocol"] = "groth16"
        z["nVars"], z["nPublic"], z["domainSize"] = struct.unpack_from("<III", h, o)
        o += 12
        sG1, sG2 = 2 * n8q, 4 * n8q
        for name, sz in (("vk_alpha_1", sG1), ("vk_beta_1", sG1), ("vk_beta_2", sG2), ("vk_gamma_2", sG2),
                         ("vk_delta_1", sG1), ("vk_delta_2", sG2)):
            z[name] = bytes(h[o:o + sz])
            o += sz
    elif proto == 2:    # plonk  zkey_utils.js:261-299
        z["protocol"] = "plonk"
        (z["nVars"], z["nPublic"], z["domainSize"], z["nAdditions"], z["nConstraints"]) = struct.unpack_from("<IIIII", h, o)
        o += 20
        z["k1"] = bytes(h[o:o + n8r]); o += n8r
        z["k2"] = bytes(h[o:o + n8r]); o += n8r
        for name in ("Qm", "Ql", "Qr", "Qo", "Qc", "S1", "S2", "S3"):
            z[name] = bytes(h[o:o + 2 * n8q]); o += 2 * n8q
        z["X_2"] = bytes(h[o:o + 4 * n8q])
    elif proto == 10:   # fflonk zkey_utils.js:301-339
        z["protocol"] = "fflonk"
        (z["nVars"], z["nPublic"], z["domainSize"], z["nAdditions"], z["nConstraints"]) = struct.unpack_from("<IIIII", h, o)
        o += 20
        for name in ("k1", "k2", "w3", "w4", "w8", "wr"):
            z[name] = bytes(h[o:o + n8r]); o += n8r
        z["X_2"] = bytes(h[o:o + 4 * n8q]); o += 4 * n8q
        z["C0"] = bytes(h[o:o + 2 * n8q])
    else:
        raise ValueError("Protocol not supported")
    z["power"] = int(z["domainSize"]).bit_length() - 1
    return z


# ----------------------------------------------------------------------------- zkey new (Groth16 setup)
def zkey_new(r1cs_path, ptau_path) -> bytes:
    """Restates src/zkey_new.js:36-586 (no contributions: gamma2 = delta2 = G2 gen, delta1 = G1 gen).
    The contribution-hash section (10) is filled with 64 zero bytes + u32 0: the circuit hash
    (blake2b over uncompressed points) is not on the proving path."""
    r1 = read_r1cs(r1cs_path)
    pdata, psecs = read_binfile(ptau_path, "ptau", 1)
    ph = read_ptau_header(pdata, psecs)
    ci = curve_from_q(ph["q"])
    if r1["prime"] != ci.r:
        raise ValueError("r1cs curve does not match powers of tau ceremony curve")
    n8q, n8r = ci.n8q, ci.n8r
    sG1, sG2 = 2 * n8q, 4 * n8q
    nC = r1["nConstraints"]
    nPublic = r1["nOutputs"] + r1["nPubInputs"]
    cirPower = (nC + nPublic + 1 - 1).bit_length() - 1 + 1           # zkey_new.js:59  log2(x)+1
    if cirPower > ph["power"]:
        raise ValueError("circuit too big for this power of tau ceremony")
    if 12 not in psecs:
        raise ValueError("Powers of tau is not prepared.")
    domainSize = 1 << cirPower
    nVars = r1["nVars"]

    def psec(sid, lo, hi):
        p, _ = psecs[sid][0]
        return bytes(pdata[p + lo:p + hi])

    hdr = struct.pack("<I", n8q) + ci.q.to_bytes(n8q, "little") + struct.pack("<I", n8r) + ci.r.to_bytes(n8r, "little")
    hdr += struct.pack("<III", nVars, nPublic, domainSize)
    hdr += psec(4, 0, sG1) + psec(5, 0, sG1) + psec(6, 0, sG2)                   # alpha1, beta1, beta2 (:101-116)
    bg1, bg2 = ci.g1_affine_bytes(ci.g1), ci.g2_affine_bytes(ci.g2)
    hdr += bg2 + bg1 + bg2                                                       # gamma2, delta1, delta2 (:127-129)

    # Lagrange-basis points for this domain (:145-151)
    sTauG1 = psec(12, (domainSize - 1) * sG1, (2 * domainSize - 1) * sG1)
    sTauG2 = psec(13, (domainSize - 1) * sG2, (2 * domainSize - 1) * sG2)
    sAlphaTauG1 = psec(14, (domainSize - 1) * sG1, (2 * domainSize - 1) * sG1)
    sBetaTauG1 = psec(15, (domainSize - 1) * sG1, (2 * domainSize - 1) * sG1)
    TAU_G1, TAU_G2, ALPHATAU_G1, BETATAU_G1 = 0, 1, 2, 3
    sb = [sTauG1, sTauG2, sAlphaTauG1, sBetaTauG1]
    ss = [sG1, sG2, sG1, sG1]

    # processConstraints (:213-330)
    A = [[] for _ in range(nVars)]
    B1 = [[] for _ in range(nVars)]
    B2 = [[] for _ in range(nVars)]
    C = [[] for _ in range(nVars - nPublic - 1)]
    IC = [[] for _ in range(nPublic + 1)]
    coefs = []
    for c, (la, lb, lc) in enumerate(r1["constraints"]):
        for s, v in la:
            A[s].append((TAU_G1, c, v))
            (IC[s] if s <= nPublic else C[s - nPublic - 1]).append((BETATAU_G1, c, v))
            coefs.append((0, c, s, v))
        for s, v in lb:
            B1[s].append((TAU_G1, c, v))
            B2[s].append((TAU_G2, c, v))
            (IC[s] if s <= nPublic else C[s - nPublic - 1]).append((ALPHATAU_G1, c, v))
            coefs.append((1, c, s, v))
        for s, v in lc:
            (IC[s] if s <= nPublic else C[s - nPublic - 1]).append((TAU_G1, c, v))
    for s in range(nPublic + 1):
        A[s].append((TAU_G1, nC + s, 1))
        IC[s].append((BETATAU_G1, nC + s, 1))
        coefs.append((0, nC + s, s, 1))

    R2r = (ci.Rr * ci.Rr) % ci.r
    sec4 = bytearray(struct.pack("<I", len(coefs)))
    for m, c, s, v in coefs:
        # writeCoef (:316-330): Fr.mul(n, R2r) with n taken as a Montgomery residue => n*R mod r stored... the
        # stored value is n*R^2*R^-1 = n*R ... careful: curve.Fr.fromRprLE(n) gives the element whose *value* is n
        # (internally n*R); Fr.mul by the element R2r (value R^2) gives value n*R^2; toRprLE writes the value.
        sec4 += struct.pack("<III", m, c, s) + ((v * R2r) % ci.r).to_bytes(n8r, "little")

    def compose(arr, group):
        """composeAndWritePoints (:338-470): point[s] = sum coef * Lagrange[c] (an MSM per signal)."""
        sG = sG1 if group == 1 else sG2
        out = bytearray()
        for terms in arr:
            if not terms:
                out += bytes(sG)
                continue
            bases = b"".join(sb[t][c * ss[t]:(c + 1) * ss[t]] for t, c, _v in terms)
            scal = b"".join((v % ci.r).to_bytes(n8r, "little") for _t, _c, v in terms)
            # a signal in a few constraints has a few terms: the plain sum of products is the same point, without the
            # Pippenger's per-call thread start-up over its 256 one-bit windows (about 8 ms)
            jac = multiexp_naive(ci.id, group, bases, scal) if len(terms) < 8 else multiexp_affine(ci.id, group, bases, scal, 1)
            out += g_to_affine(ci.id, group, jac)
        return bytes(out)

    # writeHs (:182-200): odd entries of the 2n Lagrange basis
    if cirPower < fr_s(ci.id):
        big = psec(12, (2 * domainSize - 1) * sG1, (4 * domainSize - 1) * sG1)
        sec9 = b"".join(big[(2 * i + 1) * sG1:(2 * i + 2) * sG1] for i in range(domainSize))
    else:
        raise ValueError("Circuit too big")

    secs = [
        (1, struct.pack("<I", 1)),
        (2, hdr),
        (4, bytes(sec4)),
        (3, compose(IC, 1)),
        (9, sec9),
        (8, compose(C, 1)),
        (5, compose(A, 1)),
        (6, compose(B1, 1)),
        (7, compose(B2, 2)),
        (10, bytes(64) + struct.pack("<I", 0)),
    ]
    return write_binfile("zkey", 1, secs)


# ----------------------------------------------------------------------------- Groth16 prove / verify
def groth16_prove(zkey, wtns, r_mont: bytes, s_mont: bytes, concurrency: int = 8, return_parts: bool = False):
    """Restates src/groth16_prove.js:28-144 with (r,s) injected as 32-byte Montgomery Fr elements
    (the reference draws them with Fr.random(), :103-104)."""
    zdata, zsecs = read_binfile(zkey, "zkey", 2)
    zk = read_zkey_header(zdata, zsecs)
    if zk["protocol"] != "groth16":
        raise ValueError("zkey file is not groth16")
    wh, W = read_wtns(wtns)
    if wh["q"] != zk["r"]:
        raise ValueError("Curve of the witness does not match the curve of the proving key")
    if wh["nWitness"] != zk["nVars"]:
        raise ValueError(f"Invalid witness length. Circuit: {zk['nVars']}, witness: {wh['nWitness']}")
    ci = curve_from_q(zk["q"])
    cid = ci.id
    power = zk["power"]
    n = zk["domainSize"]
    coeffs = section(zdata, zsecs, 4)
    A_T, B_T, C_T = build_abc(cid, bytes(coeffs), W, n)                     # :62
    inc = fr_root(cid, -1) if power == fr_s(cid) else fr_root(cid, power + 1)  # :64
    one = ci.fr_to_mont(1)
    odd = []
    for X in (A_T, B_T, C_T):                                               # :66-76
        x = fr_fft(cid, X, inverse=True)
        x = fr_batch_apply_key(cid, x, one, inc)
        odd.append(fr_fft(cid, x))
    P = qap_join_abc(cid, odd[0], odd[1], odd[2])                            # :79
    G1, G2 = 1, 2
    Wb = np.frombuffer(W, dtype=np.uint8)
    msm = {}
    msm["A"] = multiexp_affine(cid, G1, section(zdata, zsecs, 5), Wb, concurrency)
    msm["B1"] = multiexp_affine(cid, G1, section(zdata, zsecs, 6), Wb, concurrency)
    msm["B2"] = multiexp_affine(cid, G2, section(zdata, zsecs, 7), Wb, concurrency)
    msm["C"] = multiexp_affine(cid, G1, section(zdata, zsecs, 8), Wb[(zk["nPublic"] + 1) * 32:], concurrency)
    msm["H"] = multiexp_affine(cid, G1, section(zdata, zsecs, 9), P, concurrency)
    proof_jac = groth16_assemble(ci, zk, msm, r_mont, s_mont)
    pub = [int.from_bytes(W[i * 32:(i + 1) * 32], "little") for i in range(1, zk["nPublic"] + 1)]
    proof = proof_to_object(ci, proof_jac)
    if return_parts:
        parts = {"A_T": A_T, "B_T": B_T, "C_T": C_T, "odd": odd, "P": P,
                 "msm_affine": {k: g_to_affine(cid, 2 if k == "B2" else 1, v) for k, v in msm.items()}}
        return proof, pub, parts
    return proof, pub


def groth16_assemble(ci: CurveInfo, zk, msm, r_mont: bytes, s_mont: bytes):
    """src/groth16_prove.js:106-120 — returns affine bytes (pi_a 2n8q, pi_b 4n8q, pi_c 2n8q)."""
    cid = ci.id
    fa = lambda b: g_from_affine(cid, 1, b)
    fa2 = lambda b: g_from_affine(cid, 2, b)
    delta1, delta2 = fa(zk["vk_delta_1"]), fa2(zk["vk_delta_2"])
    pi_a = g_add(cid, 1, msm["A"], fa(zk["vk_alpha_1"]))
    pi_a = g_add(cid, 1, pi_a, g_times_fr(cid, 1, delta1, r_mont))
    pi_b = g_add(cid, 2, msm["B2"], fa2(zk["vk_beta_2"]))
    pi_b = g_add(cid, 2, pi_b, g_times_fr(cid, 2, delta2, s_mont))
    pib1 = g_add(cid, 1, msm["B1"], fa(zk["vk_beta_1"]))
    pib1 = g_add(cid, 1, pib1, g_times_fr(cid, 1, delta1, s_mont))
    pi_c = g_add(cid, 1, msm["C"], msm["H"])
    pi_c = g_add(cid, 1, pi_c, g_times_fr(cid, 1, pi_a, s_mont))
    pi_c = g_add(cid, 1, pi_c, g_times_fr(cid, 1, pib1, r_mont))
    rs = field_op(ci.fr, 3, field_op(ci.fr, 2, r_mont, s_mont))
    pi_c = g_add(cid, 1, pi_c, g_times_fr(cid, 1, delta1, rs))
    return (g_to_affine(cid, 1, pi_a), g_to_affine(cid, 2, pi_b), g_to_affine(cid, 1, pi_c))


def proof_to_object(ci: CurveInfo, affine3) -> dict:
    """G.toObject + stringifyBigInts (src/groth16_prove.js:130-141)."""
    a, b, c = affine3
    pa = ci.g1_from_affine_bytes(a)
    pb = ci.g2_from_affine_bytes(b)
    pc = ci.g1_from_affine_bytes(c)

    def o1(p):
        return ["0", "1", "0"] if p is None else [str(p[0]), str(p[1]), "1"]

    def o2(p):
        if p is None:
            return [["0", "0"], ["1", "0"], ["0", "0"]]
        return [[str(p[0][0]), str(p[0][1])], [str(p[1][0]), str(p[1][1])], ["1", "0"]]

    return {"pi_a": o1(pa), "pi_b": o2(pb), "pi_c": o1(pc), "protocol": "groth16", "curve": ci.name}


def zkey_vk(zkey) -> dict:
    """Verification-key pieces straight from the zkey (src/zkey_export_verificationkey.js semantics)."""
    zdata, zsecs = read_binfile(zkey, "zkey", 2)
    zk = read_zkey_header(zdata, zsecs)
    ci = curve_from_q(zk["q"])
    ic = bytes(section(zdata, zsecs, 3))
    sG1 = 2 * ci.n8q
    return {"curve": ci, "nPublic": zk["nPublic"],
            "alpha1": ci.g1_from_affine_bytes(zk["vk_alpha_1"]), "beta2": ci.g2_from_affine_bytes(zk["vk_beta_2"]),
            "gamma2": ci.g2_from_affine_bytes(zk["vk_gamma_2"]), "delta2": ci.g2_from_affine_bytes(zk["vk_delta_2"]),
            "IC": [ci.g1_from_affine_bytes(ic[i * sG1:(i + 1) * sG1]) for i in range(zk["nPublic"] + 1)]}


# --- BN254 optimal-ate pairing over plain Python ints (verifier only; small inputs only) ---------------------
_Q = P_BN_Q


class _FQ12:
    """Fq[w]/(w^12 - 18 w^6 + 82); Fq2 embeds with u = w^6 - 9."""
    __slots__ = ("c",)
    MOD = (82, 0, 0, 0, 0, 0, -18, 0, 0, 0, 0, 0)

    def __init__(self, c):
        self.c = [x % _Q for x in c]

    @staticmethod
    def one():
        return _FQ12([1] + [0] * 11)

    def __add__(self, o): return _FQ12([a + b for a, b in zip(self.c, o.c)])
    def __sub__(self, o): return _FQ12([a - b for a, b in zip(self.c, o.c)])
    def __neg__(self): return _FQ12([-a for a in self.c])
    def __eq__(self, o): return self.c == o.c

    def scale(self, k): return _FQ12([a * k for a in self.c])

    def __mul__(self, o):
        b = [0] * 23
        for i, x in enumerate(self.c):
            if x:
                for j, y in enumerate(o.c):
                    b[i + j] += x * y
        for i in range(22, 11, -1):
            t = b[i]
            if t:
                b[i - 6] += 18 * t
                b[i - 12] -= 82 * t
        return _FQ12(b[:12])

    def __pow__(self, e):
        r, b = _FQ12.one(), self
        while e:
            if e & 1:
                r = r * b
            b = b * b
            e >>= 1
        return r

    def inv(self):
        # extended Euclid over Fq[x]
        lm, hm = [1] + [0] * 12, [0] * 13
        low, high = self.c + [0], [m % _Q for m in self.MOD] + [1]

        def deg(p):
            d = len(p) - 1
            while d and p[d] == 0:
                d -= 1
            return d

        def pdiv(a, b):
            da, db = deg(a), deg(b)
            t = list(a)
            o = [0] * len(a)
            ib = pow(b[db], -1, _Q)
            for i in range(da - db, -1, -1):
                o[i] = (o[i] + t[db + i] * ib) % _Q
                for c in range(db + 1):
                    t[c + i] = (t[c + i] - o[i] * b[c]) % _Q
            return o[:deg(o) + 1]

        while deg(low):
            r = pdiv(high, low)
            r += [0] * (13 - len(r))
            nm, new = list(hm), list(high)
            for i in range(13):
                for j in range(13 - i):
                    nm[i + j] -= lm[i] * r[j]
                    new[i + j] -= low[i] * r[j]
            nm = [x % _Q for x in nm]
            new = [x % _Q for x in new]
            lm, low, hm, high = nm, new, lm, low
        il = pow(low[0], -1, _Q)
        return _FQ12([x * il for x in lm[:12]])


def _fq12_from_fq(x): return _FQ12([x] + [0] * 11)


def _twist(pt):
    (x0, x1), (y0, y1) = pt
    nx = _FQ12([x0 - 9 * x1] + [0] * 5 + [x1] + [0] * 5)
    ny = _FQ12([y0 - 9 * y1] + [0] * 5 + [y1] + [0] * 5)
    w = _FQ12([0, 1] + [0] * 10)
    return (nx * w * w, ny * w * w * w)


def _ec12_double(p):
    x, y = p
    m = (x * x).scale(3) * (y.scale(2)).inv()
    nx = m * m - x.scale(2)
    return (nx, m * (x - nx) - y)


def _ec12_add(p, q):
    if p is None:
        return q
    if q is None:
        return p
    x1, y1 = p
    x2, y2 = q
    if x1 == x2:
        return _ec12_double(p) if y1 == y2 else None
    m = (y2 - y1) * (x2 - x1).inv()
    nx = m * m - x1 - x2
    return (nx, m * (x1 - nx) - y1)


def _linefunc(p1, p2, t):
    x1, y1 = p1
    x2, y2 = p2
    xt, yt = t
    if not (x1 == x2):
        m = (y2 - y1) * (x2 - x1).inv()
        return m * (xt - x1) - (yt - y1)
    if y1 == y2:
        m = (x1 * x1).scale(3) * (y1.scale(2)).inv()
        return m * (xt - x1) - (yt - y1)
    return xt - x1


_ATE = 29793968203157093288


def _miller(Q2, P1):
    """Miller loop of the optimal ate pairing (no final exponentiation)."""
    if Q2 is None or P1 is None:
        return _FQ12.one()
    Q = _twist(Q2)
    P = (_fq12_from_fq(P1[0]), _fq12_from_fq(P1[1]))
    R, f = Q, _FQ12.one()
    for i in range(63, -1, -1):
        f = f * f * _linefunc(R, R, P)
        R = _ec12_double(R)
        if _ATE & (1 << i):
            f = f * _linefunc(R, Q, P)
            R = _ec12_add(R, Q)
    Q1 = (Q[0] ** _Q, Q[1] ** _Q)
    nQ2 = (Q1[0] ** _Q, -(Q1[1] ** _Q))
    f = f * _linefunc(R, Q1, P)
    R = _ec12_add(R, Q1)
    f = f * _linefunc(R, nQ2, P)
    return f


def _final_exp(f):
    return f ** ((_Q ** 12 - 1) // P_BN_R)


def pairing_product_is_one(pairs) -> bool:
    """prod e(P_i, Q_i) == 1 for (G1 affine ints, G2 affine ints) pairs — BN254 only."""
    f = _FQ12.one()
    for p1, q2 in pairs:
        f = f * _miller(q2, p1)
    return _final_exp(f) == _FQ12.one()


def _g1_add_int(p, q):
    if p is None:
        return q
    if q is None:
        return p
    if p[0] == q[0]:
        if (p[1] + q[1]) % _Q == 0:
            return None
        m = 3 * p[0] * p[0] * pow(2 * p[1], -1, _Q) % _Q
    else:
        m = (q[1] - p[1]) * pow(q[0] - p[0], -1, _Q) % _Q
    x = (m * m - p[0] - q[0]) % _Q
    return (x, (m * (p[0] - x) - p[1]) % _Q)


def _g1_mul_int(p, k):
    r = None
    while k:
        if k & 1:
            r = _g1_add_int(r, p)
        p = _g1_add_int(p, p)
        k >>= 1
    return r


def groth16_verify(vk: dict, public_signals: List[int], proof: dict) -> bool:
    """src/groth16_verify.js:25-85: public inputs must be < r (aliasing check :41-46), then
    e(-A,B) e(alpha,beta) e(vk_x,gamma) e(C,delta) == 1.  BN254 through the pairing above, BLS12-381 through pairing_bls.py."""
    ci: CurveInfo = vk["curve"]
    if ci.id == BN254:
        add, mul, pairing, q, b = _g1_add_int, _g1_mul_int, pairing_product_is_one, _Q, 3
    else:
        from . import pairing_bls as pb
        add, mul, pairing, q, b = pb.g1_add, pb.g1_mul, pb.pairing_product_is_one, pb.Q, 4
    if len(public_signals) != vk["nPublic"]:
        return False
    for s in public_signals:
        if not (0 <= int(s) < ci.r):
            return False
    cpub = vk["IC"][0]
    for i, s in enumerate(public_signals):
        cpub = add(cpub, mul(vk["IC"][i + 1], int(s)))
    A = (int(proof["pi_a"][0]), int(proof["pi_a"][1]))
    B = ((int(proof["pi_b"][0][0]), int(proof["pi_b"][0][1])), (int(proof["pi_b"][1][0]), int(proof["pi_b"][1][1])))
    C = (int(proof["pi_c"][0]), int(proof["pi_c"][1]))
    negA = (A[0], (-A[1]) % q)
    # on-curve checks (G1.isValid / G2.isValid :48-63)
    if (A[1] * A[1] - A[0] ** 3 - b) % q or (C[1] * C[1] - C[0] ** 3 - b) % q:
        return False
    return pairing([(negA, B), (vk["alpha1"], vk["beta2"]), (cpub, vk["gamma2"]), (C, vk["delta2"])])
