"""fflonk.prove on the GPU — host-side mirror of src/fflonk_prove.js:51-267.

ProvingKey(zkey) puts the fflonk key in HBM once (sb_fflonk_load); prove() runs the five rounds on the device
(sb_fflonk_prove) and returns the {polynomials: {C1, C2, W1, W2}, evaluations: {ql .. t2w, inv}} object and the
publicSignals the reference writes (src/proof.js:62-82, fflonk_prove.js:240-262).  The blinders b_1..b_9 may be injected
as Montgomery field elements; otherwise they are drawn like Fr.random().  BN254 only, like the reference."""
from __future__ import annotations

import ctypes
import struct

import numpy as np

from .curve import Curve, SbError, _arr, _ptr, getCurveFromQ
from .groth16 import _from_mont, random_fr, read_binfile, read_wtns_header
from .plonk import ReplicatedProvingKey as _PlonkReplicated
from .plonk import ShardedProvingKey as _PlonkSharded
from .plonk import _prove_batch

POINTS = ("C1", "C2", "W1", "W2")
EVALS = ("ql", "qr", "qm", "qo", "qc", "s1", "s2", "s3", "a", "b", "c", "z", "zw", "t1w", "t2w", "inv")


def read_zkey_header_fflonk(data: bytes) -> dict:
    """src/zkey_utils.js:301-339"""
    secs = read_binfile(data, "zkey", 2)
    if struct.unpack_from("<I", data, secs[1][0])[0] != 10:
        raise SbError("zkey file is not fflonk")                                   # src/fflonk_prove.js:71-73
    p = secs[2][0]
    n8q = struct.unpack_from("<I", data, p)[0]
    q = int.from_bytes(data[p + 4:p + 4 + n8q], "little")
    n8r = struct.unpack_from("<I", data, p + 4 + n8q)[0]
    r = int.from_bytes(data[p + 8 + n8q:p + 8 + n8q + n8r], "little")
    o = p + 8 + n8q + n8r
    n_vars, n_public, domain, n_add, n_cons = struct.unpack_from("<IIIII", data, o)
    return {"protocol": "fflonk", "n8q": n8q, "q": q, "n8r": n8r, "r": r, "nVars": n_vars, "nPublic": n_public,
            "domainSize": domain, "nAdditions": n_add, "nConstraints": n_cons, "power": domain.bit_length() - 1}


def proof_to_object(curve: Curve, raw: bytes) -> dict:
    """Proof.toObjectProof() + stringifyBigInts (src/proof.js:62-82)."""
    n8, q = curve.n8q, curve.q
    pols = {}
    for i, name in enumerate(POINTS):
        p = raw[2 * n8 * i:2 * n8 * (i + 1)]
        pols[name] = ["0", "1", "0"] if p == bytes(2 * n8) else [str(_from_mont(p[:n8], q, n8)), str(_from_mont(p[n8:], q, n8)), "1"]
    base = 2 * n8 * len(POINTS)
    evs = {name: str(_from_mont(raw[base + 32 * i:base + 32 * (i + 1)], curve.r, 32)) for i, name in enumerate(EVALS)}
    return {"polynomials": pols, "evaluations": evs, "protocol": "fflonk", "curve": curve.name}


class ProvingKey:
    """An fflonk zkey resident on one device."""

    def __init__(self, zkey: bytes, curve: Curve | None = None, device: int = 0):
        zkey = bytes(zkey)
        self.header = read_zkey_header_fflonk(zkey)
        self.curve = curve or getCurveFromQ(self.header["q"], device)
        self._own_curve = curve is None
        h = ctypes.c_uint64()
        buf = np.frombuffer(zkey, np.uint8)
        self.curve.check(self.curve.lib.sb_fflonk_load(self.curve.handle, _ptr(buf), buf.size, ctypes.byref(h)))
        self.handle = h.value
        for k in ("nVars", "nPublic", "domainSize", "nAdditions"):
            setattr(self, k, self.header[k])

    @classmethod
    def from_file(cls, path: str, curve: Curve):
        """Loads the key from disk (sb_fflonk_load_file: mapped read-only, streamed to HBM section by section)."""
        self = cls.__new__(cls)
        self.curve, self._own_curve = curve, False
        h = ctypes.c_uint64()
        curve.check(curve.lib.sb_fflonk_load_file(curve.handle, path.encode(), ctypes.byref(h)))   # validates the container
        self.handle = h.value
        nv, npub, ds, na = ctypes.c_uint32(), ctypes.c_uint32(), ctypes.c_uint32(), ctypes.c_uint32()
        curve.check(curve.lib.sb_fflonk_info(curve.handle, self.handle, ctypes.byref(nv), ctypes.byref(npub), ctypes.byref(ds), ctypes.byref(na)))
        self.nVars, self.nPublic, self.domainSize, self.nAdditions = nv.value, npub.value, ds.value, na.value
        self.header = {"protocol": "fflonk", "r": curve.r, "q": curve.q, "nVars": nv.value, "nPublic": npub.value, "domainSize": ds.value,
                       "nAdditions": na.value, "power": ds.value.bit_length() - 1}
        return self

    def prove_raw(self, witness, blinders: bytes) -> bytes:
        """witness = wtns section 2 ((nVars - nAdditions) x 32 bytes, plain LE), or None to reuse the witness the previous
        proof on this key left in HBM (sb_fflonk_prove_resident); blinders = 9 x 32 Montgomery bytes."""
        if len(blinders) != 9 * 32:
            raise SbError("blinders must be 9 field elements")
        lib, c = self.curve.lib, self.curve
        out = np.empty(lib.sb_fflonk_proof_bytes(c.handle), np.uint8)
        if witness is None:
            c.check(lib.sb_fflonk_prove_resident(c.handle, self.handle, bytes(blinders), _ptr(out)))
        else:
            w = _arr(witness)
            c.check(lib.sb_fflonk_prove(c.handle, self.handle, _ptr(w), w.size // 32, bytes(blinders), _ptr(out)))
        return out.tobytes()

    def prove_batch_raw(self, witnesses, blinders_list) -> list:
        """One sb_fflonk_prove_batch call: witnesses = wtns section-2 payloads ((nVars - nAdditions) x 32 bytes each),
        blinders_list = one 9 x 32-byte Montgomery blinder string per witness.  Returns one proof (bytes, as prove_raw) per
        witness, or None for a proof the reference would have rejected; raises SbError for argument and device errors."""
        return _prove_batch(self.curve, "fflonk", 9, witnesses, blinders_list,
                            lambda w, n_wit, count, bl, out, st: self.curve.lib.sb_fflonk_prove_batch(self.curve.handle, self.handle, w, n_wit, count, bl, out, st))

    def release(self):
        if self.handle:
            self.curve.lib.sb_fflonk_release(self.curve.handle, self.handle)
            self.handle = 0
        if self._own_curve:
            self.curve.terminate()


class ShardedProvingKey(_PlonkSharded):
    """An fflonk zkey spread over several contexts so that one proof uses all of them (sb_fflonk_load_multi /
    sb_fflonk_prove_multi), with the interface of plonk.ShardedProvingKey: curves[0] is rank 0, every context holds a
    range of the 9n + 18 PTau points and its part of each commitment; curves may also be device indices."""

    PROTO, N_BLINDERS = "fflonk", 9
    read_header = staticmethod(read_zkey_header_fflonk)
    to_object = staticmethod(proof_to_object)


class ReplicatedProvingKey(_PlonkReplicated):
    """An fflonk zkey loaded whole on several contexts (sb_fflonk_load_replicas), so that a batch of proofs is split over
    them (sb_fflonk_prove_batch_multi), with the interface of plonk.ReplicatedProvingKey."""

    PROTO, N_BLINDERS = "fflonk", 9
    read_header = staticmethod(read_zkey_header_fflonk)


def prove(zkey, wtns: bytes, blinders: bytes | None = None, logger=None, options=None):
    """fflonkProve(zkeyFileName, witnessFileName) -> (proof, publicSignals); zkey may be bytes or a ProvingKey."""
    pk = zkey if isinstance(zkey, ProvingKey) else ProvingKey(zkey)
    try:
        wh, W = read_wtns_header(bytes(wtns))
        if wh["q"] != pk.header["r"]:
            raise SbError("Curve of the witness does not match the curve of the proving key")          # :75-77
        if blinders is None:
            blinders = b"".join(random_fr(pk.curve) for _ in range(9))                                   # :321-324
        raw = pk.prove_raw(np.frombuffer(W, np.uint8), blinders)
        pub = [str(int.from_bytes(W[i * 32:(i + 1) * 32], "little")) for i in range(1, pk.nPublic + 1)]
        return proof_to_object(pk.curve, raw), pub
    finally:
        if not isinstance(zkey, ProvingKey):
            pk.release()


def prove_batch(zkey, wtns_list, blinders=None):
    """fflonkProve over many witnesses of one circuit in one device call: [(proof, publicSignals), ...] in the order of
    wtns_list.  zkey may be bytes or a ProvingKey; every .wtns container is checked as prove checks it; blinders = one
    9 x 32-byte Montgomery string per witness, drawn like Fr.random() when not given.  A witness the reference would
    reject raises SbError with the reference's text for the first such witness."""
    pk = zkey if isinstance(zkey, ProvingKey) else ProvingKey(zkey)
    try:
        ws = []
        for wtns in wtns_list:
            wh, W = read_wtns_header(bytes(wtns))
            if wh["q"] != pk.header["r"]:
                raise SbError("Curve of the witness does not match the curve of the proving key")          # :75-77
            ws.append(W)
        if blinders is None:
            blinders = [b"".join(random_fr(pk.curve) for _ in range(9)) for _ in ws]                      # :321-324
        if len(blinders) != len(ws):
            raise SbError("one blinder set per witness")
        raws = pk.prove_batch_raw([np.frombuffer(W, np.uint8) for W in ws], blinders)                   # length check in C (:79-81)
        if any(r is None for r in raws):
            raise SbError(pk.curve.lib.sb_last_error(pk.curve.handle).decode())
        out = []
        for W, raw in zip(ws, raws):
            pub = [str(int.from_bytes(W[i * 32:(i + 1) * 32], "little")) for i in range(1, pk.nPublic + 1)]
            out.append((proof_to_object(pk.curve, raw), pub))
        return out
    finally:
        if not isinstance(zkey, ProvingKey):
            pk.release()


# ------------------------------------------------------------------ verification (src/fflonk_verify.js:28-597)
# status -> (log level, the reference's message), as plonk.VERIFY_MESSAGES
VERIFY_MESSAGES = {1: ("warn", "Invalid Proof"), 2: ("error", "Public inputs are not valid."),
                   3: ("error", "Proof commitments are not valid"), 4: ("error", "Proof evaluations are not valid."),
                   5: ("error", "Number of public signals does not match with vk")}
VK_FR = ("k1", "k2", "w", "w3", "w4", "w8", "wr")


def verification_key(zkey) -> dict:
    """zkey export verificationkey for an fflonk key (src/zkey_export_verificationkey.js:119-148), as decimal strings."""
    from .plonk import _g1_json, _g2_json, _vk_header, fr_root
    data, z, o = _vk_header(zkey, "fflonk")
    n8, q, r = z["n8q"], z["q"], z["r"]
    fr = [str(_from_mont(data[o + 32 * i:o + 32 * (i + 1)], r, 32)) for i in range(6)]   # k1 k2 w3 w4 w8 wr
    o += 6 * 32
    vk = {"protocol": "fflonk", "curve": "bn128" if n8 == 32 else "bls12381", "nPublic": z["nPublic"], "power": z["power"],
          "k1": fr[0], "k2": fr[1], "w": str(fr_root(r, z["power"])), "w3": fr[2], "w4": fr[3], "w8": fr[4], "wr": fr[5],
          "X_2": _g2_json(data[o:o + 4 * n8], n8, q), "C0": _g1_json(data[o + 4 * n8:o + 6 * n8], n8, q)}
    return vk


def vk_bytes(vk: dict) -> bytes:
    """The verification key as sb_fflonk_verify_batch takes it: C0 || X_2 || k1 k2 w w3 w4 w8 wr."""
    from .groth16 import _curve_of, point_bytes
    from .plonk import fr_bytes
    n8, q, r, _name = _curve_of(vk["curve"])
    return point_bytes(vk["C0"], 1, n8, q) + point_bytes(vk["X_2"], 2, n8, q) + b"".join(fr_bytes(vk[k], r) for k in VK_FR)


def proof_bytes(proof: dict, n8: int, q: int, r: int) -> bytes:
    """A JSON proof as sb_fflonk_prove writes it: C1 C2 W1 W2, then the 16 evaluations (Montgomery, as plonk.fr_bytes)."""
    from .groth16 import point_bytes
    from .plonk import fr_bytes
    ev = proof["evaluations"]
    return (b"".join(point_bytes(proof["polynomials"][k], 1, n8, q) for k in POINTS)
            + b"".join(fr_bytes(ev.get(k, 0), r) for k in EVALS))


def verify_status(vk_verifier: dict, items, curve: Curve | None = None) -> list:
    """sb_fflonk_verify_batch over [(publicSignals, proof), ...]: one status per item (0 verifies, else a key of
    VERIFY_MESSAGES).  A C0 that is not on the curve fails every item with 3, as the reference checks vk.C0 per proof."""
    from .groth16 import _curve_of
    from .plonk import _g1_valid, _verify_status
    n8, q, _r, _name = _curve_of(vk_verifier["curve"])
    vkb = vk_bytes(vk_verifier)
    if not _g1_valid(vkb[:2 * n8], n8, q):
        vkb = None
    return _verify_status("sb_fflonk_verify_batch", vk_verifier, vkb, items, proof_bytes, len(POINTS), True, curve)


def verify_batch(vk_verifier: dict, items, logger=None, curve: Curve | None = None) -> list:
    """fflonkVerify over many (publicSignals, proof) pairs against one verification key, in one device call -> [bool]."""
    from .plonk import _log_status
    st = verify_status(vk_verifier, items, curve)
    for s in st:
        _log_status(logger, VERIFY_MESSAGES, s, "PROOF VERIFIED SUCCESSFULLY")
    return [s == 0 for s in st]


def verify(vk_verifier: dict, publicSignals, proof: dict, logger=None, curve: Curve | None = None) -> bool:
    """fflonkVerify(vk_verifier, publicSignals, proof, logger) (src/fflonk_verify.js:28-137): True, or False with the
    reference's log message.  Two divergences: without a logger the reference throws on a signal count other than
    nPublic (its logger.error call there is unguarded), and this returns False; an X_2 off its curve raises SbError,
    because sb_fflonk_verify_batch refuses such a key, where the reference decodes X_2 without checking it and returns a
    verdict (an invalid C0 is the reference's own per-proof check, status 3).  verify_batch and verify_status raise
    alike."""
    from .plonk import _log_status
    s = verify_status(vk_verifier, [(publicSignals, proof)], curve)[0]
    _log_status(logger, VERIFY_MESSAGES, s, "PROOF VERIFIED SUCCESSFULLY")
    return s == 0
