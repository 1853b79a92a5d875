"""plonk.prove on the GPU — host-side mirror of src/plonk_prove.js:47-165.

ProvingKey(zkey) puts the PLONK key in HBM once (sb_plonk_load); prove() runs the five rounds on the device
(sb_plonk_prove: plonk.cuh kernels + NTT + table-mode MSM, transcript hashing on the host) and returns the same
{A, B, C, Z, T1, T2, T3, Wxi, Wxiw, eval_*} object and publicSignals the reference writes (src/proof.js:62-82).
The blinders b_1..b_11 may be injected as Montgomery field elements; otherwise they are drawn like Fr.random()."""
from __future__ import annotations

import ctypes
import struct

import numpy as np

from .curve import Curve, SbError, _arr, _ptr, getCurveFromQ
from .groth16 import KeyOnContexts, _from_mont, random_fr, read_binfile, read_wtns_header

POINTS = ("A", "B", "C", "Z", "T1", "T2", "T3", "Wxi", "Wxiw")
EVALS = ("eval_a", "eval_b", "eval_c", "eval_s1", "eval_s2", "eval_zw")


def read_zkey_header_plonk(data: bytes) -> dict:
    """src/zkey_utils.js:261-299"""
    secs = read_binfile(data, "zkey", 2)
    if struct.unpack_from("<I", data, secs[1][0])[0] != 2:
        raise SbError("zkey file is not plonk")                                    # src/plonk_prove.js:58-60
    p = secs[2][0]
    n8q = struct.unpack_from("<I", data, p)[0]
    q = int.from_bytes(data[p + 4:p + 4 + n8q], "little")
    n8r = struct.unpack_from("<I", data, p + 4 + n8q)[0]
    r = int.from_bytes(data[p + 8 + n8q:p + 8 + n8q + n8r], "little")
    o = p + 8 + n8q + n8r
    n_vars, n_public, domain, n_add, n_cons = struct.unpack_from("<IIIII", data, o)
    return {"protocol": "plonk", "n8q": n8q, "q": q, "n8r": n8r, "r": r, "nVars": n_vars, "nPublic": n_public,
            "domainSize": domain, "nAdditions": n_add, "nConstraints": n_cons, "power": domain.bit_length() - 1}


def proof_to_object(curve: Curve, raw: bytes) -> dict:
    """Proof.toObjectProof(false) + stringifyBigInts (src/proof.js:62-82, src/plonk_prove.js:153-163)."""
    n8, q = curve.n8q, curve.q
    out = {}
    for i, name in enumerate(POINTS):
        p = raw[2 * n8 * i:2 * n8 * (i + 1)]
        out[name] = ["0", "1", "0"] if p == bytes(2 * n8) else [str(_from_mont(p[:n8], q, n8)), str(_from_mont(p[n8:], q, n8)), "1"]
    base = 2 * n8 * len(POINTS)
    for i, name in enumerate(EVALS):
        out[name] = str(_from_mont(raw[base + 32 * i:base + 32 * (i + 1)], curve.r, 32))
    out["protocol"] = "plonk"
    out["curve"] = curve.name
    return out


def _prove_batch(curve: Curve, proto: str, n_blinders: int, witnesses, blinders_list, call) -> list:
    """prove_batch_raw of the PLONK and fflonk keys: checks the arguments, then call(witnesses, n_witness, count, blinders,
    proofs, status) (pointers and sizes) makes the device call.  One proof (bytes) per witness, None for a proof the
    reference would have rejected; SbError for argument and device errors."""
    parts = [_arr(x) for x in witnesses]
    count = len(parts)
    if len(blinders_list) != count:
        raise SbError("one blinder set per witness")
    if count == 0:
        return []
    for b in blinders_list:
        if len(b) != n_blinders * 32:
            raise SbError(f"blinders must be {n_blinders} field elements")
    n_wit = parts[0].size // 32
    for x in parts:
        if x.size != parts[0].size:
            raise SbError("witnesses of one batch must have the same length")
    w = np.concatenate(parts)
    bl = np.frombuffer(b"".join(bytes(b) for b in blinders_list), np.uint8)
    pb = getattr(curve.lib, f"sb_{proto}_proof_bytes")(curve.handle)
    out = np.empty(count * pb, np.uint8)
    status = np.zeros(count, np.int32)
    rc = call(_ptr(w), n_wit, count, _ptr(bl), _ptr(out), _ptr(status))
    if rc != 0 and not status.any():
        curve.check(rc)
    return [None if status[i] else out[i * pb:(i + 1) * pb].tobytes() for i in range(count)]


class ProvingKey:
    """A PLONK zkey resident on one device."""

    def __init__(self, zkey: bytes, curve: Curve | None = None, device: int = 0):
        zkey = bytes(zkey)
        self.header = read_zkey_header_plonk(zkey)
        self.curve = curve or getCurveFromQ(self.header["q"], device)
        self._own_curve = curve is None
        h = ctypes.c_uint64()
        buf = np.frombuffer(zkey, np.uint8)
        self.curve.check(self.curve.lib.sb_plonk_load(self.curve.handle, _ptr(buf), buf.size, ctypes.byref(h)))
        self.handle = h.value
        for k in ("nVars", "nPublic", "domainSize", "nAdditions"):
            setattr(self, k, self.header[k])

    @classmethod
    def from_file(cls, path: str, curve: Curve):
        """Loads the key from disk (sb_plonk_load_file: mapped read-only, streamed to HBM section by section)."""
        self = cls.__new__(cls)
        self.curve, self._own_curve = curve, False
        h = ctypes.c_uint64()
        curve.check(curve.lib.sb_plonk_load_file(curve.handle, path.encode(), ctypes.byref(h)))   # validates the container
        self.handle = h.value
        nv, npub, ds, na = ctypes.c_uint32(), ctypes.c_uint32(), ctypes.c_uint32(), ctypes.c_uint32()
        curve.check(curve.lib.sb_plonk_info(curve.handle, self.handle, ctypes.byref(nv), ctypes.byref(npub), ctypes.byref(ds), ctypes.byref(na)))
        self.nVars, self.nPublic, self.domainSize, self.nAdditions = nv.value, npub.value, ds.value, na.value
        self.header = {"protocol": "plonk", "r": curve.r, "q": curve.q, "nVars": nv.value, "nPublic": npub.value, "domainSize": ds.value,
                       "nAdditions": na.value, "power": ds.value.bit_length() - 1}
        return self

    def prove_raw(self, witness, blinders: bytes) -> bytes:
        """witness = wtns section 2 ((nVars - nAdditions) x 32 bytes, plain LE), or None to reuse the witness the previous
        proof on this key left in HBM (sb_plonk_prove_resident); blinders = 11 x 32 Montgomery bytes."""
        if len(blinders) != 11 * 32:
            raise SbError("blinders must be 11 field elements")
        lib, c = self.curve.lib, self.curve
        out = np.empty(lib.sb_plonk_proof_bytes(c.handle), np.uint8)
        if witness is None:
            c.check(lib.sb_plonk_prove_resident(c.handle, self.handle, bytes(blinders), _ptr(out)))
        else:
            w = _arr(witness)
            c.check(lib.sb_plonk_prove(c.handle, self.handle, _ptr(w), w.size // 32, bytes(blinders), _ptr(out)))
        return out.tobytes()

    def prove_batch_raw(self, witnesses, blinders_list) -> list:
        """One sb_plonk_prove_batch call: witnesses = wtns section-2 payloads ((nVars - nAdditions) x 32 bytes each),
        blinders_list = one 11 x 32-byte Montgomery blinder string per witness.  Returns one proof (bytes, as prove_raw) per
        witness, or None for a proof the reference would have rejected; raises SbError for argument and device errors."""
        return _prove_batch(self.curve, "plonk", 11, witnesses, blinders_list,
                            lambda w, n_wit, count, bl, out, st: self.curve.lib.sb_plonk_prove_batch(self.curve.handle, self.handle, w, n_wit, count, bl, out, st))

    def release(self):
        if self.handle:
            self.curve.lib.sb_plonk_release(self.curve.handle, self.handle)
            self.handle = 0
        if self._own_curve:
            self.curve.terminate()


class ShardedProvingKey(KeyOnContexts):
    """A PLONK zkey spread over several contexts so that one proof uses all of them (sb_plonk_load_multi /
    sb_plonk_prove_multi).  curves[0] is rank 0: it holds the key and runs the proof; every context holds a contiguous
    range of the PTau points and computes that part of each commitment.  curves are Curve objects of the key's curve
    (several may be on one device) or device indices, for which the key makes its own Curve and closes it on release().
    Proofs are byte-identical to ProvingKey.prove_raw with the same witness and blinders."""

    PROTO, LOAD, N_BLINDERS = "plonk", "load_multi", 11
    FIELDS = ("nVars", "nPublic", "domainSize", "nAdditions")
    read_header = staticmethod(read_zkey_header_plonk)
    to_object = staticmethod(proof_to_object)

    def prove_raw(self, witness, blinders: bytes) -> bytes:
        """witness = wtns section 2 ((nVars - nAdditions) x 32 bytes, plain LE); blinders = N_BLINDERS x 32 Montgomery bytes."""
        if len(blinders) != self.N_BLINDERS * 32:
            raise SbError(f"blinders must be {self.N_BLINDERS} field elements")
        if witness is None:
            raise SbError("a sharded key proves from a host witness only")
        c = self.curves[0]
        out = np.empty(getattr(c.lib, f"sb_{self.PROTO}_proof_bytes")(c.handle), np.uint8)
        w = _arr(witness)
        c.check(getattr(c.lib, f"sb_{self.PROTO}_prove_multi")(self._ctxs, self.handles, len(self.curves), _ptr(w), w.size // 32,
                                                                bytes(blinders), _ptr(out)))
        return out.tobytes()

    def prove(self, wtns: bytes, blinders: bytes | None = None):
        """(proof, publicSignals) as the module's prove."""
        wh, W = read_wtns_header(bytes(wtns))
        if wh["q"] != self.header["r"]:
            raise SbError("Curve of the witness does not match the curve of the proving key")
        if blinders is None:
            blinders = b"".join(random_fr(self.curve) for _ in range(self.N_BLINDERS))
        raw = self.prove_raw(np.frombuffer(W, np.uint8), blinders)
        pub = [str(int.from_bytes(W[i * 32:(i + 1) * 32], "little")) for i in range(1, self.nPublic + 1)]
        return self.to_object(self.curve, raw), pub


class ReplicatedProvingKey(KeyOnContexts):
    """A PLONK zkey loaded whole on several contexts (sb_plonk_load_replicas), so that a batch of proofs is split over
    them (sb_plonk_prove_batch_multi): context i proves a contiguous share of the batch.  curves as for
    ShardedProvingKey."""

    PROTO, LOAD, N_BLINDERS = "plonk", "load_replicas", 11
    FIELDS = ("nVars", "nPublic", "domainSize", "nAdditions")
    read_header = staticmethod(read_zkey_header_plonk)

    def prove_batch_raw(self, witnesses, blinders_list) -> list:
        """As ProvingKey.prove_batch_raw, over every context: the proofs and statuses are those of one context's batch."""
        fn = getattr(self.curve.lib, f"sb_{self.PROTO}_prove_batch_multi")
        return _prove_batch(self.curve, self.PROTO, self.N_BLINDERS, witnesses, blinders_list,
                            lambda w, n_wit, count, bl, out, st: fn(self._ctxs, self.handles, len(self.curves), w, n_wit, count, bl, out, st))


def prove(zkey, wtns: bytes, blinders: bytes | None = None, logger=None, options=None):
    """plonk16Prove(zkeyFileName, witnessFileName) -> (proof, publicSignals); zkey may be bytes or a ProvingKey."""
    pk = zkey if isinstance(zkey, ProvingKey) else ProvingKey(zkey)
    try:
        wh, W = read_wtns_header(bytes(wtns))
        if wh["q"] != pk.header["r"]:
            raise SbError("Curve of the witness does not match the curve of the proving key")          # :62-64
        if blinders is None:
            blinders = b"".join(random_fr(pk.curve) for _ in range(11))                                  # :246-249
        raw = pk.prove_raw(np.frombuffer(W, np.uint8), blinders)                                         # length check in C (:66-68)
        pub = [str(int.from_bytes(W[i * 32:(i + 1) * 32], "little")) for i in range(1, pk.nPublic + 1)]
        return proof_to_object(pk.curve, raw), pub
    finally:
        if not isinstance(zkey, ProvingKey):
            pk.release()


def prove_batch(zkey, wtns_list, blinders=None):
    """plonk16Prove over many witnesses of one circuit in one device call: [(proof, publicSignals), ...] in the order of
    wtns_list.  zkey may be bytes or a ProvingKey; every .wtns container is checked as prove checks it; blinders = one
    11 x 32-byte Montgomery string per witness, drawn like Fr.random() when not given.  A witness the reference would
    reject raises SbError with the reference's text for the first such witness."""
    pk = zkey if isinstance(zkey, ProvingKey) else ProvingKey(zkey)
    try:
        ws = []
        for wtns in wtns_list:
            wh, W = read_wtns_header(bytes(wtns))
            if wh["q"] != pk.header["r"]:
                raise SbError("Curve of the witness does not match the curve of the proving key")          # :62-64
            ws.append(W)
        if blinders is None:
            blinders = [b"".join(random_fr(pk.curve) for _ in range(11)) for _ in ws]                     # :246-249
        if len(blinders) != len(ws):
            raise SbError("one blinder set per witness")
        raws = pk.prove_batch_raw([np.frombuffer(W, np.uint8) for W in ws], blinders)                   # length check in C (:66-68)
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


# ------------------------------------------------------------------ verification (src/plonk_verify.js:29-421)
# status -> (log level, the reference's message); 5 is the wrappers' own: a signal count other than nPublic never reaches
# the device, because the C entry takes one n_public for the whole batch
VERIFY_MESSAGES = {1: ("warn", "Invalid Proof"), 2: ("error", "Public inputs are not valid."),
                   3: ("error", "Proof commitments are not valid."), 4: ("error", "Proof evaluations are not valid"),
                   5: ("error", "Invalid number of public inputs")}
WRONG_COUNT = 5


def fr_root(r: int, k: int) -> int:
    """Fr.w[k] (build/snarkjs.js:12866-12889): nqr = the first non-residue from 2, w[s] = nqr^((r-1)/2^s) for the
    2-adicity s, w[k] = w[s]^(2^(s-k))."""
    s = ((r - 1) & -(r - 1)).bit_length() - 1
    if not 0 <= k <= s:
        raise SbError(f"power {k} is above the 2-adicity {s} of Fr")
    nqr = 2
    while pow(nqr, (r - 1) // 2, r) != r - 1:
        nqr += 1
    return pow(nqr, ((r - 1) >> s) << (s - k), r)


def fr_bytes(v, r: int) -> bytes:
    """Fr.fromObject (build/snarkjs.js:13042-13046): the value written into 32 bytes (toRprLE, :198, silently mod 2^256),
    then toMontgomery, which reduces it mod r.  So a JSON evaluation of eval + r, or eval + 2^256, is eval."""
    return ((int(v) % (1 << 256)) % r * (1 << 256) % r).to_bytes(32, "little")


def _g1_valid(pb: bytes, n8: int, q: int) -> bool:
    """G1.isValid of affine Montgomery bytes (point_bytes output: coordinates already below q)."""
    if pb == bytes(2 * n8):
        return True
    x, y = _from_mont(pb[:n8], q, n8), _from_mont(pb[n8:], q, n8)
    return (y * y - x * x * x - (3 if n8 == 32 else 4)) % q == 0


def _g1_json(p: bytes, n8: int, q: int) -> list:
    return ["0", "1", "0"] if p == bytes(2 * n8) else [str(_from_mont(p[:n8], q, n8)), str(_from_mont(p[n8:], q, n8)), "1"]


def _g2_json(p: bytes, n8: int, q: int) -> list:
    if p == bytes(4 * n8):
        return [["0", "0"], ["1", "0"], ["0", "0"]]
    f = lambda i: str(_from_mont(p[i * n8:(i + 1) * n8], q, n8))
    return [[f(0), f(1)], [f(2), f(3)], ["1", "0"]]


def _vk_header(zkey, proto: str) -> tuple:
    """(header dict, byte offset of k1 in section 2) of a PLONK or fflonk zkey."""
    from .fflonk import read_zkey_header_fflonk
    data = bytes(zkey)
    z = read_zkey_header_plonk(data) if proto == "plonk" else read_zkey_header_fflonk(data)
    secs = read_binfile(data, "zkey", 2)
    return data, z, secs[2][0] + 8 + z["n8q"] + z["n8r"] + 20


def verification_key(zkey) -> dict:
    """zkey export verificationkey for a PLONK key (src/zkey_export_verificationkey.js:92-117), as decimal strings."""
    data, z, o = _vk_header(zkey, "plonk")
    n8, q, r = z["n8q"], z["q"], z["r"]
    fr = lambda i: str(_from_mont(data[o + 32 * i:o + 32 * (i + 1)], r, 32))
    vk = {"protocol": "plonk", "curve": "bn128" if n8 == 32 else "bls12381", "nPublic": z["nPublic"], "power": z["power"],
          "k1": fr(0), "k2": fr(1)}
    o += 64
    for i, name in enumerate(("Qm", "Ql", "Qr", "Qo", "Qc", "S1", "S2", "S3")):
        vk[name] = _g1_json(data[o + 2 * n8 * i:o + 2 * n8 * (i + 1)], n8, q)
    o += 16 * n8
    vk["X_2"] = _g2_json(data[o:o + 4 * n8], n8, q)
    vk["w"] = str(fr_root(r, z["power"]))
    return vk


def vk_bytes(vk: dict) -> bytes:
    """The verification key as sb_plonk_verify_batch takes it: Qm Ql Qr Qo Qc S1 S2 S3 || X_2 || k1 || k2."""
    from .groth16 import _curve_of, point_bytes
    n8, q, r, _name = _curve_of(vk["curve"])
    return (b"".join(point_bytes(vk[k], 1, n8, q) for k in ("Qm", "Ql", "Qr", "Qo", "Qc", "S1", "S2", "S3"))
            + point_bytes(vk["X_2"], 2, n8, q) + fr_bytes(vk["k1"], r) + fr_bytes(vk["k2"], r))


def proof_bytes(proof: dict, n8: int, q: int, r: int) -> bytes:
    """A JSON proof as sb_plonk_prove writes it: the nine points, then the six evaluations (Montgomery, as fr_bytes)."""
    from .groth16 import point_bytes
    return b"".join(point_bytes(proof[k], 1, n8, q) for k in POINTS) + b"".join(fr_bytes(proof[k], r) for k in EVALS)


def _verify_status(fn: str, vk: dict, vkb: bytes | None, items, encode, n_points: int, count_first: bool, curve) -> list:
    """The statuses of [(publicSignals, proof), ...] for sb_plonk_verify_batch / sb_fflonk_verify_batch (fn).  vkb = None: a
    key point the reference checks per proof (fflonk's C0) is not valid, so every proof fails with 3.  Items the device
    call cannot take (a signal count other than nPublic, a signal outside [0, r)) are decided here, with the reference's
    check order: the count first for fflonk (count_first), after the commitments for PLONK."""
    from .groth16 import _curve_of, publics_bytes
    n8, q, r, name = _curve_of(vk["curve"])
    n_public, power = int(vk["nPublic"]), int(vk["power"])
    status = [None] * len(items)
    pubs, prfs, slots = [], [], []
    for k, (signals, proof) in enumerate(items):
        prf = encode(proof, n8, q, r)
        points_ok = lambda: all(_g1_valid(prf[2 * n8 * i:2 * n8 * (i + 1)], n8, q) for i in range(n_points))
        if count_first and len(signals) != n_public:
            status[k] = WRONG_COUNT
        elif vkb is None:
            status[k] = 3
        elif len(signals) != n_public:
            status[k] = WRONG_COUNT if points_ok() else 3
        else:
            pb = publics_bytes(signals, r)
            if pb is None:                    # evaluations from JSON are always below r (fr_bytes), so 4 cannot come first
                status[k] = 2 if points_ok() else 3
            else:
                pubs.append(pb)
                prfs.append(prf)
                slots.append(k)
    if not slots:
        return status
    own = curve is None
    cv = curve or Curve(name)
    try:
        count = len(slots)
        out = np.zeros(count, np.int32)
        key = np.frombuffer(vkb, np.uint8)
        pub = np.frombuffer(b"".join(pubs) or b"\0", np.uint8)
        prf = np.frombuffer(b"".join(prfs), np.uint8)
        cv.check(getattr(cv.lib, fn)(cv.handle, _ptr(key), key.size, n_public, power, _ptr(pub), _ptr(prf), count,
                                     out.ctypes.data_as(ctypes.c_void_p)))
    finally:
        if own:
            cv.terminate()
    for j, k in enumerate(slots):
        status[k] = int(out[j])
    return status


def _log_status(logger, messages: dict, s: int, ok: str):
    if not logger:
        return
    if s == 0:
        logger.info(ok)
        return
    if s != 1:
        logger.error(messages[s][1])
    else:
        getattr(logger, messages[1][0])(messages[1][1])


def verify_status(vk_verifier: dict, items, curve: Curve | None = None) -> list:
    """sb_plonk_verify_batch over [(publicSignals, proof), ...]: one status per item (0 verifies, else a key of
    VERIFY_MESSAGES)."""
    return _verify_status("sb_plonk_verify_batch", vk_verifier, vk_bytes(vk_verifier), items, proof_bytes, len(POINTS), False, curve)


def verify_batch(vk_verifier: dict, items, logger=None, curve: Curve | None = None) -> list:
    """plonkVerify over many (publicSignals, proof) pairs against one verification key, in one device call -> [bool]."""
    st = verify_status(vk_verifier, items, curve)
    for s in st:
        _log_status(logger, VERIFY_MESSAGES, s, "OK!")
    return [s == 0 for s in st]


def verify(vk_verifier: dict, publicSignals, proof: dict, logger=None, curve: Curve | None = None) -> bool:
    """plonkVerify(vk_verifier, publicSignals, proof, logger) (src/plonk_verify.js:29-124): True, or False with the
    reference's log message.  Two divergences: without a logger the reference throws on invalid commitments (its
    logger.error call there is unguarded), and this returns False; a key point (Qm .. S3, X_2) off its curve raises
    SbError, because sb_plonk_verify_batch refuses such a key, where the reference decodes the key without checking it
    and returns a verdict.  verify_batch and verify_status raise alike."""
    s = verify_status(vk_verifier, [(publicSignals, proof)], curve)[0]
    _log_status(logger, VERIFY_MESSAGES, s, "OK!")
    return s == 0
