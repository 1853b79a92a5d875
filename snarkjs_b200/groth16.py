"""groth16.prove on the GPU — host-side mirror of src/groth16_prove.js:28-144.

Two routes, same results:
  * prove(...)            fused path: sb_groth16_load once per zkey + sb_groth16_prove per witness (QAP, NTTs, MSMs all
                          in HBM); this is what bench.py measures.
  * prove_dropin(...)     the reference's own call sequence through the curve object's bulk methods
                          (Fr.ifft / batchApplyKey / fft, qap join, G1/G2.multiExpAffine with host buffers) — what the
                          N-API shim gives an unmodified snarkjs.
(r, s) may be injected as 32-byte Montgomery Fr elements; otherwise they are drawn like Fr.random() (:103-104)."""
from __future__ import annotations

import ctypes
import os
import struct

import numpy as np

from . import _native as N
from .curve import Curve, SbError, _arr, _ptr, getCurveFromQ


# ------------------------------------------------------------------ container readers (binfileutils 17468-17598)
def read_binfile(data: bytes, magic: str, max_version: int):
    if data[:4] != magic.encode():
        raise SbError(f"{magic}: Invalid File format")
    ver, nsec = struct.unpack_from("<II", data, 4)
    if ver > max_version:
        raise SbError("Version not supported")
    pos, secs = 12, {}
    for _ in range(nsec):
        sid, ln = struct.unpack_from("<IQ", data, pos)
        pos += 12
        if sid in secs:
            raise SbError(f"Section Duplicated {sid}")
        secs[sid] = (pos, ln)
        pos += ln
    if pos != len(data):
        raise SbError("Invalid file size")
    return secs


def read_wtns_header(data: bytes):
    """src/wtns_utils.js:62-72"""
    secs = read_binfile(data, "wtns", 2)
    p, _ = secs[1]
    n8 = struct.unpack_from("<I", data, p)[0]
    q = int.from_bytes(data[p + 4:p + 4 + n8], "little")
    nw = struct.unpack_from("<I", data, p + 4 + n8)[0]
    wp, wl = secs[2]
    return {"n8": n8, "q": q, "nWitness": nw}, memoryview(data)[wp:wp + wl]


def read_zkey_header_groth16(data: bytes):
    """src/zkey_utils.js:229-259"""
    secs = read_binfile(data, "zkey", 2)
    if struct.unpack_from("<I", data, secs[1][0])[0] != 1:
        raise SbError("zkey file is not groth16")
    p = secs[2][0]
    n8q = struct.unpack_from("<I", data, p)[0]
    q = int.from_bytes(data[p + 4:p + 4 + n8q], "little")
    n8r = struct.unpack_from("<I", data, p + 4 + n8q)[0]
    r = int.from_bytes(data[p + 8 + n8q:p + 8 + n8q + n8r], "little")
    o = p + 8 + n8q + n8r
    nVars, nPublic, domainSize = struct.unpack_from("<III", data, o)
    o += 12
    z = {"n8q": n8q, "q": q, "n8r": n8r, "r": r, "nVars": nVars, "nPublic": nPublic, "domainSize": domainSize,
         "power": domainSize.bit_length() - 1, "sections": secs}
    for name, sz in (("vk_alpha_1", 2 * n8q), ("vk_beta_1", 2 * n8q), ("vk_beta_2", 4 * n8q), ("vk_gamma_2", 4 * n8q),
                     ("vk_delta_1", 2 * n8q), ("vk_delta_2", 4 * n8q)):
        z[name] = bytes(data[o:o + sz])
        o += sz
    return z


def random_fr(curve: Curve) -> bytes:
    """Fr.random(): a uniform value below r, used directly as the Montgomery representation (13019-13035)."""
    nbytes = 32
    while True:
        v = int.from_bytes(os.urandom(nbytes), "little") >> (256 - curve.r.bit_length())
        if v < curve.r:
            return v.to_bytes(32, "little")


def _from_mont(x: bytes, p: int, n8: int) -> int:
    return int.from_bytes(x, "little") * pow(1 << (8 * n8), -1, p) % p


def proof_to_object(curve: Curve, affine: bytes) -> dict:
    """G.toObject + stringifyBigInts (src/groth16_prove.js:130-141)."""
    n8, q = curve.n8q, curve.q
    f = lambda b: str(_from_mont(b, q, n8))
    a, b, c = affine[:2 * n8], affine[2 * n8:6 * n8], affine[6 * n8:8 * n8]

    def g1(p):
        return ["0", "1", "0"] if p == bytes(2 * n8) else [f(p[:n8]), f(p[n8:]), "1"]

    def g2(p):
        if p == bytes(4 * n8):
            return [["0", "0"], ["1", "0"], ["0", "0"]]
        return [[f(p[:n8]), f(p[n8:2 * n8])], [f(p[2 * n8:3 * n8]), f(p[3 * n8:])], ["1", "0"]]

    return {"pi_a": g1(a), "pi_b": g2(b), "pi_c": g1(c), "protocol": "groth16", "curve": curve.name}


def _batch_inputs(n_vars: int, witnesses, rs):
    """(witnesses back to back, r's, s's, count) from prove_batch_raw's arguments, checked as the batch entries need them."""
    count = len(rs)
    if isinstance(witnesses, (list, tuple)):
        if len(witnesses) != count:
            raise SbError(f"{len(witnesses)} witnesses but {count} (r, s) pairs")
        parts = [_arr(x) for x in witnesses]
        for x in parts:
            if x.size != 32 * n_vars:
                raise SbError(f"Invalid witness length. Circuit: {n_vars}, witness: {x.size // 32}")
        w = np.concatenate(parts) if parts else np.zeros(0, np.uint8)
    else:
        w = _arr(witnesses)
        if w.size != 32 * n_vars * count:
            raise SbError(f"{w.size} witness bytes are not {count} witnesses of {n_vars} elements")
    if count == 0:
        return w, None, None, 0
    r = np.frombuffer(b"".join(bytes(x[0]) for x in rs), np.uint8)
    s = np.frombuffer(b"".join(bytes(x[1]) for x in rs), np.uint8)
    if r.size != 32 * count or s.size != 32 * count:
        raise SbError("r and s must be 32-byte Fr elements")
    return w, r, s, count


class KeyOnContexts:
    """A zkey loaded on several contexts by one sb_<PROTO>_<LOAD> call.  curves are Curve objects of the key's curve
    (several may be on one device) or device indices, for which the key makes its own Curve and closes it on release().
    curves[0] is rank 0: errors of the multi-context calls are reported on it."""

    PROTO, LOAD = "groth16", "load_replicas"
    FIELDS = ("nVars", "nPublic", "domainSize")
    read_header = staticmethod(read_zkey_header_groth16)

    def __init__(self, zkey: bytes, curves):
        zkey = bytes(zkey)
        self.header = self.read_header(zkey)
        if not curves:
            raise SbError("at least one curve is needed")
        self.curves, self._own, self.handles = [], [], None
        try:
            for c in curves:
                if isinstance(c, int):
                    c = getCurveFromQ(self.header["q"], c)
                    self._own.append(c)
                self.curves.append(c)
            n = len(self.curves)
            self._ctxs = (ctypes.c_void_p * n)(*[c.handle.value for c in self.curves])
            handles = (ctypes.c_uint64 * n)()
            buf = np.frombuffer(zkey, np.uint8)
            c0 = self.curves[0]
            c0.check(getattr(c0.lib, f"sb_{self.PROTO}_{self.LOAD}")(self._ctxs, n, _ptr(buf), buf.size, handles))
            self.handles = handles
        except BaseException:
            self.release()
            raise
        for k in self.FIELDS:
            setattr(self, k, self.header[k])

    @property
    def curve(self):
        return self.curves[0]

    def release(self):
        if self.handles is not None:
            for c, h in zip(self.curves, self.handles):
                getattr(c.lib, f"sb_{self.PROTO}_release")(c.handle, h)
            self.handles = None
        for c in self._own:
            c.terminate()
        self._own = []


class ReplicatedProvingKey(KeyOnContexts):
    """A Groth16 zkey loaded whole on several contexts (sb_groth16_load_replicas), so that a batch of proofs is split
    over them (sb_groth16_prove_batch_multi): context i proves a contiguous share of the batch."""

    def prove_batch_raw(self, witnesses, rs) -> list:
        """As ProvingKey.prove_batch_raw, over every context: the proofs are byte-identical to it."""
        w, r, s, count = _batch_inputs(self.nVars, witnesses, rs)
        if count == 0:
            return []
        c = self.curves[0]
        pb = 8 * c.n8q
        out = np.empty(count * pb, np.uint8)
        c.check(c.lib.sb_groth16_prove_batch_multi(self._ctxs, self.handles, len(self.curves), _ptr(w), w.size // 32 // count, count,
                                                   _ptr(r), _ptr(s), _ptr(out)))
        return [out[i * pb:(i + 1) * pb].tobytes() for i in range(count)]


class ProvingKey:
    """A Groth16 zkey registered on one device (bases + CSR coefficients resident in HBM)."""

    def __init__(self, zkey: bytes, curve: Curve | None = None, device: int = 0, shard: int = 0, n_shards: int = 1):
        zkey = bytes(zkey)
        self.header = read_zkey_header_groth16(zkey)
        self.curve = curve or getCurveFromQ(self.header["q"], device)
        self._own_curve = curve is None
        h = ctypes.c_uint64()
        buf = np.frombuffer(zkey, np.uint8)
        if n_shards > 1:   # multi-GPU: keep only this rank's point range of every base set (and its window tables)
            self.curve.check(self.curve.lib.sb_groth16_load_sharded(self.curve.handle, _ptr(buf), buf.size, shard, n_shards, ctypes.byref(h)))
        else:
            self.curve.check(self.curve.lib.sb_groth16_load(self.curve.handle, _ptr(buf), buf.size, ctypes.byref(h)))
        self.handle = h.value
        self.nVars, self.nPublic, self.domainSize = self.header["nVars"], self.header["nPublic"], self.header["domainSize"]

    @classmethod
    def from_file(cls, path: str, curve: Curve):
        """Loads the key from disk (sb_groth16_load_file: mapped read-only, streamed to HBM section by section)."""
        self = cls.__new__(cls)
        self.curve, self._own_curve = curve, False
        h = ctypes.c_uint64()
        curve.check(curve.lib.sb_groth16_load_file(curve.handle, path.encode(), ctypes.byref(h)))   # validates the container
        self.handle = h.value
        nv, npub, ds = ctypes.c_uint32(), ctypes.c_uint32(), ctypes.c_uint32()
        curve.check(curve.lib.sb_groth16_info(curve.handle, self.handle, ctypes.byref(nv), ctypes.byref(npub), ctypes.byref(ds)))
        self.nVars, self.nPublic, self.domainSize = nv.value, npub.value, ds.value
        self.header = {"n8q": curve.n8q, "q": curve.q, "n8r": 32, "r": curve.r, "nVars": nv.value, "nPublic": npub.value, "domainSize": ds.value}
        return self

    def prove_raw(self, witness, r: bytes, s: bytes) -> bytes:
        """witness = section-2 payload (nVars * 32 bytes, plain LE) -> affine proof bytes."""
        w = _arr(witness)
        out = np.empty(8 * self.curve.n8q, np.uint8)
        self.curve.check(self.curve.lib.sb_groth16_prove(self.curve.handle, self.handle, _ptr(w), w.size // 32, bytes(r), bytes(s), _ptr(out)))
        return out.tobytes()

    def prove_batch_raw(self, witnesses, rs) -> list:
        """witnesses = a sequence of section-2 payloads (nVars * 32 bytes each) or one buffer of them back to back;
        rs = [(r, s), ...] one pair per witness -> affine proof bytes per witness, each equal to prove_raw's."""
        w, r, s, count = _batch_inputs(self.nVars, witnesses, rs)
        if count == 0:
            return []
        pb = 8 * self.curve.n8q
        out = np.empty(count * pb, np.uint8)
        self.curve.check(self.curve.lib.sb_groth16_prove_batch(self.curve.handle, self.handle, _ptr(w), w.size // 32 // count, count,
                                                               _ptr(r), _ptr(s), _ptr(out)))
        return [out[i * pb:(i + 1) * pb].tobytes() for i in range(count)]

    def prove_shard(self, witness, shard: int, n_shards: int) -> np.ndarray:
        w = _arr(witness)
        out = np.empty(self.curve.lib.sb_groth16_partials_bytes(self.curve.handle), np.uint8)
        self.curve.check(self.curve.lib.sb_groth16_prove_shard(self.curve.handle, self.handle, _ptr(w), w.size // 32, shard, n_shards, _ptr(out)))
        return out

    def finish(self, partials_all, n_shards: int, r: bytes, s: bytes) -> bytes:
        p = _arr(partials_all)
        out = np.empty(8 * self.curve.n8q, np.uint8)
        self.curve.check(self.curve.lib.sb_groth16_finish(self.curve.handle, self.handle, _ptr(p), n_shards, bytes(r), bytes(s), _ptr(out)))
        return out.tobytes()

    def prove_dist(self, witness, r: bytes, s: bytes, want_proof: bool = True):
        """One proof across the ranks of the curve's communicator (Curve.comm_init): a collective call.  The key must be
        this rank's shard (ProvingKey(..., shard=rank, n_shards=world)).  witness=None reuses the resident witness."""
        w = None if witness is None else _arr(witness)
        out = np.empty(8 * self.curve.n8q, np.uint8) if want_proof else None
        self.curve.check(self.curve.lib.sb_groth16_prove_dist(self.curve.handle, self.handle, None if w is None else _ptr(w),
                                                               self.nVars if w is None else w.size // 32, bytes(r), bytes(s),
                                                               None if out is None else _ptr(out)))
        return None if out is None else out.tobytes()

    def release(self):
        if self.handle:
            self.curve.lib.sb_groth16_release(self.curve.handle, self.handle)
            self.handle = 0
        if self._own_curve:
            self.curve.terminate()


def prove(zkey, wtns: bytes, r: bytes | None = None, s: bytes | None = None, logger=None, options=None):
    """groth16Prove(zkeyFileName, witnessFileName) -> (proof, publicSignals); zkey may be bytes or a ProvingKey."""
    pk = zkey if isinstance(zkey, ProvingKey) else ProvingKey(zkey)
    try:
        wh, W = read_wtns_header(bytes(wtns))
        if wh["q"] != pk.header["r"]:
            raise SbError("Curve of the witness does not match the curve of the proving key")
        if wh["nWitness"] != pk.nVars:
            raise SbError(f"Invalid witness length. Circuit: {pk.nVars}, witness: {wh['nWitness']}")
        r = r or random_fr(pk.curve)
        s = s or random_fr(pk.curve)
        aff = pk.prove_raw(np.frombuffer(W, np.uint8), r, s)
        pub = [str(int.from_bytes(W[i * 32:(i + 1) * 32], "little")) for i in range(1, pk.nPublic + 1)]
        return proof_to_object(pk.curve, aff), pub
    finally:
        if not isinstance(zkey, ProvingKey):
            pk.release()


def prove_batch(zkey, wtns_list, rs=None):
    """groth16Prove over many witnesses of one circuit in one device call: [(proof, publicSignals), ...] in the order of
    wtns_list.  zkey may be bytes or a ProvingKey; every .wtns container is checked as prove checks it (curve, nWitness);
    rs = [(r, s), ...] (32-byte Montgomery Fr), drawn like Fr.random() when not given."""
    pk = zkey if isinstance(zkey, ProvingKey) else ProvingKey(zkey)
    try:
        ws = []
        for wtns in wtns_list:
            wh, W = read_wtns_header(bytes(wtns))
            if wh["q"] != pk.header["r"]:
                raise SbError("Curve of the witness does not match the curve of the proving key")
            if wh["nWitness"] != pk.nVars:
                raise SbError(f"Invalid witness length. Circuit: {pk.nVars}, witness: {wh['nWitness']}")
            ws.append(W)
        if rs is None:
            rs = [(random_fr(pk.curve), random_fr(pk.curve)) for _ in ws]
        if len(rs) != len(ws):
            raise SbError("one (r, s) pair per witness")
        affs = pk.prove_batch_raw([np.frombuffer(W, np.uint8) for W in ws], rs)
        out = []
        for W, aff in zip(ws, affs):
            pub = [str(int.from_bytes(W[i * 32:(i + 1) * 32], "little")) for i in range(1, pk.nPublic + 1)]
            out.append((proof_to_object(pk.curve, aff), pub))
        return out
    finally:
        if not isinstance(zkey, ProvingKey):
            pk.release()


# ------------------------------------------------------------------ verification (src/groth16_verify.js:26-87)
VERIFY_MESSAGES = {1: "Invalid proof", 2: "Public inputs are not valid.", 3: "Proof commitments are not valid."}


def _curve_of(name: str):
    """(n8q, q, r, snarkjs name) of a curve named as snarkjs names it."""
    from .curve import _Q, _R
    key = {"BN128": "bn128", "BN254": "bn128", "ALTBN128": "bn128", "BLS12381": "bls12381"}.get(
        str(name).upper().replace("-", "").replace("_", ""), name)
    if key not in _R:
        raise SbError(f"Curve not supported: {name}")
    n8q = 32 if key == "bn128" else 48
    return n8q, _Q[(n8q,)], _R[key], key


def verification_key(zkey) -> dict:
    """zkey export verificationkey for a Groth16 key (src/zkey_export_verificationkey.js): the fields groth16Verify reads, as
    decimal strings (G.toObject + stringifyBigInts).  vk_alphabeta_12 is not produced."""
    data = bytes(zkey)
    z = read_zkey_header_groth16(data)
    n8, q = z["n8q"], z["q"]
    name = "bn128" if n8 == 32 else "bls12381"
    f = lambda b: str(_from_mont(b, q, n8))

    def g1(p):
        return ["0", "1", "0"] if p == bytes(2 * n8) else [f(p[:n8]), f(p[n8:]), "1"]

    def g2(p):
        if p == bytes(4 * n8):
            return [["0", "0"], ["1", "0"], ["0", "0"]]
        return [[f(p[:n8]), f(p[n8:2 * n8])], [f(p[2 * n8:3 * n8]), f(p[3 * n8:])], ["1", "0"]]

    pos, _ = z["sections"][3]
    ic = [g1(data[pos + i * 2 * n8:pos + (i + 1) * 2 * n8]) for i in range(z["nPublic"] + 1)]
    return {"protocol": "groth16", "curve": name, "nPublic": z["nPublic"], "vk_alpha_1": g1(z["vk_alpha_1"]),
            "vk_beta_2": g2(z["vk_beta_2"]), "vk_gamma_2": g2(z["vk_gamma_2"]), "vk_delta_2": g2(z["vk_delta_2"]), "IC": ic}


def _f2_mul(a, b, q):
    return ((a[0] * b[0] - a[1] * b[1]) % q, (a[0] * b[1] + a[1] * b[0]) % q)


def _f2_inv(a, q):
    n = pow((a[0] * a[0] + a[1] * a[1]) % q, -1, q)
    return (a[0] * n % q, -a[1] * n % q)


def point_bytes(obj, group: int, n8q: int, q: int) -> bytes:
    """G.fromObject (build/snarkjs.js:13486-13495 over F.fromObject :13042-13046) then affine Montgomery bytes: the object is
    Jacobian (x, y, z), every coordinate taken mod q; z = 0 is infinity (all-zero bytes), otherwise (x/z^2, y/z^3)."""
    R = 1 << (8 * n8q)
    enc = lambda v: (v * R % q).to_bytes(n8q, "little")
    if group == 1:
        x, y = int(obj[0]) % q, int(obj[1]) % q
        z = int(obj[2]) % q if len(obj) > 2 else 1
        if z == 0:
            return bytes(2 * n8q)
        zi = pow(z, -1, q)
        z2 = zi * zi % q
        return enc(x * z2 % q) + enc(y * z2 * zi % q)
    x = (int(obj[0][0]) % q, int(obj[0][1]) % q)
    y = (int(obj[1][0]) % q, int(obj[1][1]) % q)
    z = (int(obj[2][0]) % q, int(obj[2][1]) % q) if len(obj) > 2 else (1, 0)
    if z == (0, 0):
        return bytes(4 * n8q)
    zi = _f2_inv(z, q)
    z2 = _f2_mul(zi, zi, q)
    ax, ay = _f2_mul(x, z2, q), _f2_mul(y, _f2_mul(z2, zi, q), q)
    return enc(ax[0]) + enc(ax[1]) + enc(ay[0]) + enc(ay[1])


def vk_bytes(vk_verifier: dict) -> bytes:
    """The verification key as sb_groth16_verify_batch takes it: alpha1 || beta2 || gamma2 || delta2 || IC[0..nPublic]."""
    n8, q, _r, _name = _curve_of(vk_verifier["curve"])
    ic = vk_verifier["IC"]
    if len(ic) != int(vk_verifier["nPublic"]) + 1:
        raise SbError(f"IC has {len(ic)} points, nPublic is {vk_verifier['nPublic']}")
    return (point_bytes(vk_verifier["vk_alpha_1"], 1, n8, q) + b"".join(point_bytes(vk_verifier[k], 2, n8, q)
            for k in ("vk_beta_2", "vk_gamma_2", "vk_delta_2")) + b"".join(point_bytes(p, 1, n8, q) for p in ic))


def proof_bytes(proof: dict, n8q: int, q: int) -> bytes:
    return point_bytes(proof["pi_a"], 1, n8q, q) + point_bytes(proof["pi_b"], 2, n8q, q) + point_bytes(proof["pi_c"], 1, n8q, q)


def publics_bytes(public_signals, r: int):
    """Plain LE 32-byte public signals, or None when one cannot be written in 32 bytes (then it is >= r: status 2)."""
    vals = [int(s) for s in public_signals]
    if any(v < 0 or v >= r for v in vals):
        return None
    return b"".join(v.to_bytes(32, "little") for v in vals)


def verify_status(vk_verifier: dict, items, curve: Curve | None = None) -> list:
    """sb_groth16_verify_batch over [(publicSignals, proof), ...]: one status per item (0 verifies, else the key of
    VERIFY_MESSAGES).  A proof with a signal count other than nPublic gets 1, as the reference's pairing would give it."""
    n8, q, r, name = _curve_of(vk_verifier["curve"])
    n_public = int(vk_verifier["nPublic"])
    vk = np.frombuffer(vk_bytes(vk_verifier), np.uint8)
    status = [None] * len(items)
    pubs, prfs, slots = [], [], []
    for k, (signals, proof) in enumerate(items):
        pb = publics_bytes(signals, r)
        if pb is None:
            status[k] = 2
        elif len(signals) != n_public:
            status[k] = 1
        else:
            pubs.append(pb)
            prfs.append(proof_bytes(proof, n8, q))
            slots.append(k)
    own = curve is None
    cv = curve or Curve(name)
    try:
        count = len(slots)
        out = np.zeros(max(count, 1), np.int32)
        pub = np.frombuffer(b"".join(pubs) or b"\0", np.uint8)
        prf = np.frombuffer(b"".join(prfs) or b"\0", np.uint8)
        cv.check(cv.lib.sb_groth16_verify_batch(cv.handle, _ptr(vk), vk.size, n_public, _ptr(pub), _ptr(prf), count,
                                                out.ctypes.data_as(ctypes.c_void_p)))
    finally:
        if own:
            cv.terminate()
    for j, k in enumerate(slots):
        status[k] = int(out[j])
    return status


def verify_batch(vk_verifier: dict, items, logger=None, curve: Curve | None = None) -> list:
    """groth16Verify over many (publicSignals, proof) pairs against one verification key, in one device call -> [bool]."""
    st = verify_status(vk_verifier, items, curve)
    if logger:
        for s in st:
            if s:
                logger.error(VERIFY_MESSAGES[s])
    return [s == 0 for s in st]


def verify(vk_verifier: dict, publicSignals, proof: dict, logger=None, curve: Curve | None = None) -> bool:
    """groth16Verify(vk_verifier, publicSignals, proof, logger) (src/groth16_verify.js:26-87): True, or False with the
    reference's log message."""
    s = verify_status(vk_verifier, [(publicSignals, proof)], curve)[0]
    if logger:
        if s:
            logger.error(VERIFY_MESSAGES[s])
        else:
            logger.info("OK!")
    return s == 0
