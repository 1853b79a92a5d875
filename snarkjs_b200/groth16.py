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
