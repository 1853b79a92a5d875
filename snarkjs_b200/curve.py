"""Host-side mirror of the ffjavascript `curve` object for the bulk methods snarkjs' provers call
(SURVEY.md §8b): same method names, argument meaning and error strings as the reference
(build/snarkjs.js:14666-14668 multiExpAffine, 15101-15107 fft/ifft, 14273-14384 batchApplyKey,
12895-12896 batchTo/FromMontgomery), executed on the GPU through the C ABI.

Buffers are bytes / bytearray / numpy uint8 arrays (the reference takes Uint8Array or BigBuffer); results are
numpy uint8 arrays (fresh buffers, like the reference's).  Methods are synchronous here — the N-API shim
(INTEGRATION.md) wraps the same C calls in napi async work to return Promises."""
from __future__ import annotations

import ctypes

import numpy as np

from . import _native as N


class SbError(Exception):
    pass


def _arr(b) -> np.ndarray:
    if isinstance(b, np.ndarray):
        return np.ascontiguousarray(b.view(np.uint8).reshape(-1))
    if hasattr(b, "buffers"):          # BigBuffer-like: flatten pages (build/snarkjs.js:12692-12778)
        return np.concatenate([_arr(x) for x in b.buffers]) if b.buffers else np.zeros(0, np.uint8)
    return np.frombuffer(bytes(b), dtype=np.uint8)


def _ptr(a: np.ndarray):
    return a.ctypes.data_as(ctypes.c_void_p)


class _Ctx:
    def __init__(self, curve_id: int, device: int):
        self.lib = N.lib()
        h = ctypes.c_void_p()
        rc = self.lib.sb_create(curve_id, device, ctypes.byref(h))
        if rc != 0:
            raise SbError({-5: "no CUDA device available (libsnarkb200 has no CPU fallback)"}.get(rc, f"sb_create failed rc={rc}"))
        self.h = h

    def check(self, rc):
        if rc != 0:
            raise SbError(self.lib.sb_last_error(self.h).decode() or f"error {rc}")

    def close(self):
        if self.h:
            self.lib.sb_destroy(self.h)
            self.h = None


class Fr:
    """curve.Fr — bulk methods only (per-element ops stay on the JS side in the reference)."""

    def __init__(self, ctx: _Ctx, n8: int = 32):
        self._c = ctx
        self.n8 = n8
        out = np.empty(32, np.uint8)
        self.s = ctx.lib.sb_fr_root(ctx.h, 0, _ptr(out))
        self.w = [self._root(i) for i in range(self.s + 1)]
        self.shift = self._root(-1)
        self.nqr = self._root(-2)

    def _root(self, what) -> bytes:
        out = np.empty(32, np.uint8)
        self._c.lib.sb_fr_root(self._c.h, what, _ptr(out))
        return out.tobytes()

    def _fft(self, buff, inverse):
        a = _arr(buff)
        n = a.size // self.n8
        if a.size % self.n8 or n == 0 or n & (n - 1):
            raise SbError("fft must be multiple of 2")          # build/snarkjs.js:14745-14747
        out = np.empty_like(a)
        self._c.check(self._c.lib.sb_ntt_fr(self._c.h, _ptr(a), n, int(inverse), _ptr(out)))
        return out

    def fft(self, buff, inType="", outType="", logger=None, txt=""):
        return self._fft(buff, False)

    def ifft(self, buff, inType="", outType="", logger=None, txt=""):
        return self._fft(buff, True)

    def batchApplyKey(self, buff, first: bytes, inc: bytes):
        a = _arr(buff)
        out = np.empty_like(a)
        self._c.check(self._c.lib.sb_fr_batch_apply_key(self._c.h, _ptr(a), a.size // self.n8, bytes(first), bytes(inc), _ptr(out)))
        return out

    def _convert(self, buff, fn):
        a = _arr(buff)
        if a.size % self.n8:
            raise SbError("Invalid buffer size")                # build/snarkjs.js:12780-12830
        out = np.empty_like(a)
        self._c.check(fn(self._c.h, _ptr(a), a.size // self.n8, _ptr(out)))
        return out

    def batchToMontgomery(self, buff):
        return self._convert(buff, self._c.lib.sb_fr_batch_to_montgomery)

    def batchFromMontgomery(self, buff):
        return self._convert(buff, self._c.lib.sb_fr_batch_from_montgomery)


class Group:
    """curve.G1 / curve.G2 — multiExpAffine plus the registered-bases extension."""

    def __init__(self, ctx: _Ctx, gid: int, n8q: int):
        self._c = ctx
        self.gid = gid
        self.n8 = n8q * gid                      # bytes per coordinate (Fq or Fq2)
        self.sAffine = 2 * self.n8
        self.sJacobian = 3 * self.n8
        one = (1 << (8 * n8q)) % (_Q[(n8q, )])
        z = bytes(self.n8)
        self.zero = z + one.to_bytes(n8q, "little") + bytes(self.n8 - n8q) + z     # (0, 1, 0)
        self._s = ctx.lib.sb_fr_root(ctx.h, 0, _ptr(np.empty(32, np.uint8)))     # Fr.s

    def multiExpAffine(self, buffBases, buffScalars, logger=None, logText=""):
        b, s = _arr(buffBases), _arr(buffScalars)
        n = b.size // self.sAffine
        if n == 0:
            return np.frombuffer(self.zero, np.uint8).copy()   # build/snarkjs.js:14561, 14627
        ss = s.size // n
        if ss * n != s.size:
            raise SbError("Scalar size does not match")         # build/snarkjs.js:14562-14565
        out = np.empty(self.sJacobian, np.uint8)
        fn = self._c.lib.sb_msm_g1_affine if self.gid == 1 else self._c.lib.sb_msm_g2_affine
        self._c.check(fn(self._c.h, _ptr(b), _ptr(s), ss, n, _ptr(out)))
        return out

    def _size(self, t: str) -> int:
        return self.sJacobian if t == "jacobian" else self.sAffine

    def _fft(self, buff, inverse, inType, outType):
        a = _arr(buff)
        sin, sout = self._size(inType or "affine"), self._size(outType or "affine")
        n = a.size // sin
        if n * sin != a.size or n == 0 or n & (n - 1):
            raise SbError("fft must be multiple of 2")          # build/snarkjs.js:14745-14747
        out = np.empty(n * sout, np.uint8)
        self._c.check(self._c.lib.sb_group_fft(self._c.h, self.gid, _ptr(a), int(sin == self.sJacobian), n, int(inverse),
                                               int(sout == self.sJacobian), _ptr(out)))
        return out

    def fft(self, buff, inType="affine", outType="affine", logger=None, loggerTxt=""):
        """G.fft (build/snarkjs.js:15101-15103); Jacobian output is normalised to Z = 1 (infinity (0,1,0))."""
        return self._fft(buff, False, inType, outType)

    def ifft(self, buff, inType="affine", outType="affine", logger=None, loggerTxt=""):
        """G.ifft (build/snarkjs.js:15105-15107)."""
        return self._fft(buff, True, inType, outType)

    def lagrangeEvaluations(self, buff, inType="affine", outType="affine", logger=None, loggerTxt=""):
        """G.lagrangeEvaluations (build/snarkjs.js:15109-15176): the ifft for log2(n) <= Fr.s; log2(n) = Fr.s + 1 (the
        reference's two-half path) is refused by the library like Fr.fft's fftExt path."""
        sin = self._size(inType or "affine")
        nbytes = buff.nbytes if isinstance(buff, np.ndarray) else _arr(buff).size
        n = nbytes // sin
        bits = max(n.bit_length() - 1, 0)
        if (1 << bits) * sin != nbytes:
            raise SbError("lagrangeEvaluations invalid Input size")
        if bits > self._s + 1:
            raise SbError("lagrangeEvaluations input too big")
        return self.ifft(buff, inType, outType, logger, loggerTxt)

    def batchApplyKey(self, buff, first: bytes, inc: bytes, inType="affine", outType="affine"):
        """G.batchApplyKey (build/snarkjs.js:14268-14385): out[i] = in[i] * first * inc^i; first / inc Montgomery Fr;
        the point count is floor(bytes / point size)."""
        a = _arr(buff)
        sin, sout = self._size(inType or "affine"), self._size(outType or "affine")
        n = a.size // sin
        out = np.empty(n * sout, np.uint8)
        self._c.check(self._c.lib.sb_group_batch_apply_key(self._c.h, self.gid, _ptr(a), int(sin == self.sJacobian), n,
                                                           bytes(first), bytes(inc), int(sout == self.sJacobian), _ptr(out)))
        return out

    def toAffine(self, jac) -> np.ndarray:
        """Our MSM results are normalised (Z = 1 or the zero point), so toAffine is a slice."""
        j = _arr(jac)
        z = j[2 * self.n8:]
        if not z.any():
            return np.zeros(self.sAffine, np.uint8)
        return j[:2 * self.n8].copy()

    def registerBases(self, buffBases) -> int:
        b = _arr(buffBases)
        h = ctypes.c_uint64()
        self._c.check(self._c.lib.sb_bases_register(self._c.h, self.gid, _ptr(b), b.size // self.sAffine, ctypes.byref(h)))
        return h.value

    def multiExpRegistered(self, handle: int, buffScalars, first: int = 0, n: int | None = None):
        s = _arr(buffScalars)
        if n is None:
            n = s.size // 32
        out = np.empty(self.sJacobian, np.uint8)
        if n == 0:
            return np.frombuffer(self.zero, np.uint8).copy()
        self._c.check(self._c.lib.sb_msm_registered(self._c.h, handle, first, _ptr(s), s.size // n, n, _ptr(out)))
        return out

    def multiExpRegisteredBatch(self, handle: int, buffScalars, count: int, first: int = 0, n: int | None = None):
        """count MSMs over the registered bases [first, first+n): buffScalars holds count rows of n scalars back to back.
        Returns a (count, sJacobian) array; row k equals multiExpRegistered on scalar row k."""
        s = _arr(buffScalars)
        out = np.empty((count, self.sJacobian), np.uint8)
        if count == 0:
            return out
        if n is None:
            n = s.size // (32 * count)
        if n == 0:
            out[:] = np.frombuffer(self.zero, np.uint8)
            return out
        sb = s.size // (n * count)
        if sb * n * count != s.size:
            raise SbError("Scalar size does not match")
        self._c.check(self._c.lib.sb_msm_registered_batch(self._c.h, handle, first, _ptr(s), sb, n, count, _ptr(out)))
        return out


_Q = {(32,): 0x30644e72e131a029b85045b68181585d97816a916871ca8d3c208c16d87cfd47,
      (48,): 0x1a0111ea397fe69a4b1ba7b6434bacd764774b84f38512bf6730d2a0f6b0f6241eabfffeb153ffffb9feffffffffaaab}
_R = {"bn128": 0x30644e72e131a029b85045b68181585d2833e84879b9709143e1f593f0000001,
      "bls12381": 0x73eda753299d7d483339d80809a1d80553bda402fffe5bfeffffffff00000001}


class Curve:
    def __init__(self, name: str, device: int = 0):
        name = {"BN128": "bn128", "BN254": "bn128", "ALTBN128": "bn128", "BLS12381": "bls12381"}.get(name.upper().replace("-", "").replace("_", ""), name)
        if name not in ("bn128", "bls12381"):
            raise SbError(f"Curve not supported: {name}")       # src/curves.js:36-53
        self.name = name
        self.id = N.SB_BN254 if name == "bn128" else N.SB_BLS12_381
        self.n8q = 32 if name == "bn128" else 48
        self.q = _Q[(self.n8q,)]
        self.r = _R[name]
        self._ctx = _Ctx(self.id, device)
        self.Fr = Fr(self._ctx)
        self.G1 = Group(self._ctx, 1, self.n8q)
        self.G2 = Group(self._ctx, 2, self.n8q)

    @property
    def handle(self):
        return self._ctx.h

    @property
    def lib(self):
        return self._ctx.lib

    def check(self, rc):
        self._ctx.check(rc)

    def launch_count(self) -> int:
        return int(self._ctx.lib.sb_launch_count(self._ctx.h))

    def last_ms(self, which=0) -> float:
        return float(self._ctx.lib.sb_last_ms(self._ctx.h, which))

    # ---- multi-GPU: one NCCL rank per context (include/snarkb200.h, sb_comm_*)
    @staticmethod
    def comm_unique_id() -> bytes:
        out = np.zeros(128, np.uint8)
        if N.lib().sb_comm_unique_id(_ptr(out)) != 0:
            raise SbError("sb_comm_unique_id failed (libnccl.so.2 not loadable?)")
        return out.tobytes()

    def comm_init(self, world: int, rank: int, unique_id: bytes):
        idb = np.frombuffer(bytes(unique_id), np.uint8)
        self.check(self.lib.sb_comm_init_rank(self.handle, world, rank, _ptr(idb)))

    def terminate(self):
        self._ctx.close()


def getCurveFromName(name: str, device: int = 0) -> Curve:
    """src/curves.js:36-53"""
    return Curve(name, device)


def getCurveFromQ(q: int, device: int = 0) -> Curve:
    """src/curves.js:23-34"""
    for k, v in _Q.items():
        if v == q:
            return Curve("bn128" if k == (32,) else "bls12381", device)
    raise SbError(f"Curve not supported: {q}")


def getCurveFromR(r: int, device: int = 0) -> Curve:
    for k, v in _R.items():
        if v == r:
            return Curve(k, device)
    raise SbError(f"Curve not supported: {r}")
