"""CPU reference of the group FFT and group batchApplyKey (test infrastructure): ctypes over tests/host/group_fft_oracle.cpp,
which builds on the CPU oracle's field and point arithmetic.  The library is compiled on first use into the system's
temporary directory (keyed by the hash of its sources), never into the repository."""
import ctypes
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from oracle import oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "host", "group_fft_oracle.cpp")
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        h = hashlib.sha256()
        for p in (SRC, os.path.join(ROOT, "oracle", "snark_oracle.cpp")):
            h.update(open(p, "rb").read())
        so = os.path.join(tempfile.gettempdir(), f"snarkb200_gfft_oracle_{os.getuid()}_{h.hexdigest()[:16]}.so")
        if not os.path.exists(so):
            gomp = "/usr/lib/gcc/x86_64-linux-gnu/13/"          # as oracle/Makefile: some g++ installs miss libgomp.spec
            tmp = f"{so}.{os.getpid()}.tmp"
            subprocess.check_call([os.environ.get("CXX", "g++"), "-O3", "-march=x86-64-v3", "-fopenmp"] +
                                  (["-B" + gomp] if os.path.isdir(gomp) else []) +
                                  ["-fPIC", "-std=c++17", "-shared", "-o", tmp, SRC])
            os.replace(tmp, so)
        _LIB = ctypes.CDLL(so)
    return _LIB


def group_fft(curve: int, group: int, data, inverse: bool = False, in_jacobian: bool = False,
              out_jacobian: bool = False) -> np.ndarray:
    """G.fft / G.ifft (build/snarkjs.js:15101-15107 -> _fft 14675-14918): natural order in and out; Jacobian output is
    not normalised."""
    n8 = O.CURVES[curve].n8q * group
    a = O._in(data)
    sin = (3 if in_jacobian else 2) * n8
    n = a.size // sin
    if n == 0 or n & (n - 1) or n * sin != a.size:
        raise ValueError("fft must be multiple of 2")     # build/snarkjs.js:14745-14747
    out = O._buf(n * (3 if out_jacobian else 2) * n8)
    O._chk(lib().gfo_group_fft(curve, group, O._p(a), int(in_jacobian), ctypes.c_uint64(n), int(inverse), int(out_jacobian),
                               O._p(out)), "group_fft")
    return out


def group_batch_apply_key(curve: int, group: int, data, first: bytes, inc: bytes, in_jacobian: bool = False,
                          out_jacobian: bool = False) -> np.ndarray:
    """G.batchApplyKey (build/snarkjs.js:14268-14385): out[i] = in[i] * first * inc^i (first, inc Montgomery Fr)."""
    n8 = O.CURVES[curve].n8q * group
    a = O._in(data)
    n = a.size // ((3 if in_jacobian else 2) * n8)
    out = O._buf(n * (3 if out_jacobian else 2) * n8)
    O._chk(lib().gfo_group_batch_apply_key(curve, group, O._p(a), int(in_jacobian), ctypes.c_uint64(n), first, inc,
                                           int(out_jacobian), O._p(out)), "group_batch_apply_key")
    return out
