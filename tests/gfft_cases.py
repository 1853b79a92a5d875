"""Shared inputs of the group FFT tests: the reference's prepared-ptau fixture data and small point sets with infinity,
repeated points and P / -P pairs (test_oracle_group_fft.py on the CPU, test_gpu_group_fft.py on the GPU)."""
import hashlib
import os
import struct

import numpy as np

from oracle import oracle as O

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
CASES = [(O.BN254, 1), (O.BN254, 2), (O.BLS12_381, 1), (O.BLS12_381, 2)]
# power-k blocks of the fixture's sections 12..15 with a digest in ptau_prepare_goldens.npz: (section, input section, group, max k)
SECTIONS = [(12, 2, 1, 12), (13, 3, 2, 10), (14, 4, 1, 10), (15, 5, 1, 10)]
TRUNC_POWER = 10


def goldens():
    p = np.load(os.path.join(GOLDEN, "ptau_goldens.npz"))
    q = np.load(os.path.join(GOLDEN, "ptau_prepare_goldens.npz"))
    return {"tauG1": p["tauG1"], "tauG2": p["tauG2"], **{k: q[k] for k in q.files}}


def section_points(g, sid):
    """The fixture's prefix of ptau section 2..5 (affine Montgomery bytes) kept in the goldens."""
    return {2: g["tauG1"], 3: g["tauG2"], 4: g["alphaTauG1"], 5: g["betaTauG1"]}[sid]


def digest(b) -> bytes:
    return hashlib.sha256(bytes(b)).digest()


def block_digests(g, sid):
    return g[f"s{sid}_sha256"].reshape(-1, 32)


def truncated_ptau(g, power=TRUNC_POWER) -> bytes:
    """A power-`power` ptau with sections 1-7 cut from the fixture's prefixes (the header's power fields rewritten)."""
    hdr = bytearray(g["header"].tobytes())
    n8 = struct.unpack_from("<I", hdr, 0)[0]
    struct.pack_into("<II", hdr, 4 + n8, power, power)
    n = 1 << power
    secs = [(1, bytes(hdr)), (2, g["tauG1"][:(2 * n - 1) * 64].tobytes()), (3, g["tauG2"][:n * 128].tobytes()),
            (4, g["alphaTauG1"][:n * 64].tobytes()), (5, g["betaTauG1"][:n * 64].tobytes()),
            (6, g["section6"].tobytes()), (7, g["section7"].tobytes())]
    return O.write_binfile("ptau", 1, secs)


def sections(ptau: bytes):
    data, secs = O.read_binfile(ptau, "ptau", 1)
    return {sid: bytes(O.section(data, secs, sid)) for sid in secs}


def fr_plain(cid, x: int) -> bytes:
    return (x % O.CURVES[cid].r).to_bytes(32, "little")


def fr_mont(cid, x: int) -> bytes:
    return O.CURVES[cid].fr_to_mont(x)


def generator_jac(cid, grp) -> bytes:
    ci = O.CURVES[cid]
    return O.g_from_affine(cid, grp, ci.g1_affine_bytes(ci.g1) if grp == 1 else ci.g2_affine_bytes(ci.g2))


def degenerate_scalars(cid, n, seed=3):
    """Discrete logs k_i of the points k_i G of a test input: infinity (0), a repeated point, a P / -P pair, the rest
    pseudo-random."""
    r = O.CURVES[cid].r
    rng = np.random.default_rng(seed + n)
    ks = [int.from_bytes(rng.bytes(32), "little") % r for _ in range(n)]
    if n >= 2:
        ks[1] = 0
    if n >= 4:
        ks[2] = ks[0]
        ks[3] = r - ks[0]
    if n >= 8:
        ks[5] = ks[4]
        ks[6] = r - ks[4]
        ks[7] = 0
    return ks


def points_jac(cid, grp, ks) -> np.ndarray:
    """k_i G as un-normalised Jacobian bytes (Z != 1; infinity (0,1,0))."""
    g = generator_jac(cid, grp)
    return np.frombuffer(b"".join(O.g_times(cid, grp, g, fr_plain(cid, k)) for k in ks), np.uint8)


def normalise_jac(cid, grp, jac) -> np.ndarray:
    """Jacobian bytes -> the normalised form of the GPU output: (x, y, 1), infinity (0, 1, 0)."""
    ci = O.CURVES[cid]
    n8 = ci.n8q * grp
    aff = O.batch_to_affine(cid, grp, jac).reshape(-1, 2 * n8)
    one = ci.fq_to_mont(1) + bytes(n8 - ci.n8q)
    out = []
    for a in aff:
        a = a.tobytes()
        out.append(bytes(n8) + one + bytes(n8) if a == bytes(2 * n8) else a + one)
    return np.frombuffer(b"".join(out), np.uint8)
