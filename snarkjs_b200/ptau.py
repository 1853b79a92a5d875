"""powersoftau prepare phase2 on the GPU — mirror of src/powersoftau_preparephase2.js:23-100.

The Lagrange-basis sections 12-15 of a prepared ptau are the group iFFTs (G.lagrangeEvaluations) of every power-of-two
prefix of sections 2-5; each of them runs on the GPU through the curve object (curve.py Group.lagrangeEvaluations ->
sb_group_fft)."""
from __future__ import annotations

import struct

from .curve import SbError, getCurveFromQ
from .groth16 import read_binfile


def read_ptau_header(data: bytes, secs):
    """src/powersoftau_utils.js:52-71 -> (n8, q, power, ceremonyPower)."""
    if 1 not in secs:
        raise SbError("ptau: File has no  header")
    p, ln = secs[1]
    n8 = struct.unpack_from("<I", data, p)[0]
    q = int.from_bytes(data[p + 4:p + 4 + n8], "little")
    power, ceremony_power = struct.unpack_from("<II", data, p + 4 + n8)
    if 12 + n8 != ln:
        raise SbError("Invalid PTau header size")
    return n8, q, power, ceremony_power


def _ptau_header(n8: int, q: int, power: int) -> bytes:
    """writePTauHeader(fd, curve, power) (src/powersoftau_utils.js:26-50): ceremonyPower = power."""
    return struct.pack("<I", n8) + q.to_bytes(n8, "little") + struct.pack("<II", power, power)


def prepare_phase2(ptau: bytes, curve=None) -> bytes:
    """`snarkjs powersoftau prepare phase2`: returns the prepared ptau (version 1, sections 1-7 then 12-15).
    `curve` defaults to the GPU curve of the file's q; any object with q, n8q and G1/G2.lagrangeEvaluations will do."""
    data = bytes(ptau)
    secs = read_binfile(data, "ptau", 1)
    n8, q, power, _ceremony = read_ptau_header(data, secs)
    if curve is None:
        curve = getCurveFromQ(q)
    if curve.n8q != n8:
        raise SbError("ptau: Invalid size")

    def sec(sid) -> bytes:
        if sid not in secs:
            raise SbError(f"Missing section {sid}")
        p, ln = secs[sid]
        return data[p:p + ln]

    out = [(1, _ptau_header(n8, q, power))] + [(sid, sec(sid)) for sid in range(2, 8)]
    for old, new, grp in ((2, 12, 1), (3, 13, 2), (4, 14, 1), (5, 15, 1)):
        G = curve.G1 if grp == 1 else curve.G2
        sG = 2 * n8 * grp
        src = sec(old)
        blocks = []
        for p in range(power + 2 if old == 2 else power + 1):
            n = 1 << p
            if p == power + 1:       # one more block of section 12: 2^p - 1 points and one point at infinity (:78-80)
                pts = src[:(n - 1) * sG] + bytes(sG)
            else:
                pts = src[:n * sG]
            if len(pts) != n * sG:
                raise SbError(f"ptau: section {old} is shorter than 2^{p} points")
            blocks.append(bytes(G.lagrangeEvaluations(pts, "affine", "affine")))
        out.append((new, b"".join(blocks)))
    body = bytearray(b"ptau" + struct.pack("<II", 1, len(out)))
    for sid, payload in out:
        body += struct.pack("<IQ", sid, len(payload)) + payload
    return bytes(body)
