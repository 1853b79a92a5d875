"""oracle/synth_setup.py — synthetic inputs for `zkey new` with KNOWN toxic waste.  TEST INFRASTRUCTURE ONLY.

The reference ships one prepared powers-of-tau file, on BN254.  To exercise the Groth16 path on BLS12-381 with keys whose
proofs *verify* (not only compare), this module writes, for any curve:
  * chain_r1cs(...)        an .r1cs container (r1csfile layout, SURVEY Appendix A) for the chain x_{i+1} = x_i^2 + b with one
                           public output, plus its witness — the shape of test/groth16/circuit.circom;
  * prepared_ptau(...)     the sections of a prepared .ptau that src/zkey_new.js:101-151,182-200 reads (4 alphaTauG1,
                           5 betaTauG1, 6 betaG2, and the Lagrange-basis sections 12-15 for one domain size and its double),
                           computed from chosen tau, alpha, beta instead of a ceremony;
  * plonk_ptau(...)        the sections src/plonk_setup.js and src/fflonk_setup.js read (2 tau^i G1, 3 tau G2, 12 the
                           Lagrange basis of one domain size), from a chosen tau or from pseudo-random points.
oracle.zkey_new(r1cs_bytes, ptau_bytes), oracle.plonk.plonk_setup and oracle.fflonk.fflonk_setup then build the zkey exactly
as for the reference's files."""
from __future__ import annotations

import struct
from typing import List, Tuple

from . import oracle as orc


def chain_r1cs(curve: int, n_constraints: int, seed: int = 5) -> Tuple[bytes, List[int]]:
    """Wires: 0 = one, 1 = x_m (public output), 2 = x_0, 3.. = x_1..x_{m-1}; constraint i: x_i * x_i = x_{i+1} - b."""
    ci = orc.CURVES[curve]
    r = ci.r
    m = n_constraints
    b = (seed * 7919 + 3) % r
    x = [(seed * 104729 + 11) % r]
    for _ in range(m):
        x.append((x[-1] * x[-1] + b) % r)
    wire = [2 + i for i in range(m)] + [1]
    wit = [1, x[m]] + x[:m]
    n8 = 32

    def lc(terms):
        out = struct.pack("<I", len(terms))
        for w, v in terms:
            out += struct.pack("<I", w) + (v % r).to_bytes(n8, "little")
        return out

    body = b""
    for i in range(m):
        body += lc([(wire[i], 1)]) + lc([(wire[i], 1)]) + lc([(wire[i + 1], 1), (0, -b)])
    n_wires = len(wit)
    hdr = struct.pack("<I", n8) + r.to_bytes(n8, "little") + struct.pack("<IIII", n_wires, 1, 0, m) + struct.pack("<Q", n_wires) + struct.pack("<I", m)
    labels = b"".join(struct.pack("<Q", i) for i in range(n_wires))
    return orc.write_binfile("r1cs", 1, [(1, hdr), (2, body), (3, labels)]), wit


def _lagrange_at(ci, size: int, tau: int) -> List[int]:
    """L_j(tau) = (tau^n - 1) w^j / (n (tau - w^j)) for the size-n domain, j < n."""
    r = ci.r
    w = ci.fr_from_mont(orc.fr_root(ci.id, size.bit_length() - 1))
    zt = (pow(tau, size, r) - 1) % r
    inv_n = pow(size, -1, r)
    out, wj = [], 1
    for _ in range(size):
        out.append(zt * wj % r * inv_n % r * pow((tau - wj) % r, -1, r) % r)
        wj = wj * w % r
    return out


def _points(ci, group: int, scalars) -> bytes:
    """s * G for each s, affine Montgomery bytes."""
    g = orc.g_from_affine(ci.id, group, ci.g1_affine_bytes(ci.g1) if group == 1 else ci.g2_affine_bytes(ci.g2))
    jac = b"".join(orc.g_times(ci.id, group, g, (s % ci.r).to_bytes(32, "little")) for s in scalars)
    return bytes(orc.batch_to_affine(ci.id, group, jac))


def _ptau_header(ci, power: int) -> bytes:
    return struct.pack("<I", ci.n8q) + ci.q.to_bytes(ci.n8q, "little") + struct.pack("<II", power, power)


def prepared_ptau(curve: int, domain_size: int, tau: int, alpha: int, beta: int) -> bytes:
    """Sections 1, 4, 5, 6, 12, 13, 14, 15 of a prepared ptau, filled only where zkey_new reads: the Lagrange bases of size n
    (offset n - 1) and, for section 12, of size 2n (offset 2n - 1)."""
    ci = orc.CURVES[curve]
    r, n = ci.r, domain_size
    power = n.bit_length() - 1
    sG1, sG2 = 2 * ci.n8q, 4 * ci.n8q
    Ln, L2n = _lagrange_at(ci, n, tau), _lagrange_at(ci, 2 * n, tau)
    sec12 = bytes((n - 1) * sG1) + _points(ci, 1, Ln) + _points(ci, 1, L2n)
    sec13 = bytes((n - 1) * sG2) + _points(ci, 2, Ln)
    sec14 = bytes((n - 1) * sG1) + _points(ci, 1, [alpha * x % r for x in Ln])
    sec15 = bytes((n - 1) * sG1) + _points(ci, 1, [beta * x % r for x in Ln])
    return orc.write_binfile("ptau", 1, [(1, _ptau_header(ci, power + 1)), (4, _points(ci, 1, [alpha])), (5, _points(ci, 1, [beta])),
                                         (6, _points(ci, 2, [beta])), (12, sec12), (13, sec13), (14, sec14), (15, sec15)])


def plonk_ptau(curve: int, power: int, tau: int, n_g1: int, structured: bool = True) -> bytes:
    """Sections 1, 2, 3 and 12 of a prepared ptau, filled where oracle.plonk.plonk_setup and oracle.fflonk.fflonk_setup
    read: n_g1 powers tau^i G1 (n + 6 for PLONK, 9n + 18 for fflonk), G2 and tau G2, and the Lagrange basis of size
    n = 2^power at offset n - 1.  structured=False fills sections 2, 3 and 12 with pseudo-random valid points instead
    (seeded by tau): the keys' proofs do not verify, but their bytes are defined."""
    from .plonk import _g2_times_gen, _tau_powers
    ci = orc.CURVES[curve]
    n = 1 << power
    sG1 = 2 * ci.n8q
    if structured:
        g1 = _tau_powers(ci, tau, n_g1)
        g2 = ci.g2_affine_bytes(ci.g2) + _g2_times_gen(ci, tau)
        lag = _points(ci, 1, _lagrange_at(ci, n, tau))
    else:
        seed = tau & 0xFFFFFFFF
        g1 = bytes(orc.gen_points(ci.id, 1, seed, n_g1))
        g2 = bytes(orc.gen_points(ci.id, 2, seed + 1, 2))
        lag = bytes(orc.gen_points(ci.id, 1, seed + 2, n))
    return orc.write_binfile("ptau", 1, [(1, _ptau_header(ci, power)), (2, g1), (3, g2), (12, bytes((n - 1) * sG1) + lag)])
