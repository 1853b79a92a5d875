"""Base and scalar sets for the MSM tests: degenerate bases (repeated, opposite and infinity points) and scalars at the
edges of the signed-digit recoding for a window size c.  tests/test_gpu_msm_sweep.py runs them through the CUDA MSM and
tests/test_oracle_msm_degenerate.py checks the CPU oracle's Pippenger on them against its naive sum.

The MSM recodes a scalar of `sbytes` bytes into W = ceil((8*sbytes + 1) / c) signed digits: a raw c-bit digit plus the
carry in is kept when it is at most half = 2^(c-1) (bucket raw - 1), otherwise it becomes raw - 2^c with a carry out."""
import functools

import numpy as np

from oracle import oracle as O

BASE_SETS = ("all_p", "p_neg_p", "inf_every_3rd", "all_inf", "q_blocks")
Q_BLOCK = 64


def point_bytes(cid, grp):
    return O.CURVES[cid].n8q * 2 * grp


def windows(c, sbytes):
    return (8 * sbytes + 1 + c - 1) // c


@functools.lru_cache(maxsize=None)
def random_bases(cid, grp, n, seed=7):
    a = O.gen_points(cid, grp, seed, n)
    a.setflags(write=False)
    return a


def negate(cid, grp, pts):
    """-P of affine Montgomery points: every y coordinate (one Fq element in G1, two in G2) becomes q - y; the all-zero
    infinity encoding stays all-zero."""
    ci = O.CURVES[cid]
    n8, sz = ci.n8q, point_bytes(cid, grp)
    a = np.array(pts, np.uint8).reshape(-1, sz).copy()
    for k in range(grp, 2 * grp):
        col = slice(k * n8, (k + 1) * n8)
        for row in a:
            v = int.from_bytes(row[col].tobytes(), "little")
            row[col] = np.frombuffer(((ci.q - v) % ci.q).to_bytes(n8, "little"), np.uint8)
    return a


@functools.lru_cache(maxsize=None)
def base_set(cid, grp, name, n, seed=7):
    """all_p: n copies of P.  p_neg_p: P, -P, P, ... (the last base is at infinity when n is odd, so equal scalars sum to
    zero).  inf_every_3rd: random points with bases 0, 3, 6, ... at infinity.  all_inf: every base at infinity.
    q_blocks: Q_k repeated Q_BLOCK times, then -Q_k repeated Q_BLOCK times, for k = 0, 1, ..."""
    sz = point_bytes(cid, grp)
    pts = random_bases(cid, grp, n, seed).reshape(n, sz)
    if name == "all_p":
        out = np.repeat(pts[:1], n, 0)
    elif name == "p_neg_p":
        out = np.repeat(pts[:1], n, 0)
        out[1::2] = negate(cid, grp, pts[:1])
        if n % 2:
            out[-1] = 0
    elif name == "inf_every_3rd":
        out = pts.copy()
        out[::3] = 0
    elif name == "all_inf":
        out = np.zeros_like(pts)
    elif name == "q_blocks":
        k = np.arange(n) // (2 * Q_BLOCK)
        qs = pts[:k[-1] + 1]
        out = qs[k].copy()
        neg = (np.arange(n) // Q_BLOCK) % 2 == 1
        out[neg] = negate(cid, grp, qs)[k[neg]]
    else:
        raise ValueError(name)
    out = out.reshape(-1)
    out.setflags(write=False)
    return out


def boundary_values(r, sbytes, c):
    """Scalar values (reduced mod 2^(8*sbytes)) where the recoding of window size c is at its edges."""
    bits = 8 * sbytes
    mask = (1 << bits) - 1
    W = windows(c, sbytes)
    half = 1 << (c - 1)

    def every(d):
        return sum(d << (w * c) for w in range(W))
    top = (W - 1) * c
    vals = [every(half),                    # raw == half in every window: positive digit, last bucket, no carry
            every(half + 1),                # negative digit with a carry in every window
            every((1 << c) - 1),            # digit -1 with a carry everywhere
            half, half + 1, (1 << c) - 1, half - 1,
            mask,                           # 2^(8*sbytes) - 1: the carry runs through every window into the top one
            r - 1, r, r + 1, (1 << 256) - 1, 1, 0,
            ones_value(c, sbytes)]
    if top < bits:                          # a single non-zero digit in the top window: smallest and largest
        vals += [1 << top, (mask >> top) << top]
    return [v & mask for v in vals]


def ones_value(c, sbytes):
    """A scalar whose W signed digits are all non-zero (digit 1 in every window), so an MSM over n such scalars consumes
    exactly n*W (digit, point) entries.  When the top window lies above the scalar's bits it is reached by the carry:
    the window below holds 2^c - 1 (digit -1, carry 1)."""
    W = windows(c, sbytes)
    if (W - 1) * c < 8 * sbytes:
        return sum(1 << (w * c) for w in range(W))
    return sum(1 << (w * c) for w in range(W - 2)) + (((1 << c) - 1) << ((W - 2) * c))


def pack(values, sbytes):
    return np.frombuffer(b"".join(int(v).to_bytes(sbytes, "little") for v in values), np.uint8).copy()


@functools.lru_cache(maxsize=None)
def scalar_set(cid, name, n, sbytes=32, c=None, seed=11):
    """uniform: below r (32-byte) or uniform bytes (other widths).  uniform256: uniform bytes (at 32 bytes most values are
    >= r).  equal: one value for every point.  zero.  boundary: boundary_values(c) repeated over the n points."""
    r = O.CURVES[cid].r
    rng = np.random.default_rng(seed + 1000 * sbytes + (c or 0))
    if name == "uniform":
        out = O.random_scalars(seed, n, r) if sbytes == 32 else rng.integers(0, 256, n * sbytes, dtype=np.uint8)
    elif name == "uniform256":
        out = rng.integers(0, 256, n * sbytes, dtype=np.uint8)
    elif name == "equal":
        one = O.random_scalars(seed + 1, 1, r)[:sbytes] if sbytes <= 32 else rng.integers(0, 256, sbytes, dtype=np.uint8)
        out = np.tile(one, n)
    elif name == "zero":
        out = np.zeros(n * sbytes, np.uint8)
    elif name == "boundary":
        vals = boundary_values(r, sbytes, c)
        out = pack([vals[i % len(vals)] for i in range(n)], sbytes)
    elif name == "ones":
        out = np.tile(pack([ones_value(c, sbytes)], sbytes), n)
    else:
        raise ValueError(name)
    out = np.ascontiguousarray(out, np.uint8).reshape(-1)
    out.setflags(write=False)
    return out
