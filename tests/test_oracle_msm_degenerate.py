"""The oracle's Pippenger (O.multiexp_affine) against its naive double-and-add sum (O.multiexp_naive) on the degenerate
bases and boundary scalars that tests/test_gpu_msm_sweep.py compares the CUDA MSM with, so that the reference is
trustworthy on exactly those inputs.  CPU only."""
from concurrent.futures import ThreadPoolExecutor

import pytest

from oracle import oracle as O
from tests import msm_sets as S

BN, BLS = O.BN254, O.BLS12_381
GROUPS = [(BN, 1), (BN, 2), (BLS, 1), (BLS, 2)]
GROUP_IDS = ["bn254_g1", "bn254_g2", "bls12381_g1", "bls12381_g2"]
N = 257
SHAPE_C = (3, 8, 11, 12, 14, 16, 20, 22)
WIDTHS = (1, 4, 5, 13, 31, 32, 33, 40, 64)
WIDTH_C = (3, 8, 11, 12, 16, 20, 22)
TOP_HALF = ((4, 3), (4, 11), (13, 3), (13, 5), (13, 7), (13, 15), (13, 21))


def _check(cases):
    """cases: (label, cid, grp, bases, scalars).  The naive sums run in threads (the oracle's C calls release the GIL)."""
    def one(case):
        label, cid, grp, bases, sc = case
        fast = O.g_to_affine(cid, grp, O.multiexp_affine(cid, grp, bases, sc))
        slow = O.g_to_affine(cid, grp, O.multiexp_naive(cid, grp, bases, sc))
        return label, fast == slow
    with ThreadPoolExecutor(8) as ex:
        bad = [label for label, ok in ex.map(one, cases) if not ok]
    assert not bad, bad


@pytest.mark.parametrize("bname", S.BASE_SETS)
@pytest.mark.parametrize("cid,grp", GROUPS, ids=GROUP_IDS)
def test_pippenger_equals_naive_on_degenerate_bases(cid, grp, bname):
    bases = S.base_set(cid, grp, bname, N)
    cases = [((k,), cid, grp, bases, S.scalar_set(cid, k, N)) for k in ("uniform", "uniform256", "equal", "zero")]
    cases += [(("boundary", c), cid, grp, bases, S.scalar_set(cid, "boundary", N, 32, c)) for c in SHAPE_C]
    _check(cases)


@pytest.mark.parametrize("cid,grp", GROUPS, ids=GROUP_IDS)
def test_pippenger_equals_naive_on_boundary_scalars_by_width(cid, grp):
    bases = S.random_bases(cid, grp, N)
    pairs = sorted({(sb, c) for sb in WIDTHS for c in WIDTH_C} | set(TOP_HALF))
    _check([((sb, c), cid, grp, bases, S.scalar_set(cid, "boundary", N, sb, c)) for sb, c in pairs])


def test_boundary_values_hit_the_recoding_edges():
    """The boundary set reaches what it is meant to: a top digit of half through the carry where c divides 8*sbytes + 1,
    and digit 1 in every window for the entry-count scalar."""
    def digits(v, c, sbytes):
        out, carry = [], 0
        for w in range(S.windows(c, sbytes)):
            raw = ((v >> (w * c)) & ((1 << c) - 1)) + carry
            carry = int(raw > (1 << (c - 1)))
            out.append(raw - (carry << c))
        assert carry == 0
        return out
    r = O.CURVES[BN].r
    for sbytes, c in TOP_HALF:
        assert any(digits(v, c, sbytes)[-1] == 1 << (c - 1) for v in S.boundary_values(r, sbytes, c)), (sbytes, c)
    for sbytes in WIDTHS:
        for c in range(3, 23):
            d = digits(S.ones_value(c, sbytes), c, sbytes)
            assert all(d) and S.ones_value(c, sbytes) < 1 << (8 * sbytes), (sbytes, c)
