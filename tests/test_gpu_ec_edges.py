"""GPU: the XYZZ point formulas of csrc/ec.cuh (add_affine, add_i, add, dbl, dbl_affine) as compiled for sm_90a, on all four
groups, through sb_field_eval over every record of tests/ec_edges.py: bit for bit the bytes of the formulas restated on
Python integers, and for on-curve records the textbook group law.  add_i and add meet the same expected bytes, so they are
pinned equal on the device.  The CPU twin of this test is tests/test_host_ec_edges.py."""
import numpy as np
import pytest

from tests import ec_edges as EC

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    import snarkjs_b200
    c = snarkjs_b200.getCurveFromName("bn128")      # the group does not depend on the context's curve
    yield c
    c.terminate()


def _ptr(a):
    from snarkjs_b200.curve import _ptr as p
    return p(a)


@pytest.mark.parametrize("group,op", EC.all_sets(),
                         ids=[f"{EC.GROUPS[g].replace(' ', '_')}-{EC.OP_NAMES[o]}" for g, o in EC.all_sets()])
def test_point_formula_edges(ctx, group, op):
    recs = EC.records(group, op)
    inp, want = EC.pack(group, recs)
    a = np.frombuffer(inp, np.uint8)
    out = np.zeros(len(want), np.uint8)
    ctx.check(ctx.lib.sb_field_eval(ctx.handle, group, op, _ptr(a), len(recs), _ptr(out)))
    bad = EC.mismatches(group, op, out.tobytes())
    if bad:
        pytest.fail(f"{len(bad)}+ failing records, first ones:\n" + "\n".join(bad))
