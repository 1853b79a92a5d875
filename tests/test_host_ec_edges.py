"""CPU: the XYZZ point formulas (csrc/ec.cuh) through sb_field_eval's per-record dispatch compiled with g++, with the PTX
carry chains emulated and with the host multiply, on every record of tests/ec_edges.py: the bytes of the restated formulas
and, for on-curve records, the textbook group law.  Also pins the Python reference itself.  The GPU twin of this test is
tests/test_gpu_ec_edges.py."""
import os
import struct
import subprocess

import pytest

from tests import ec_edges as EC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("flags", [["-DSB_HOST_EMULATE_PTX"], []], ids=["emulated-ptx", "host-mul"])
def test_host_ec_edges(tmp_path, flags):
    exe = str(tmp_path / "field_eval_host")
    subprocess.check_call(["g++", "-O2", "-std=c++17", *flags, "-o", exe, os.path.join(ROOT, "tests", "host", "field_eval_host.cpp")])
    sets = EC.all_sets()
    blob = bytearray()
    for g, op in sets:
        recs = EC.records(g, op)
        blob += struct.pack("<iiQ", g, op, len(recs)) + EC.pack(g, recs)[0]
    (tmp_path / "in.bin").write_bytes(bytes(blob))
    subprocess.check_call([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], timeout=600)
    out = (tmp_path / "out.bin").read_bytes()
    bad, pos = [], 0
    for g, op in sets:
        size = len(EC.pack(g, EC.records(g, op))[1])
        bad += EC.mismatches(g, op, out[pos:pos + size])
        pos += size
    assert pos == len(out), (pos, len(out))
    assert not bad, "\n".join(bad[:20])
    for g, op in [(1, EC.EC_OPS["add"]), (3, EC.EC_OPS["dbl"]), (4, EC.FE_NOPS)]:   # no group over Fr, no op 21
        (tmp_path / "in.bin").write_bytes(struct.pack("<iiQ", g, op, 1) + bytes(8 * 96))
        r = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True)
        assert r.returncode == 2 and "not defined" in r.stderr, (g, op, r.stderr)


@pytest.mark.parametrize("group", list(EC.GROUPS), ids=[n.replace(" ", "_") for n in EC.GROUPS.values()])
def test_reference_formulas_mean_the_group_law(group):
    """(a) satisfies (b) on every on-curve record, every crafted class takes its branch (records() raises otherwise), and
    every special case of the formulas is reached on every op."""
    C = EC.curve(group)
    assert C.smul(C.r, C.g) is None and C.smul(C.r - 1, C.g) == C.neg(C.g)        # the generator has order r
    assert C.on_curve(C.phi(C.g)) and C.phi(C.g) != C.g
    wanted = {"add_affine": {"acc=inf", "dbl", "dbl y=0", "cancel", "generic", "generic R=0"},
              "dbl": {"inf", "y=0", "formula"}, "dbl_affine": {"y=0", "formula"}}
    wanted["add_i"] = wanted["add"] = wanted["add_affine"] | {"q=inf"}
    for op in EC.EC_OPS.values():
        recs = EC.records(group, op)
        assert sum(1 for r in recs if r[0] == "random") >= EC.N_RANDOM
        assert {r[4] for r in recs} == wanted[EC.OP_NAMES[op]], EC.OP_NAMES[op]
        for i, (label, args, res, on_curve, _) in enumerate(recs):
            if on_curve:
                assert all(C.on_curve(P) for P in EC.operands(C, op, args)), EC.describe(group, op, i, recs[i])
                why = EC.meaning(C, op, args, res)
                assert why is None, EC.describe(group, op, i, recs[i], why)


def test_ops_refused_outside_the_groups():
    with pytest.raises(ValueError):
        EC.records(1, EC.EC_OPS["add"])
    with pytest.raises(ValueError):
        EC.records(0, 15)
