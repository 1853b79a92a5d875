"""CPU: sb_field_eval's per-record dispatch (csrc/field_eval.cuh) compiled with g++, with the PTX carry chains emulated and
with the host multiply, on every edge and random record of tests/field_edges.py, against the Python big-integer results.
The GPU twin of this test is tests/test_gpu_field_edges.py."""
import os
import struct
import subprocess

import pytest

from tests import field_edges as FE

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("flags", [["-DSB_HOST_EMULATE_PTX"], []], ids=["emulated-ptx", "host-mul"])
def test_host_field_edges(tmp_path, flags):
    exe = str(tmp_path / "field_eval_host")
    subprocess.check_call(["g++", "-O2", "-std=c++17", *flags, "-o", exe, os.path.join(ROOT, "tests", "host", "field_eval_host.cpp")])
    sets = FE.all_sets()
    blob = bytearray()
    for f, op in sets:
        recs = FE.records(f, op)
        blob += struct.pack("<iiQ", f, op, len(recs)) + FE.pack(f, recs)[0]
    (tmp_path / "in.bin").write_bytes(bytes(blob))
    subprocess.check_call([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], timeout=600)
    out = (tmp_path / "out.bin").read_bytes()
    bad, pos = [], 0
    for f, op in sets:
        size = len(FE.pack(f, FE.records(f, op))[1])
        bad += FE.mismatches(f, op, out[pos:pos + size])
        pos += size
    assert pos == len(out), (pos, len(out))
    assert not bad, "\n".join(bad[:20])


def test_generator_classes_reach_their_targets():
    """Every crafted class hits what it aims at (records() raises otherwise), and the ops listed per field are exactly the
    ones sb_field_eval defines: mul2 wherever 3p < R, so not on BLS12-381 Fr."""
    for f, op in FE.all_sets():
        assert FE.records(f, op)
    assert FE.FP_OPS["mul2"] in FE.ops(0) and FE.FP_OPS["mul2"] in FE.ops(1) and FE.FP_OPS["mul2"] in FE.ops(2)
    assert FE.FP_OPS["mul2"] not in FE.ops(3)
    with pytest.raises(ValueError):
        FE.records(3, FE.FP_OPS["mul2"])
