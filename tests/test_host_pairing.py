"""CPU: the device pairing's template code (snarkjs_b200/csrc/pairing.cuh) compiled with g++ and fp.cuh's host multiply,
through the records of sb_pairing_eval (tests/host/pairing_eval_host.cpp): tower products, squarings, inverse and Frobenius
maps against Python big integers in the oracle's flat basis, the final exponentiation against f^(c (q^12 - 1)/r), and the
pairing against the oracle's.  The GPU twin is tests/test_gpu_groth16_verify.py."""
import os
import random
import struct
import subprocess

import pytest

from oracle import oracle as O
from tests import pairing_ref as PR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("pairing") / "pairing_eval_host")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-o", path, os.path.join(ROOT, "tests", "host", "pairing_eval_host.cpp")])
    return path


def run(exe, tmp_path, cid, op, recs, out_elems):
    blob = struct.pack("<iiQ", 0 if cid == O.BN254 else 1, op, len(recs)) + b"".join(PR.pack(cid, r) for r in recs)
    (tmp_path / "in.bin").write_bytes(blob)
    subprocess.check_call([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], timeout=300)
    vals = PR.unpack(cid, (tmp_path / "out.bin").read_bytes())
    return [vals[i:i + 12] for i in range(0, len(vals), 12)]


@pytest.mark.parametrize("cid", PR.CURVES, ids=["bn254", "bls12381"])
def test_host_pairing(exe, tmp_path, cid):
    rng = random.Random(17 + cid)
    fl = lambda t: PR.to_flat(cid, t)
    q = PR.Q[cid]
    a, b = PR.rand_fq12(cid, rng), PR.rand_fq12(cid, rng)
    cyc = PR.from_flat(cid, PR.easy_part(cid, fl(a)))
    assert fl(run(exe, tmp_path, cid, 0, [a + b], 12)[0]) == PR.fmul(cid, fl(a), fl(b))
    assert fl(run(exe, tmp_path, cid, 1, [a], 12)[0]) == PR.fmul(cid, fl(a), fl(a))
    assert fl(run(exe, tmp_path, cid, 2, [cyc], 12)[0]) == PR.fmul(cid, fl(cyc), fl(cyc))
    assert PR.fmul(cid, fl(run(exe, tmp_path, cid, 3, [a], 12)[0]), fl(a)) == PR.ONE
    assert [fl(x) for x in run(exe, tmp_path, cid, 4, [a], 36)] == [PR.fpow(cid, fl(a), q ** k) for k in (1, 2, 3)]
    assert fl(run(exe, tmp_path, cid, 6, [a], 12)[0]) == PR.final_exp_ref(cid, fl(a))
    ci = O.CURVES[cid]
    P = PR.g_mul(cid, 1, ci.g1, 5)
    e = run(exe, tmp_path, cid, 7, [PR.pt_vals(P, ci.g2), PR.pt_vals(None, ci.g2), PR.pt_vals(P, None)], 12)
    assert fl(e[0]) == PR.pairing_ref(cid, P, ci.g2)
    assert fl(e[1]) == PR.ONE and fl(e[2]) == PR.ONE


def test_undefined_op(exe, tmp_path):
    (tmp_path / "in.bin").write_bytes(struct.pack("<iiQ", 0, 8, 1) + bytes(32 * 12))
    r = subprocess.run([exe, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], capture_output=True, text=True)
    assert r.returncode == 2 and "not defined" in r.stderr
