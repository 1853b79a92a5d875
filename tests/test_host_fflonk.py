"""CPU: the fflonk control flow (snarkjs_b200/csrc/fflonk_flow.h) and the element functions the CUDA kernels call
(fflonk.cuh, plonk.cuh), compiled with g++ behind a host backend (tests/host/host_fflonk.cpp; NTT / MSM borrowed from
the oracle) and compared with oracle/fflonk.py proof for proof on the reference's own fflonk fixture key."""
import ctypes
import json
import os
import re
import struct
import subprocess

import pytest

from oracle import fflonk
from oracle import oracle as orc
from oracle import plonk

from tests import r1cs_shapes as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BLINDERS = [0x5000 + 15485863 * i for i in range(9)]


@pytest.fixture(scope="module")
def hostlib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("hf") / "libhostfflonk.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so,
                           os.path.join(ROOT, "tests", "host", "host_fflonk.cpp"), "-ldl"])
    lib = ctypes.CDLL(so)
    lib.hp_fflonk_prove.restype = ctypes.c_int
    lib.hp_fflonk_prove.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_uint64, ctypes.c_char_p, ctypes.c_uint64,
                                    ctypes.c_char_p, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_int]
    return lib


def host_prove(lib, zkey: bytes, wtns: bytes, blinders):
    ci = orc.CURVES[orc.BN254]
    _, wit = orc.read_wtns(wtns)
    out = ctypes.create_string_buffer(4 * 64 + 16 * 32)
    err = ctypes.create_string_buffer(256)
    bl = b"".join(ci.fr_to_mont(b) for b in blinders)
    rc = lib.hp_fflonk_prove(orc.build().encode(), zkey, len(zkey), wit, len(wit) // 32, bl, out, err, 256)
    return rc, err.value.decode(), out.raw


def proof_from_bytes(raw: bytes):
    ci = orc.CURVES[orc.BN254]
    pols = {k: plonk._g1_obj(ci.g1_from_affine_bytes(raw[64 * i:64 * i + 64])) for i, k in enumerate(("C1", "C2", "W1", "W2"))}
    evs = {k: str(ci.fr_from_mont(raw[256 + 32 * i:288 + 32 * i])) for i, k in enumerate(fflonk.EVAL_NAMES + ("inv",))}
    return {"polynomials": pols, "evaluations": evs, "protocol": "fflonk", "curve": "bn128"}


def test_host_fflonk_reference_fixture(hostlib, golden):
    g = golden("fflonk_case.npz")
    zkey, wtns = bytes(g["zkey"]), bytes(g["wtns"])
    rc, err, raw = host_prove(hostlib, zkey, wtns, BLINDERS)
    assert rc == 0, err
    want, public = fflonk.fflonk_prove(zkey, wtns, BLINDERS)
    got = proof_from_bytes(raw)
    assert got == want
    assert fflonk.fflonk_verify(json.loads(bytes(g["vk_json"])), public, got)


@pytest.mark.parametrize("n_gates,n_pub,with_additions", [(13, 1, True), (120, 1, True), (29, 3, True), (60, 5, False), (500, 1, True)]
                         + [pytest.param(label, None, None, id=label) for label, c in S.PLONK_CASES.items() if c[1] == orc.BN254])
def test_host_fflonk_synthetic(hostlib, n_gates, n_pub, with_additions):
    """Chain keys from fflonk_setup_synth; a label instead of a gate count takes the key fflonk_setup builds from a circuit
    of tests/r1cs_shapes.py, and where the reference rejects it the flow gives the same text."""
    if isinstance(n_gates, str):
        circ = S.case(n_gates)
        zkey, wtns, verify = S.fflonk_zkey(n_gates), circ.wtns(), S.PLONK_CASES[n_gates][3]
    else:
        gates, adds, n_vars, n_pub, wit = plonk.chain_gates(n_gates, n_pub=n_pub, with_additions=with_additions)
        zkey = fflonk.fflonk_setup_synth(gates, adds, n_vars, n_pub, tau=0xFACE0FF + n_gates, structured=n_gates < 200)
        wtns, verify = plonk.wtns_bytes(wit), n_gates < 200
    rc, err, raw = host_prove(hostlib, zkey, wtns, BLINDERS)
    if n_gates in S.FFLONK_ERRORS:
        assert rc != 0 and err == S.FFLONK_ERRORS[n_gates]
        with pytest.raises(ValueError, match=re.escape(err)):
            fflonk.fflonk_prove(zkey, wtns, BLINDERS)
        return
    assert rc == 0, err
    want, public = fflonk.fflonk_prove(zkey, wtns, BLINDERS)
    got = proof_from_bytes(raw)
    assert got == want
    if verify:
        assert fflonk.fflonk_verify(fflonk.fflonk_vk(zkey), public, got)


def test_host_fflonk_c0_section_not_the_interleave(hostlib):
    """The opening values of C0 are derived from ql..s3 only when section 17 equals the interleave of sections 7-14 (checked
    at load); a key whose section 17 differs takes the reference's direct evaluations instead.  Either way: oracle parity."""
    gates, adds, n_vars, n_pub, wit = plonk.chain_gates(40)
    zkey = bytearray(fflonk.fflonk_setup_synth(gates, adds, n_vars, n_pub, tau=77))
    data, secs = orc.read_binfile(bytes(zkey), "zkey", 2)
    pos = secs[17][0][0] + 5 * 32                       # one coefficient of C0
    zkey[pos] ^= 1
    wtns = plonk.wtns_bytes(wit)
    rc, err, raw = host_prove(hostlib, bytes(zkey), wtns, BLINDERS)
    assert rc == 0, err
    want, public = fflonk.fflonk_prove(bytes(zkey), wtns, BLINDERS)
    assert proof_from_bytes(raw) == want
    assert not fflonk.fflonk_verify(fflonk.fflonk_vk(bytes(zkey)), public, want)   # such a key cannot produce valid proofs


def test_host_fflonk_errors(hostlib, golden):
    g = golden("fflonk_case.npz")
    zkey, wtns = bytes(g["zkey"]), bytes(g["wtns"])
    _, w = orc.read_wtns(wtns)
    wit = [int.from_bytes(w[i:i + 32], "little") for i in range(0, len(w), 32)]
    bad = list(wit)
    bad[3] = (bad[3] + 1) % orc.P_BN_R
    rc, err, _ = host_prove(hostlib, zkey, plonk.wtns_bytes(bad), BLINDERS)
    assert rc != 0 and ("Copy constraints does not match" in err or "not divisible" in err)
    rc, err, _ = host_prove(hostlib, zkey, plonk.wtns_bytes(wit[:-1]), BLINDERS)
    assert rc != 0 and err.startswith("Invalid witness length. Circuit: ")
    rc, err, _ = host_prove(hostlib, bytes(golden("plonk_case.npz")["zkey"]), wtns, BLINDERS)
    assert rc != 0 and err == "zkey file is not fflonk"
    bad = bytearray(zkey) + struct.pack("<IQ", 20, 0) * 2                 # a section id fflonk does not use, twice
    struct.pack_into("<I", bad, 8, struct.unpack_from("<I", zkey, 8)[0] + 2)
    rc, err, _ = host_prove(hostlib, bytes(bad), wtns, BLINDERS)
    assert rc != 0 and err == "Section Duplicated 20"
