"""CPU: the PLONK control flow (snarkjs_b200/csrc/plonk_flow.h: rounds, Keccak transcript, round-5 scalars) and the
per-element functions the CUDA kernels call (plonk.cuh), compiled with g++ behind a host backend
(tests/host/host_plonk.cpp; NTT / MSM borrowed from the oracle) and compared with oracle/plonk.py proof for proof."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from oracle import oracle as orc
from oracle import plonk

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BLINDERS = [0x2000 + 7919 * i for i in range(11)]


@pytest.fixture(scope="module")
def hostlib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("hp") / "libhostplonk.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so,
                           os.path.join(ROOT, "tests", "host", "host_plonk.cpp"), "-ldl"])
    lib = ctypes.CDLL(so)
    lib.hp_plonk_prove.restype = ctypes.c_int
    lib.hp_plonk_prove.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_uint64, ctypes.c_char_p, ctypes.c_uint64,
                                   ctypes.c_char_p, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_int]
    lib.hp_keccak256.argtypes = [ctypes.c_char_p, ctypes.c_uint64, ctypes.c_char_p]
    return lib


def host_prove(lib, zkey: bytes, wtns: bytes, blinders, ci=orc.CURVES[orc.BN254]):
    _, wit = orc.read_wtns(wtns)
    out = ctypes.create_string_buffer(9 * 2 * ci.n8q + 6 * 32)
    err = ctypes.create_string_buffer(256)
    bl = b"".join(ci.fr_to_mont(b) for b in blinders)
    rc = lib.hp_plonk_prove(orc.build().encode(), zkey, len(zkey), wit, len(wit) // 32, bl, out, err, 256)
    return rc, err.value.decode(), out.raw


def proof_from_bytes(raw: bytes, ci=orc.CURVES[orc.BN254]):
    names = ["A", "B", "C", "Z", "T1", "T2", "T3", "Wxi", "Wxiw"]
    sg = 2 * ci.n8q
    proof = {k: plonk._g1_obj(ci.g1_from_affine_bytes(raw[sg * i:sg * i + sg])) for i, k in enumerate(names)}
    for i, k in enumerate(["eval_a", "eval_b", "eval_c", "eval_s1", "eval_s2", "eval_zw"]):
        proof[k] = str(ci.fr_from_mont(raw[9 * sg + 32 * i:9 * sg + 32 * i + 32]))
    proof["protocol"] = "plonk"
    proof["curve"] = ci.name
    return proof


def test_host_keccak(hostlib):
    for msg in (b"", b"abc", b"x" * 135, b"y" * 136, b"z" * 500):
        out = ctypes.create_string_buffer(32)
        hostlib.hp_keccak256(msg, len(msg), out)
        assert out.raw == plonk.keccak256(msg)


def test_host_flow_reference_fixture(hostlib, golden):
    g = golden("plonk_case.npz")
    zkey, wtns = bytes(g["zkey"]), bytes(g["wtns"])
    rc, err, raw = host_prove(hostlib, zkey, wtns, BLINDERS)
    assert rc == 0, err
    want, _ = plonk.plonk_prove(zkey, wtns, BLINDERS)
    assert proof_from_bytes(raw) == want


@pytest.mark.parametrize("n_gates", [13, 120, 500])
def test_host_flow_synthetic(hostlib, n_gates):
    gates, adds, n_vars, n_pub, wit = plonk.chain_gates(n_gates)
    zkey = plonk.plonk_setup_synth(gates, adds, n_vars, n_pub, tau=0xABCDEF0123456789)
    wtns = plonk.wtns_bytes(wit)
    rc, err, raw = host_prove(hostlib, zkey, wtns, BLINDERS)
    assert rc == 0, err
    want, public = plonk.plonk_prove(zkey, wtns, BLINDERS)
    got = proof_from_bytes(raw)
    assert got == want
    assert plonk.plonk_verify(plonk.plonk_vk(zkey), public, got)


@pytest.mark.parametrize("n_gates,n_pub,with_additions", [(29, 3, True), (60, 5, False), (16, 1, False), (8, 2, False)])
def test_host_flow_shapes(hostlib, n_gates, n_pub, with_additions):
    """Several public inputs (PI(X) sums several Lagrange polynomials), no additions at all, a gate count equal to the
    domain size, and the minimum domain (8)."""
    gates, adds, n_vars, n_pub, wit = plonk.chain_gates(n_gates, n_pub=n_pub, with_additions=with_additions)
    zkey = plonk.plonk_setup_synth(gates, adds, n_vars, n_pub, tau=31337 + n_gates)
    wtns = plonk.wtns_bytes(wit)
    rc, err, raw = host_prove(hostlib, zkey, wtns, BLINDERS)
    assert rc == 0, err
    want, public = plonk.plonk_prove(zkey, wtns, BLINDERS)
    assert len(public) == n_pub
    got = proof_from_bytes(raw)
    assert got == want
    assert plonk.plonk_verify(plonk.plonk_vk(zkey), public, got)


def test_host_flow_reference_circuit2(hostlib, golden, reference_plonk_key):
    """The reference's larger PLONK key (test/circuit2: domain 2048, 1001 additions, 4 public signals), rebuilt byte for byte
    from its r1cs, with the reference's own witness."""
    zkey, wtns = reference_plonk_key(golden("plonk_setup_cases.npz"), "c2048")
    rc, err, raw = host_prove(hostlib, zkey, wtns, BLINDERS)
    assert rc == 0, err
    want, public = plonk.plonk_prove(zkey, wtns, BLINDERS)
    assert len(public) == 4 and proof_from_bytes(raw) == want


def test_host_flow_deep_addition_chain(hostlib):
    """Additions that each depend on the previous one: one dependency level per addition (plonk_addition_levels must keep
    the reference's sequential semantics, plonk_prove.js:166-211)."""
    gates, adds, n_vars, n_pub, wit = plonk.chain_gates(100, deep_additions=True)
    assert len(adds) > 20
    zkey = plonk.plonk_setup_synth(gates, adds, n_vars, n_pub, tau=424242)
    wtns = plonk.wtns_bytes(wit)
    rc, err, raw = host_prove(hostlib, zkey, wtns, BLINDERS)
    assert rc == 0, err
    want, public = plonk.plonk_prove(zkey, wtns, BLINDERS)
    assert proof_from_bytes(raw) == want and plonk.plonk_verify(plonk.plonk_vk(zkey), public, want)


def test_host_flow_bls12381(hostlib):
    """Same flow on BLS12-381 (12-limb base field in the transcript, 255-bit scalar field); no pairing check here."""
    ci = orc.CURVES[orc.BLS12_381]
    gates, adds, n_vars, n_pub, wit = plonk.chain_gates(120, r=ci.r)
    zkey = plonk.plonk_setup_synth(gates, adds, n_vars, n_pub, tau=99991, curve=orc.BLS12_381)
    wtns = plonk.wtns_bytes(wit, ci.r)
    rc, err, raw = host_prove(hostlib, zkey, wtns, BLINDERS, ci)
    assert rc == 0, err
    want, public = plonk.plonk_prove(zkey, wtns, BLINDERS)
    assert proof_from_bytes(raw, ci) == want
    assert plonk.plonk_verify(plonk.plonk_vk(zkey), public, want)        # BLS12-381 pairing: oracle/pairing_bls.py


def test_host_flow_errors(hostlib):
    gates, adds, n_vars, n_pub, wit = plonk.chain_gates(40)
    zkey = plonk.plonk_setup_synth(gates, adds, n_vars, n_pub, tau=12345)
    bad = list(wit)
    bad[4] = (bad[4] + 1) % orc.P_BN_R
    rc, err, _ = host_prove(hostlib, zkey, plonk.wtns_bytes(bad), BLINDERS)
    assert rc != 0 and ("Copy constraints does not match" in err or "not divisible" in err)
    rc, err, _ = host_prove(hostlib, zkey, plonk.wtns_bytes(wit[:-1]), BLINDERS)
    assert rc != 0 and err.startswith("Invalid witness length. Circuit: ")
    g16 = bytearray(zkey)
    # protocol id lives in section 1: flip it to groth16
    idx = bytes(g16).index(b"\x01\x00\x00\x00\x04\x00\x00\x00\x00\x00\x00\x00\x02\x00\x00\x00")
    g16[idx + 12] = 1
    rc, err, _ = host_prove(hostlib, bytes(g16), plonk.wtns_bytes(wit), BLINDERS)
    assert rc != 0 and err == "zkey file is not plonk"


def test_host_parser_rejects_malformed_keys(hostlib):
    """plonk_parse_zkey (used verbatim by sb_plonk_load) must fail cleanly on truncated or inconsistent containers."""
    import struct
    gates, adds, n_vars, n_pub, wit = plonk.chain_gates(13)
    zkey = plonk.plonk_setup_synth(gates, adds, n_vars, n_pub, tau=99)
    wtns = plonk.wtns_bytes(wit)
    for cut in (0, 3, 11, 12, 40, 200, len(zkey) // 2, len(zkey) - 1):
        rc, err, _ = host_prove(hostlib, zkey[:cut], wtns, BLINDERS)
        assert rc != 0 and err, cut
    bad = bytearray(zkey)
    bad[0:4] = b"wtns"
    rc, err, _ = host_prove(hostlib, bytes(bad), wtns, BLINDERS)
    assert rc != 0 and "Invalid File format" in err
    # a section length that runs past the end of the file
    bad = bytearray(zkey)
    struct.pack_into("<Q", bad, 16, 1 << 40)
    rc, err, _ = host_prove(hostlib, bytes(bad), wtns, BLINDERS)
    assert rc != 0 and err == "Invalid file size"
    # a section id PLONK does not use, twice
    bad = bytearray(zkey) + struct.pack("<IQ", 16, 0) * 2
    struct.pack_into("<I", bad, 8, struct.unpack_from("<I", zkey, 8)[0] + 2)
    rc, err, _ = host_prove(hostlib, bytes(bad), wtns, BLINDERS)
    assert rc != 0 and err == "Section Duplicated 16"
    # domain size that is not a power of two (header field at a fixed offset inside section 2)
    data, secs = orc.read_binfile(zkey, "zkey", 2)
    pos = secs[2][0][0] + 4 + 32 + 4 + 32 + 8
    bad = bytearray(zkey)
    struct.pack_into("<I", bad, pos, 12)
    rc, err, _ = host_prove(hostlib, bytes(bad), wtns, BLINDERS)
    assert rc != 0 and "power of two" in err


def test_host_flow_with_emulated_ptx_arithmetic(tmp_path, golden):
    """Same flow with fp.cuh's device code path (PTX carry chains emulated instruction by instruction) instead of the
    fast host multiply: the arithmetic the kernels execute, inside the PLONK element functions."""
    so = str(tmp_path / "libhostplonk_ptx.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-DSB_HOST_EMULATE_PTX", "-shared", "-fPIC", "-o", so,
                           os.path.join(ROOT, "tests", "host", "host_plonk.cpp"), "-ldl"])
    lib = ctypes.CDLL(so)
    lib.hp_plonk_prove.restype = ctypes.c_int
    lib.hp_plonk_prove.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_uint64, ctypes.c_char_p, ctypes.c_uint64,
                                   ctypes.c_char_p, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_int]
    g = golden("plonk_case.npz")
    zkey, wtns = bytes(g["zkey"]), bytes(g["wtns"])
    rc, err, raw = host_prove(lib, zkey, wtns, BLINDERS)
    assert rc == 0, err
    assert proof_from_bytes(raw) == plonk.plonk_prove(zkey, wtns, BLINDERS)[0]


def test_openmp_build_of_the_host_flow_gives_the_same_proof(hostlib):
    """bench.py's reference arm compiles the same sources with -O3 -fopenmp (bench_plonk.host_flow_lib): the element loops
    run in parallel, the proof bytes must not change."""
    import bench_plonk as B
    gates, adds, n_vars, n_pub, wit = plonk.chain_gates(500)
    zkey = plonk.plonk_setup_synth(gates, adds, n_vars, n_pub, tau=0xABCDEF0123456789)
    wtns = plonk.wtns_bytes(wit)
    rc, err, raw = host_prove(hostlib, zkey, wtns, [7 + i for i in range(11)])
    assert rc == 0, err
    _, w = orc.read_wtns(wtns)
    ci = orc.CURVES[orc.BN254]
    _, raw_omp = B.cpu_prove("plonk", zkey, np.frombuffer(bytes(w), np.uint8), ci.r, ci.n8q, 4)
    assert raw_omp == raw
