"""CPU: the batched fflonk control flow (snarkjs_b200/csrc/fflonk_flow.h fflonk_prove_flow_batch: K proofs in lockstep,
array-major work arrays sharing memory across rounds, commitments at the common row length 9n, per-proof status codes)
behind a host batch backend (tests/host/host_fflonk_batch.cpp; the fflonk.cuh / plonk.cuh element functions, NTT / MSM
from the oracle), compared proof for proof with the single-proof host flow and with oracle/fflonk.py."""
import ctypes
import os
import subprocess

import pytest

from oracle import fflonk
from oracle import oracle as orc
from oracle import plonk

from tests import r1cs_shapes as S

from .test_host_fflonk import host_prove, proof_from_bytes
from .test_host_plonk_batch import chain_witnesses

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PB = 4 * 64 + 16 * 32


@pytest.fixture(scope="module")
def libs(tmp_path_factory):
    d = tmp_path_factory.mktemp("hfb")
    out = {}
    for name, src in (("batch", "host_fflonk_batch.cpp"), ("single", "host_fflonk.cpp")):
        so = str(d / f"lib{name}.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so, os.path.join(ROOT, "tests", "host", src), "-ldl"])
        out[name] = ctypes.CDLL(so)
    b = out["batch"]
    b.hp_fflonk_prove_batch.restype = ctypes.c_int
    b.hp_fflonk_prove_batch.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_uint64, ctypes.c_char_p, ctypes.c_uint64, ctypes.c_uint32,
                                        ctypes.c_char_p, ctypes.c_char_p, ctypes.POINTER(ctypes.c_int32), ctypes.c_char_p, ctypes.c_int]
    b.hp_fflonk_error_text.restype = ctypes.c_char_p
    b.hp_fflonk_error_text.argtypes = [ctypes.c_int]
    s = out["single"]
    s.hp_fflonk_prove.restype = ctypes.c_int
    s.hp_fflonk_prove.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_uint64, ctypes.c_char_p, ctypes.c_uint64,
                                  ctypes.c_char_p, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_int]
    return out


def blinders_for(k):
    return [0x5000 + 15485863 * i + 7919 * k for i in range(9)]


def batch_prove(lib, zkey, wtns_list, bls_list):
    ci = orc.CURVES[orc.BN254]
    wits = [orc.read_wtns(w)[1] for w in wtns_list]
    count = len(wits)
    out = ctypes.create_string_buffer(count * PB)
    status = (ctypes.c_int32 * count)()
    err = ctypes.create_string_buffer(256)
    bl = b"".join(ci.fr_to_mont(b) for bls in bls_list for b in bls)
    rc = lib.hp_fflonk_prove_batch(orc.build().encode(), zkey, len(zkey), b"".join(wits), len(wits[0]) // 32, count, bl, out, status, err, 256)
    return rc, err.value.decode(), [out.raw[i * PB:(i + 1) * PB] for i in range(count)], list(status)


def check_batch(libs, zkey, wtns_list, oracle_checks=2):
    bls_list = [blinders_for(k) for k in range(len(wtns_list))]
    rc, err, proofs, status = batch_prove(libs["batch"], zkey, wtns_list, bls_list)
    assert rc == 0, err
    assert status == [0] * len(wtns_list)
    for k, (wtns, bls) in enumerate(zip(wtns_list, bls_list)):
        src, serr, single = host_prove(libs["single"], zkey, wtns, bls)
        assert src == 0, serr
        assert proofs[k] == single, k
        if k < oracle_checks:
            assert proof_from_bytes(proofs[k]) == fflonk.fflonk_prove(zkey, wtns, bls)[0]
    return proofs


@pytest.mark.parametrize("count", [1, 3, 5])
def test_batch_reference_fixture(libs, golden, count):
    g = golden("fflonk_case.npz")
    zkey, wtns = bytes(g["zkey"]), bytes(g["wtns"])
    check_batch(libs, zkey, [wtns] * count, oracle_checks=1)


@pytest.mark.parametrize("count", [1, 3, 5])
@pytest.mark.parametrize("n_gates,n_pub,with_additions,deep", [(13, 1, True, False), (120, 3, True, False), (500, 1, False, False),
                                                               (100, 1, True, True)])
def test_batch_synthetic(libs, count, n_gates, n_pub, with_additions, deep):
    """Chain keys: 13 gates, 120 with 3 public inputs, 500 without additions, deep additions; distinct witnesses and blinders."""
    gates, adds, n_vars, n_pub, wit = plonk.chain_gates(n_gates, n_pub=n_pub, with_additions=with_additions, deep_additions=deep)
    zkey = fflonk.fflonk_setup_synth(gates, adds, n_vars, n_pub, tau=0xFACE0FF + n_gates, structured=n_gates < 200)
    wl = [plonk.wtns_bytes(w) for w in chain_witnesses(wit, count, orc.P_BN_R)]
    proofs = check_batch(libs, zkey, wl, oracle_checks=1 if n_gates >= 200 else 2)
    assert len(set(proofs)) == count
    if count > 1 and n_gates < 200:
        _, public = fflonk.fflonk_prove(zkey, wl[1], blinders_for(1))
        assert fflonk.fflonk_verify(fflonk.fflonk_vk(zkey), public, proof_from_bytes(proofs[1]))


@pytest.mark.parametrize("count", [1, 3])
def test_batch_c0_section_not_the_interleave(libs, count):
    """The shape key "bits" with one bit of section 17 flipped: C0's opening values come from its own evaluations, which
    join round 3's reduction."""
    zkey = bytearray(S.fflonk_zkey("bits"))
    _, secs = orc.read_binfile(bytes(zkey), "zkey", 2)
    zkey[secs[17][0][0] + 5 * 32] ^= 1
    wtns = S.case("bits").wtns()
    check_batch(libs, bytes(zkey), [wtns] * count, oracle_checks=1)


@pytest.mark.parametrize("label", [label for label, c in S.PLONK_CASES.items() if c[1] == orc.BN254 and label in S.FFLONK_ERRORS])
def test_batch_refused_shape(libs, label):
    """A key no witness proves: every proof of the batch gets the single flow's text."""
    zkey, wtns = S.fflonk_zkey(label), S.case(label).wtns()
    rc, err, proofs, status = batch_prove(libs["batch"], zkey, [wtns] * 2, [blinders_for(0), blinders_for(1)])
    assert rc == 0, err
    assert [libs["batch"].hp_fflonk_error_text(s).decode() for s in status] == [S.FFLONK_ERRORS[label]] * 2
    assert proofs == [bytes(PB)] * 2


def test_batch_bad_witness_in_the_middle(libs):
    """Proof 1 of 3 breaks a copy constraint: its status maps to the single flow's text, its slot is zero, and proofs 0 and 2
    are the single flow's bytes."""
    gates, adds, n_vars, n_pub, wit = plonk.chain_gates(40)
    zkey = fflonk.fflonk_setup_synth(gates, adds, n_vars, n_pub, tau=12345)
    ws = chain_witnesses(wit, 3, orc.P_BN_R)
    ws[1][4] = (ws[1][4] + 1) % orc.P_BN_R
    wl = [plonk.wtns_bytes(w) for w in ws]
    bls_list = [blinders_for(k) for k in range(3)]
    rc, err, proofs, status = batch_prove(libs["batch"], zkey, wl, bls_list)
    assert rc == 0, err
    src, serr, _ = host_prove(libs["single"], zkey, wl[1], bls_list[1])
    assert src != 0 and status[0] == 0 and status[2] == 0
    assert libs["batch"].hp_fflonk_error_text(status[1]).decode() == serr
    assert proofs[1] == bytes(PB)
    for k in (0, 2):
        assert proofs[k] == host_prove(libs["single"], zkey, wl[k], bls_list[k])[2]


def test_batch_witness_length(libs):
    gates, adds, n_vars, n_pub, wit = plonk.chain_gates(13)
    zkey = fflonk.fflonk_setup_synth(gates, adds, n_vars, n_pub, tau=99)
    rc, err, _, _ = batch_prove(libs["batch"], zkey, [plonk.wtns_bytes(wit[:-1])] * 2, [blinders_for(0)] * 2)
    assert rc == 2 and err.startswith("Invalid witness length. Circuit: ")
