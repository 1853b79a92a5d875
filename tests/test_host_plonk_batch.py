"""CPU: the batched PLONK control flow (snarkjs_b200/csrc/plonk_flow.h plonk_prove_flow_batch: K proofs in lockstep,
array-major work arrays, commitments at the padded length n + 6, per-proof status codes) behind a host batch backend
(tests/host/host_plonk_batch.cpp; the plonk.cuh element functions, NTT / MSM from the oracle), compared proof for proof
with the single-proof host flow and with oracle/plonk.py."""
import ctypes
import os
import subprocess

import pytest

from oracle import oracle as orc
from oracle import plonk

from .test_host_plonk import host_prove, proof_from_bytes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TEXTS = {3: "Copy constraints does not match", 4: "Polynomial is not divisible", 5: "T Polynomial is not well calculated"}


@pytest.fixture(scope="module")
def libs(tmp_path_factory):
    d = tmp_path_factory.mktemp("hpb")
    out = {}
    for name, src in (("batch", "host_plonk_batch.cpp"), ("single", "host_plonk.cpp")):
        so = str(d / f"lib{name}.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so, os.path.join(ROOT, "tests", "host", src), "-ldl"])
        out[name] = ctypes.CDLL(so)
    b = out["batch"]
    b.hp_plonk_prove_batch.restype = ctypes.c_int
    b.hp_plonk_prove_batch.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_uint64, ctypes.c_char_p, ctypes.c_uint64, ctypes.c_uint32,
                                       ctypes.c_char_p, ctypes.c_char_p, ctypes.POINTER(ctypes.c_int32), ctypes.c_char_p, ctypes.c_int]
    s = out["single"]
    s.hp_plonk_prove.restype = ctypes.c_int
    s.hp_plonk_prove.argtypes = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_uint64, ctypes.c_char_p, ctypes.c_uint64,
                                 ctypes.c_char_p, ctypes.c_char_p, ctypes.c_char_p, ctypes.c_int]
    return out


def chain_witnesses(wit, count, r):
    """Further valid witnesses of a chain_gates key: its gates depend only on the constant c of x_{i+1} = x_i^2 + c, so the
    chain re-run from other x_0 satisfies the same key.  wit = [1, x_m, x_0, ..., x_{m-1}]."""
    m = len(wit) - 2
    cst = (wit[3] - wit[2] * wit[2]) % r
    out = [list(wit)]
    for t in range(1, count):
        x = [(wit[2] + 1000 * t + 1) % r]
        for _ in range(m):
            x.append((x[-1] * x[-1] + cst) % r)
        out.append([1, x[m]] + x[:m])
    return out


def blinders_for(k):
    return [0x7000 + 104729 * i + 7919 * k for i in range(11)]


def batch_prove(lib, zkey, wtns_list, bls_list, ci):
    wits = [orc.read_wtns(w)[1] for w in wtns_list]
    count = len(wits)
    pb = 9 * 2 * ci.n8q + 6 * 32
    out = ctypes.create_string_buffer(count * pb)
    status = (ctypes.c_int32 * count)()
    err = ctypes.create_string_buffer(256)
    bl = b"".join(ci.fr_to_mont(b) for bls in bls_list for b in bls)
    rc = lib.hp_plonk_prove_batch(orc.build().encode(), zkey, len(zkey), b"".join(wits), len(wits[0]) // 32, count, bl, out, status, err, 256)
    return rc, err.value.decode(), [out.raw[i * pb:(i + 1) * pb] for i in range(count)], list(status)


def check_batch(libs, zkey, wtns_list, ci, oracle_checks=2):
    bls_list = [blinders_for(k) for k in range(len(wtns_list))]
    rc, err, proofs, status = batch_prove(libs["batch"], zkey, wtns_list, bls_list, ci)
    assert rc == 0, err
    assert status == [0] * len(wtns_list)
    for k, (wtns, bls) in enumerate(zip(wtns_list, bls_list)):
        src, serr, single = host_prove(libs["single"], zkey, wtns, bls, ci)
        assert src == 0, serr
        assert proofs[k] == single, k
        if k < oracle_checks:
            assert proof_from_bytes(proofs[k], ci) == plonk.plonk_prove(zkey, wtns, bls)[0]
    return proofs


@pytest.mark.parametrize("count", [1, 3, 5])
def test_batch_reference_fixture(libs, golden, count):
    g = golden("plonk_case.npz")
    zkey, wtns = bytes(g["zkey"]), bytes(g["wtns"])
    check_batch(libs, zkey, [wtns] * count, orc.CURVES[orc.BN254], oracle_checks=1)


@pytest.mark.parametrize("count", [1, 3, 5])
@pytest.mark.parametrize("n_gates,n_pub,with_additions,deep", [(13, 1, True, False), (120, 1, True, False), (60, 5, False, False),
                                                               (29, 3, True, False), (100, 1, True, True)])
def test_batch_synthetic(libs, count, n_gates, n_pub, with_additions, deep):
    """Chain keys: 13 and 120 gates, several public inputs, no additions, deep additions; distinct witnesses and blinders."""
    gates, adds, n_vars, n_pub, wit = plonk.chain_gates(n_gates, n_pub=n_pub, with_additions=with_additions, deep_additions=deep)
    zkey = plonk.plonk_setup_synth(gates, adds, n_vars, n_pub, tau=0xBA7C4 + n_gates)
    wl = [plonk.wtns_bytes(w) for w in chain_witnesses(wit, count, orc.P_BN_R)]
    proofs = check_batch(libs, zkey, wl, orc.CURVES[orc.BN254])
    assert len(set(proofs)) == count
    if count > 1:
        ci = orc.CURVES[orc.BN254]
        _, public = plonk.plonk_prove(zkey, wl[1], blinders_for(1))
        assert plonk.plonk_verify(plonk.plonk_vk(zkey), public, proof_from_bytes(proofs[1], ci))


@pytest.mark.parametrize("count", [1, 3])
def test_batch_bls12381(libs, count):
    ci = orc.CURVES[orc.BLS12_381]
    gates, adds, n_vars, n_pub, wit = plonk.chain_gates(120, r=ci.r)
    zkey = plonk.plonk_setup_synth(gates, adds, n_vars, n_pub, tau=99991, curve=orc.BLS12_381)
    wl = [plonk.wtns_bytes(w, ci.r) for w in chain_witnesses(wit, count, ci.r)]
    check_batch(libs, zkey, wl, ci, oracle_checks=1)


def test_batch_bad_witness_in_the_middle(libs):
    """Proof 1 of 3 breaks a copy constraint: its status names the reference's error, its slot is zero, and proofs 0 and 2
    are the single flow's bytes."""
    ci = orc.CURVES[orc.BN254]
    gates, adds, n_vars, n_pub, wit = plonk.chain_gates(40)
    zkey = plonk.plonk_setup_synth(gates, adds, n_vars, n_pub, tau=12345)
    ws = chain_witnesses(wit, 3, orc.P_BN_R)
    ws[1][4] = (ws[1][4] + 1) % orc.P_BN_R
    wl = [plonk.wtns_bytes(w) for w in ws]
    bls_list = [blinders_for(k) for k in range(3)]
    rc, err, proofs, status = batch_prove(libs["batch"], zkey, wl, bls_list, ci)
    assert rc == 0, err
    src, serr, _ = host_prove(libs["single"], zkey, wl[1], bls_list[1], ci)
    assert src != 0 and status[0] == 0 and status[2] == 0 and TEXTS[status[1]] == serr
    assert proofs[1] == bytes(len(proofs[1]))
    for k in (0, 2):
        assert proofs[k] == host_prove(libs["single"], zkey, wl[k], bls_list[k], ci)[2]


def test_batch_witness_length(libs):
    ci = orc.CURVES[orc.BN254]
    gates, adds, n_vars, n_pub, wit = plonk.chain_gates(13)
    zkey = plonk.plonk_setup_synth(gates, adds, n_vars, n_pub, tau=99)
    rc, err, _, _ = batch_prove(libs["batch"], zkey, [plonk.wtns_bytes(wit[:-1])] * 2, [blinders_for(0)] * 2, ci)
    assert rc == 2 and err.startswith("Invalid witness length. Circuit: ")
