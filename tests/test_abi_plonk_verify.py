"""CPU: the PLONK / fflonk verifiers' C entry points and Python wrappers without a GPU (null context, no-device error), the
verification key export against the reference's own vk.json files, the JSON -> vk / proof byte conversion against the
oracle, the status -> message / log level mapping, the wrappers' host-side decisions (signal count, signals outside
[0, r), an invalid fflonk C0) in the reference's order, and the evaluation decoding of Fr.fromObject."""
import ctypes
import json
import os

import numpy as np
import pytest

from oracle import oracle as O
from oracle import plonk as OP
from snarkjs_b200 import _native as N
from snarkjs_b200 import fflonk, plonk

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BN = O.CURVES[O.BN254]


def _golden(name):
    g = np.load(os.path.join(ROOT, "tests", "golden", name))
    return {k: bytes(g[k]) for k in g.files}


class Log:
    def __init__(self):
        self.lines = []

    def __getattr__(self, level):
        return lambda msg: self.lines.append((level, msg))


def test_entries_refuse_null_context():
    L = N.lib()
    buf = ctypes.create_string_buffer(4096)
    st = (ctypes.c_int32 * 4)()
    for fn in (L.sb_plonk_verify_batch, L.sb_fflonk_verify_batch):
        assert fn(None, buf, 704, 1, 3, buf, buf, 1, st) == -1
        assert fn(None, buf, 704, 1, 3, buf, buf, 0, st) == -1


def test_wrappers_need_a_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    g = _golden("plonk_case.npz")
    vk, pub, proof = json.loads(g["vk_json"]), json.loads(g["public_json"]), json.loads(g["proof_json"])
    with pytest.raises(plonk.SbError, match="no CUDA device"):
        plonk.verify(vk, pub, proof)
    with pytest.raises(plonk.SbError, match="no CUDA device"):
        plonk.verify_batch(vk, [(pub, proof)])
    f = _golden("fflonk_case.npz")
    fvk = json.loads(f["vk_json"])
    fproof = {"polynomials": {k: ["1", "2", "1"] for k in fflonk.POINTS}, "evaluations": {k: "1" for k in fflonk.EVALS}}
    with pytest.raises(fflonk.SbError, match="no CUDA device"):
        fflonk.verify(fvk, json.loads(f["public_json"]), fproof)


def test_verification_keys_match_the_reference_files():
    g = _golden("plonk_case.npz")
    assert plonk.verification_key(g["zkey"]) == json.loads(g["vk_json"])
    f = _golden("fflonk_case.npz")
    assert fflonk.verification_key(f["zkey"]) == json.loads(f["vk_json"])


def test_fr_root_is_the_references():
    for cid in (O.BN254, O.BLS12_381):
        ci = O.CURVES[cid]
        for k in (0, 1, 3, 11, O.fr_s(cid)):
            assert plonk.fr_root(ci.r, k) == OP._fr_w(ci, k)
        with pytest.raises(plonk.SbError, match="2-adicity"):
            plonk.fr_root(ci.r, O.fr_s(cid) + 1)


def test_vk_and_proof_bytes():
    g = _golden("plonk_case.npz")
    zkey = g["zkey"]
    vk = plonk.verification_key(zkey)
    zk = OP.read_plonk_zkey(zkey)
    want = b"".join(zk[k] for k in ("Qm", "Ql", "Qr", "Qo", "Qc", "S1", "S2", "S3")) + zk["X_2"] + zk["k1"] + zk["k2"]
    assert plonk.vk_bytes(vk) == want                      # the zkey's own header bytes
    proof, _pub = OP.plonk_prove(zkey, g["wtns"], [0x77 + i for i in range(11)])
    raw = plonk.proof_bytes(proof, 32, BN.q, BN.r)
    assert len(raw) == 9 * 64 + 6 * 32
    assert plonk.proof_to_object(BN, raw) == {**proof, "curve": BN.name}
    f = _golden("fflonk_case.npz")
    fz = f["zkey"]
    fvk = fflonk.verification_key(fz)
    from oracle import fflonk as OF
    z = OF.read_fflonk_zkey(fz)
    assert fflonk.vk_bytes(fvk) == (z["C0"] + z["X_2"] + z["k1"] + z["k2"] + BN.fr_to_mont(OP._fr_w(BN, z["power"]))
                                    + z["w3"] + z["w4"] + z["w8"] + z["wr"])
    fproof, _ = OF.fflonk_prove(fz, f["wtns"], [0x99 + i for i in range(9)])
    raw = fflonk.proof_bytes(fproof, 32, BN.q, BN.r)
    assert len(raw) == 4 * 64 + 16 * 32
    assert fflonk.proof_to_object(BN, raw) == {**fproof, "curve": BN.name}


def test_evaluation_decoding_follows_fr_from_object():
    """Fr.fromObject writes the value into 32 bytes (mod 2^256), then toMontgomery reduces it mod r: eval + r and
    eval + 2^256 decode to eval, so from JSON "evaluations are not valid" cannot fire (the oracle's 0 <= v < r rejects)."""
    r = BN.r
    for v in (0, 1, 12345, r - 1):
        want = BN.fr_to_mont(v)
        assert plonk.fr_bytes(v, r) == want
        assert plonk.fr_bytes(v + r, r) == want
        assert plonk.fr_bytes(v + (1 << 256), r) == want
        assert plonk.fr_bytes(str(v + 3 * r), r) == want
    assert plonk.fr_bytes((1 << 256) - 1, r) == BN.fr_to_mont(((1 << 256) - 1) % r)


def test_status_messages_and_levels():
    for mod, ok, msgs in ((plonk, "OK!", {1: ("warn", "Invalid Proof"), 2: ("error", "Public inputs are not valid."),
                                           3: ("error", "Proof commitments are not valid."), 4: ("error", "Proof evaluations are not valid"),
                                           5: ("error", "Invalid number of public inputs")}),
                          (fflonk, "PROOF VERIFIED SUCCESSFULLY", {1: ("warn", "Invalid Proof"), 2: ("error", "Public inputs are not valid."),
                                                                   3: ("error", "Proof commitments are not valid"),
                                                                   4: ("error", "Proof evaluations are not valid."),
                                                                   5: ("error", "Number of public signals does not match with vk")})):
        assert mod.VERIFY_MESSAGES == msgs
        for s in range(6):
            log = Log()
            plonk._log_status(log, mod.VERIFY_MESSAGES, s, ok)
            assert log.lines == [("info", ok)] if s == 0 else [msgs[s]]


def _off_curve(p):
    return [p[0], str((int(p[1]) + 1) % BN.q), "1"]


def test_host_decisions_in_reference_order():
    """Items the device call cannot take are decided on the host, in the reference's order, without a device: PLONK checks
    the commitments before the signal count, fflonk the count first; an invalid fflonk C0 fails every item with 3."""
    g = _golden("plonk_case.npz")
    vk, pub, proof = json.loads(g["vk_json"]), json.loads(g["public_json"]), json.loads(g["proof_json"])
    bad = dict(proof, B=_off_curve(proof["B"]))
    items = [(pub[:1], proof), (pub[:1], bad), (pub + ["1"], bad), ([str(BN.r)] + pub[1:], proof),
             ([str(1 << 256)] + pub[1:], bad), (["-1"] + pub[1:], proof)]
    assert plonk.verify_status(vk, items) == [5, 3, 3, 2, 3, 2]
    log = Log()
    assert plonk.verify(vk, pub[:1], bad, logger=log) is False
    assert log.lines == [("error", "Proof commitments are not valid.")]
    assert plonk.verify(vk, pub[:1], bad) is False         # the reference throws here without a logger
    log = Log()
    assert plonk.verify_batch(vk, items[:2], logger=log) == [False, False]
    assert log.lines == [("error", "Invalid number of public inputs"), ("error", "Proof commitments are not valid.")]

    f = _golden("fflonk_case.npz")
    fvk, fpub = json.loads(f["vk_json"]), json.loads(f["public_json"])
    fproof = {"polynomials": {k: [str(BN.g1[0]), str(BN.g1[1]), "1"] for k in fflonk.POINTS},
              "evaluations": {k: "1" for k in fflonk.EVALS}}
    fbad = {"polynomials": dict(fproof["polynomials"], W1=["1", "1", "1"]), "evaluations": fproof["evaluations"]}
    short = fpub[:-1]
    items = [(short, fbad), (fpub + ["1"], fproof), ([str(BN.r)] + fpub[1:], fbad), ([str(BN.r)] + fpub[1:], fproof)]
    assert fflonk.verify_status(fvk, items) == [5, 5, 3, 2]
    c0_bad = dict(fvk, C0=_off_curve(fvk["C0"]))
    assert fflonk.verify_status(c0_bad, [(fpub, fproof), (short, fproof), (fpub, fbad)]) == [3, 5, 3]
    log = Log()
    assert fflonk.verify(c0_bad, fpub, fproof, logger=log) is False
    assert log.lines == [("error", "Proof commitments are not valid")]
    assert fflonk.verify(fvk, short, fproof) is False      # the reference throws here without a logger
