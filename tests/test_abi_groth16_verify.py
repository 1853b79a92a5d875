"""CPU: the Groth16 verifier's C entry points and Python wrappers without a GPU (null context, no-device error), the
verification key export against the oracle, the JSON -> vk / proof byte conversion (G.fromObject), the status -> bool and
message mapping, and the tower <-> flat Fq12 conversion the GPU pairing tests rely on."""
import ctypes
import os
import random

import numpy as np
import pytest

from oracle import oracle as O
from snarkjs_b200 import _native as N
from snarkjs_b200 import groth16
from tests import pairing_ref as PR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _golden_zkey():
    return np.load(os.path.join(ROOT, "tests", "golden", "groth16_case.npz"))["zkey"].tobytes()


def test_entries_refuse_null_context():
    L = N.lib()
    buf = ctypes.create_string_buffer(1024)
    st = (ctypes.c_int32 * 4)()
    assert L.sb_groth16_verify_batch(None, buf, 1024, 1, buf, buf, 1, st) == -1
    assert L.sb_groth16_verify_batch(None, buf, 1024, 1, buf, buf, 0, st) == -1
    for op in (0, 7, 8, -1):
        assert L.sb_pairing_eval(None, op, buf, 1, buf) == -1


def test_wrappers_need_a_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    vk = groth16.verification_key(_golden_zkey())
    ci = O.CURVES[O.BN254]
    proof = {"pi_a": [str(ci.g1[0]), str(ci.g1[1]), "1"], "pi_b": [[str(v) for v in ci.g2[0]], [str(v) for v in ci.g2[1]], ["1", "0"]],
             "pi_c": [str(ci.g1[0]), str(ci.g1[1]), "1"], "protocol": "groth16", "curve": "bn128"}
    pub = ["1"] * vk["nPublic"]
    with pytest.raises(groth16.SbError, match="no CUDA device"):
        groth16.verify(vk, pub, proof)
    with pytest.raises(groth16.SbError, match="no CUDA device"):
        groth16.verify_batch(vk, [(pub, proof)])


def test_verification_key_matches_oracle():
    zkey = _golden_zkey()
    vk = groth16.verification_key(zkey)
    o = O.zkey_vk(zkey)
    assert vk["protocol"] == "groth16" and vk["curve"] == "bn128" and vk["nPublic"] == o["nPublic"]
    assert "vk_alphabeta_12" not in vk
    g1 = lambda p: ["0", "1", "0"] if p is None else [str(p[0]), str(p[1]), "1"]
    g2 = lambda p: [[str(p[0][0]), str(p[0][1])], [str(p[1][0]), str(p[1][1])], ["1", "0"]]
    assert vk["vk_alpha_1"] == g1(o["alpha1"])
    assert (vk["vk_beta_2"], vk["vk_gamma_2"], vk["vk_delta_2"]) == (g2(o["beta2"]), g2(o["gamma2"]), g2(o["delta2"]))
    assert vk["IC"] == [g1(p) for p in o["IC"]]
    # the bytes handed to the C ABI: the zkey's own header points and section 3
    z = groth16.read_zkey_header_groth16(zkey)
    pos, _ = z["sections"][3]
    n8 = z["n8q"]
    want = z["vk_alpha_1"] + z["vk_beta_2"] + z["vk_gamma_2"] + z["vk_delta_2"] + zkey[pos:pos + 2 * n8 * (z["nPublic"] + 1)]
    assert groth16.vk_bytes(vk) == want


@pytest.mark.parametrize("cid", [O.BN254, O.BLS12_381], ids=["bn254", "bls12381"])
def test_point_conversion(cid):
    """G.fromObject: Jacobian (x, y, z) -> (x/z^2, y/z^3), z = 0 is infinity, coordinates taken mod q."""
    ci = O.CURVES[cid]
    q, n8 = ci.q, ci.n8q
    rng = random.Random(cid)
    x, y = ci.g1
    z = rng.randrange(2, q)
    obj = [str(x * z * z % q + q), str(y * z ** 3 % q), str(z)]
    assert groth16.point_bytes(obj, 1, n8, q) == ci.g1_affine_bytes(ci.g1)
    assert groth16.point_bytes([str(x), str(y), "1"], 1, n8, q) == ci.g1_affine_bytes(ci.g1)
    assert groth16.point_bytes(["5", "7", "0"], 1, n8, q) == bytes(2 * n8)
    assert groth16.point_bytes(["0", "1", "0"], 1, n8, q) == bytes(2 * n8)
    (x0, x1), (y0, y1) = ci.g2
    mul = lambda a, b: ((a[0] * b[0] - a[1] * b[1]) % q, (a[0] * b[1] + a[1] * b[0]) % q)
    zz = (rng.randrange(q), rng.randrange(q))
    z2 = mul(zz, zz)
    X, Y = mul((x0, x1), z2), mul((y0, y1), mul(z2, zz))
    obj = [[str(X[0]), str(X[1] + 2 * q)], [str(Y[0]), str(Y[1])], [str(zz[0]), str(zz[1])]]
    assert groth16.point_bytes(obj, 2, n8, q) == ci.g2_affine_bytes(ci.g2)
    assert groth16.point_bytes([["0", "0"], ["1", "0"], ["0", "0"]], 2, n8, q) == bytes(4 * n8)


def test_statuses_and_messages(monkeypatch):
    """verify / verify_batch map the C statuses to the reference's messages; signals >= r, or a count other than nPublic,
    are decided before the device call."""
    vk = groth16.verification_key(_golden_zkey())
    r = O.CURVES[O.BN254].r
    npub = vk["nPublic"]
    calls = []

    class FakeLib:
        def sb_groth16_verify_batch(self, h, vk_p, vk_len, n_public, pubs, prfs, count, out):
            calls.append(count)
            arr = np.ctypeslib.as_array(ctypes.cast(out, ctypes.POINTER(ctypes.c_int32)), (max(count, 1),))
            arr[:count] = [0, 1, 3][:count] + [0] * max(0, count - 3)
            return 0

    class FakeCurve:
        lib, handle = FakeLib(), None

        def check(self, rc):
            assert rc == 0

    proof = {"pi_a": ["1", "2", "1"], "pi_b": [["1", "0"], ["1", "0"], ["1", "0"]], "pi_c": ["1", "2", "1"]}
    pub = ["3"] * npub
    items = [(pub, proof), (pub, proof), ([str(r)] + pub[1:], proof), (pub, proof), (pub + ["1"], proof)]
    assert groth16.verify_status(vk, items, curve=FakeCurve()) == [0, 1, 2, 3, 1]
    assert calls == [3]

    class Log:
        def __init__(self): self.lines = []
        def error(self, m): self.lines.append(("error", m))
        def info(self, m): self.lines.append(("info", m))
    lg = Log()
    assert groth16.verify_batch(vk, items, logger=lg, curve=FakeCurve()) == [True, False, False, False, False]
    assert [m for _k, m in lg.lines] == ["Invalid proof", "Public inputs are not valid.", "Proof commitments are not valid.", "Invalid proof"]
    lg = Log()
    assert groth16.verify(vk, pub, proof, logger=lg, curve=FakeCurve()) and lg.lines == [("info", "OK!")]
    assert groth16.VERIFY_MESSAGES == {1: "Invalid proof", 2: "Public inputs are not valid.", 3: "Proof commitments are not valid."}


@pytest.mark.parametrize("cid", [O.BN254, O.BLS12_381], ids=["bn254", "bls12381"])
def test_tower_flat_conversion(cid):
    """to_flat / from_flat are inverse, map the tower's 1 and u to 1 and w^6 - beta, and multiplication commutes with them
    (the tower product done by hand: Fq12 = Fq6[w]/(w^2 - v), Fq6 = Fq2[v]/(v^3 - xi))."""
    rng = random.Random(3 + cid)
    q = PR.Q[cid]
    xi = (PR.BETA[cid], 1)
    f2m = lambda a, b: ((a[0] * b[0] - a[1] * b[1]) % q, (a[0] * b[1] + a[1] * b[0]) % q)
    f2a = lambda a, b: ((a[0] + b[0]) % q, (a[1] + b[1]) % q)

    def tmul(a, b):
        # as 6 Fq2 coefficients of w^0..w^5 with w^6 = xi
        A = [(a[(3 * (i % 2) + i // 2) * 2], a[(3 * (i % 2) + i // 2) * 2 + 1]) for i in range(6)]
        B = [(b[(3 * (i % 2) + i // 2) * 2], b[(3 * (i % 2) + i // 2) * 2 + 1]) for i in range(6)]
        c = [(0, 0)] * 11
        for i in range(6):
            for j in range(6):
                c[i + j] = f2a(c[i + j], f2m(A[i], B[j]))
        for i in range(10, 5, -1):
            c[i - 6] = f2a(c[i - 6], f2m(c[i], xi))
        out = [0] * 12
        for i in range(6):
            k, j = i % 2, i // 2
            out[(3 * k + j) * 2], out[(3 * k + j) * 2 + 1] = c[i]
        return out
    for _ in range(4):
        a, b = PR.rand_fq12(cid, rng), PR.rand_fq12(cid, rng)
        assert PR.from_flat(cid, PR.to_flat(cid, a)) == a
        assert PR.to_flat(cid, tmul(a, b)) == PR.fmul(cid, PR.to_flat(cid, a), PR.to_flat(cid, b))
    one = [1] + [0] * 11
    u = [0, 1] + [0] * 10
    assert PR.to_flat(cid, one) == PR.ONE
    assert PR.to_flat(cid, u) == [(-PR.BETA[cid]) % q] + [0] * 5 + [1] + [0] * 5
