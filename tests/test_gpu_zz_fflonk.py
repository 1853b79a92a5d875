"""GPU parity of the fflonk prover (sb_fflonk_load / sb_fflonk_prove through the C ABI) against oracle/fflonk.py:
identical proof objects for identical blinders on the reference's own fixture key (test/fflonk) and on synthetic keys,
plus the reference's error texts."""
import json

import pytest

pytestmark = pytest.mark.gpu

BLINDERS = [0x6000 + 32452843 * i for i in range(9)]


@pytest.fixture(scope="module")
def env():
    import snarkjs_b200
    from oracle import fflonk as off
    from oracle import oracle as orc
    from oracle import plonk as op
    curve = snarkjs_b200.getCurveFromName("bn128")
    ci = orc.CURVES[orc.BN254]
    yield {"sb": snarkjs_b200, "orc": orc, "op": op, "off": off, "curve": curve, "bl": b"".join(ci.fr_to_mont(b) for b in BLINDERS)}
    curve.terminate()


def test_fflonk_reference_fixture(env, golden):
    g = golden("fflonk_case.npz")
    zkey, wtns = bytes(g["zkey"]), bytes(g["wtns"])
    pk = env["sb"].fflonk.ProvingKey(zkey, env["curve"])
    try:
        proof, public = env["sb"].fflonk.prove(pk, wtns, env["bl"])
        want, wpub = env["off"].fflonk_prove(zkey, wtns, BLINDERS)
        assert public == wpub == json.loads(bytes(g["public_json"]))
        assert proof == want
        vk = json.loads(bytes(g["vk_json"]))
        assert env["off"].fflonk_verify(vk, public, proof)
        p2, _ = env["sb"].fflonk.prove(pk, wtns)                      # random blinders: another valid proof
        assert p2 != proof and env["off"].fflonk_verify(vk, public, p2)
    finally:
        pk.release()


@pytest.mark.parametrize("n_gates,n_pub,with_additions", [(13, 1, True), (120, 3, True), (500, 1, False),
                                                          (2000, 1, True)])
def test_fflonk_synthetic(env, n_gates, n_pub, with_additions):
    """2000 gates -> domain 2048, 18450 PTau points: the MSMs run in table mode."""
    op, off = env["op"], env["off"]
    gates, adds, n_vars, n_pub, wit = op.chain_gates(n_gates, n_pub=n_pub, with_additions=with_additions)
    zkey = off.fflonk_setup_synth(gates, adds, n_vars, n_pub, tau=0xFACE0FF + n_gates, structured=n_gates < 200)
    wtns = op.wtns_bytes(wit)
    pk = env["sb"].fflonk.ProvingKey(zkey, env["curve"])
    try:
        proof, public = env["sb"].fflonk.prove(pk, wtns, env["bl"])
        assert (proof, public) == off.fflonk_prove(zkey, wtns, BLINDERS)
        if n_gates < 200:
            assert off.fflonk_verify(off.fflonk_vk(zkey), public, proof)
        again, _ = env["sb"].fflonk.prove(pk, wtns, env["bl"])
        assert again == proof
    finally:
        pk.release()


def test_fflonk_key_from_file(env, golden, tmp_path):
    g = golden("fflonk_case.npz")
    zkey, wtns = bytes(g["zkey"]), bytes(g["wtns"])
    path = tmp_path / "circuit.zkey"
    path.write_bytes(zkey)
    pk = env["sb"].fflonk.ProvingKey.from_file(str(path), env["curve"])
    try:
        assert (env["sb"].fflonk.prove(pk, wtns, env["bl"])) == env["off"].fflonk_prove(zkey, wtns, BLINDERS)
    finally:
        pk.release()


def test_fflonk_errors(env, golden):
    sb, op, off, orc = env["sb"], env["op"], env["off"], env["orc"]
    g = golden("fflonk_case.npz")
    zkey, wtns = bytes(g["zkey"]), bytes(g["wtns"])
    _, w = orc.read_wtns(wtns)
    wit = [int.from_bytes(w[i:i + 32], "little") for i in range(0, len(w), 32)]
    pk = sb.fflonk.ProvingKey(zkey, env["curve"])
    try:
        bad = list(wit)
        bad[3] = (bad[3] + 1) % orc.P_BN_R
        with pytest.raises(sb.SbError, match="Copy constraints does not match|Polynomial is not divisible"):
            sb.fflonk.prove(pk, op.wtns_bytes(bad), env["bl"])
        with pytest.raises(sb.SbError, match=r"Invalid witness length. Circuit: \d+, witness: \d+, \d+"):
            sb.fflonk.prove(pk, op.wtns_bytes(wit[:-1]), env["bl"])
        proof, _ = sb.fflonk.prove(pk, wtns, env["bl"])
        assert proof == off.fflonk_prove(zkey, wtns, BLINDERS)[0]
    finally:
        pk.release()
    with pytest.raises(sb.SbError, match="zkey file is not fflonk"):
        sb.fflonk.ProvingKey(bytes(golden("plonk_case.npz")["zkey"]), env["curve"])
