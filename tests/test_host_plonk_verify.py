"""CPU: the per-proof code of the device PLONK / fflonk verifiers (snarkjs_b200/csrc/verify_plonk.cuh) compiled with g++ and
fp.cuh's host multiply (tests/host/plonk_verify_host.cpp): the shared Keccak-f[1600] sponge against the oracle's Keccak,
and for proofs from the oracle provers the challenges, L_1, PI(xi), r0 (and r1, r2, the quotients for fflonk), every
point-sum scalar and the pairing inputs against the oracle's big-integer arithmetic.  On BLS12-381 some commitments are on
the curve but outside the r-subgroup, which pins d4 = zh (T1 + xin T2 + xin^2 T3) nested as the reference nests it.  The
GPU twin is tests/test_gpu_plonk_verify.py."""
import json
import os
import random
import struct
import subprocess

import numpy as np
import pytest

from oracle import fflonk as OF
from oracle import oracle as O
from oracle import pairing_bls as PB
from oracle import plonk as OP
from snarkjs_b200 import fflonk, plonk

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BLINDERS = [0x2000 + 911 * i for i in range(11)]


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("pv") / "plonk_verify_host")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-o", path, os.path.join(ROOT, "tests", "host", "plonk_verify_host.cpp")])
    return path


def _run(exe, tmp_path, mode, blob):
    (tmp_path / "in.bin").write_bytes(blob)
    subprocess.check_call([exe, mode, str(tmp_path / "in.bin"), str(tmp_path / "out.bin")], timeout=600)
    return (tmp_path / "out.bin").read_bytes()


def test_keccak_against_oracle(exe, tmp_path):
    rng = random.Random(5)
    msgs = [bytes(rng.randrange(256) for _ in range(n)) for n in range(601)]
    blob = b"".join(struct.pack("<I", len(m)) + m for m in msgs)
    out = _run(exe, tmp_path, "keccak", blob)
    assert [out[32 * i:32 * (i + 1)] for i in range(len(msgs))] == [OP.keccak256(m) for m in msgs]


# ------------------------------------------------------------------------------------------------ per-proof scalars
PLONK_FIELDS = ["beta", "gamma", "alpha", "xi"] + [f"v{i}" for i in range(6)] + ["u", "xin", "zh", "l1", "pi", "r0"] + [f"s{j}" for j in range(18)]
FFLONK_FIELDS = (["beta", "gamma", "xi_seed", "alpha", "y", "xi", "xiw", "zh", "l1", "pi", "r0", "r1", "r2", "q1", "q2", "mulH0"]
                 + [f"S0_{i}" for i in range(8)] + [f"S1_{i}" for i in range(4)] + [f"S2_{i}" for i in range(3)]
                 + [f"S2p_{i}" for i in range(3)] + [f"s{j}" for j in range(5)])


def _record(proto, cid, vk, vkb, pub, prf):
    ci = O.CURVES[cid]
    head = struct.pack("<iiII", proto, 0 if cid == O.BN254 else 1, int(vk["nPublic"]), int(vk["power"]))
    wp = ci.fr_to_mont(plonk.fr_root(ci.r, int(vk["power"])))
    return head + vkb + ci.g1_affine_bytes(ci.g1) + ci.g2_affine_bytes(ci.g2) + wp + b"".join(int(s).to_bytes(32, "little") for s in pub) + prf


def _parse(cid, fields, out):
    ci = O.CURVES[cid]
    n8 = ci.n8q
    st = struct.unpack_from("<i", out)[0]
    vals = {f: ci.fr_from_mont(out[4 + 32 * i:4 + 32 * (i + 1)]) for i, f in enumerate(fields)}
    o = 4 + 32 * len(fields)
    pts = []
    if st == 0:
        for _ in range(2):
            pts.append(ci.g1_from_affine_bytes(out[o:o + 2 * n8]))
            o += 2 * n8
    return st, vals, pts, o


def _arith(cid):
    if cid == O.BN254:
        return O._g1_add_int, O._g1_mul_int, OP._neg
    return PB.g1_add, PB.g1_mul, PB.g1_neg


def _plonk_expected(cid, vk, pub, proof):
    """plonk_verify.js:208-421 restated on the oracle's helpers: the scalars and (p1, p2) = (-A1, B1)."""
    ci = O.CURVES[cid]
    r = ci.r
    add, mul, neg = _arith(cid)
    pr = {k: OP._g1(proof[k]) for k in plonk.POINTS}
    ev = {k: int(proof[k]) for k in plonk.EVALS}
    pr.update(ev)
    vkp = {k: OP._g1(vk[k]) for k in ("Qm", "Ql", "Qr", "Qo", "Qc", "S1", "S2", "S3")}
    k1, k2, power = int(vk["k1"]), int(vk["k2"]), int(vk["power"])
    p = [int(s) for s in pub]
    ch = OP._challenges(ci, vkp, p, pr)
    beta, gamma, alpha, xi, v, u = ch["beta"], ch["gamma"], ch["alpha"], ch["xi"], ch["v"], ch["u"]
    n = 1 << power
    xin = pow(xi, n, r)
    zh = (xin - 1) % r
    w = plonk.fr_root(r, power)
    L = [None] + [pow(w, i, r) * zh * pow(n * (xi - pow(w, i, r)), -1, r) % r for i in range(max(1, len(p)))]
    pi = -sum(s * L[i + 1] for i, s in enumerate(p)) % r
    ea, eb, ec, es1, es2, ezw = (ev[k] for k in plonk.EVALS)
    pa, pb = (ea + beta * es1 + gamma) % r, (eb + beta * es2 + gamma) % r
    e3 = pa * pb * (ec + gamma) * ezw * alpha % r
    r0 = (pi - L[1] * alpha * alpha - e3) % r
    bx = beta * xi % r
    d2 = ((ea + bx + gamma) * (eb + bx * k1 + gamma) * (ec + bx * k2 + gamma) * alpha + L[1] * alpha * alpha + u) % r
    d3 = pa * pb * (alpha * beta * ezw) % r
    e = (-r0 + sum(v[i] * x for i, x in zip(range(1, 6), (ea, eb, ec, es1, es2))) + u * ezw) % r
    s = [ea * eb % r, ea, eb, ec, d2, d3, v[1], v[2], v[3], v[4], v[5], e, xi, u * xi * w % r, u, xin, xin * xin % r, zh]
    want = dict(beta=beta, gamma=gamma, alpha=alpha, xi=xi, u=u, xin=xin, zh=zh, l1=L[1], pi=pi, r0=r0,
                **{f"v{i}": v[i] for i in range(1, 6)}, **{f"s{j}": x for j, x in enumerate(s)})
    d1 = add(add(add(add(mul(vkp["Qm"], s[0]), mul(vkp["Ql"], ea)), mul(vkp["Qr"], eb)), mul(vkp["Qo"], ec)), vkp["Qc"])
    d4 = mul(add(pr["T1"], add(mul(pr["T2"], xin), mul(pr["T3"], xin * xin % r))), zh)
    D = add(add(add(d1, mul(pr["Z"], d2)), neg(mul(vkp["S3"], d3))), neg(d4))
    F = D
    for pt, k in ((pr["A"], v[1]), (pr["B"], v[2]), (pr["C"], v[3]), (vkp["S1"], v[4]), (vkp["S2"], v[5])):
        F = add(F, mul(pt, k))
    A1 = add(pr["Wxi"], mul(pr["Wxiw"], u))
    B1 = add(add(add(mul(pr["Wxi"], xi), mul(pr["Wxiw"], s[13])), F), neg(mul(ci.g1, e)))
    return want, [neg(A1), B1]


def _fflonk_expected(vk, pub, proof):
    """fflonk_verify.js:198-542 restated on the oracle's helpers (BN254)."""
    ci = O.CURVES[O.BN254]
    r = ci.r
    add, mul, neg = _arith(O.BN254)
    pol = {k: OP._g1(proof["polynomials"][k]) for k in fflonk.POINTS}
    ev = {k: int(proof["evaluations"][k]) for k in OF.EVAL_NAMES}
    k1, k2, power = int(vk["k1"]), int(vk["k2"]), int(vk["power"])
    w, w3, w4, w8, wr = (int(vk[k]) for k in ("w", "w3", "w4", "w8", "wr"))
    C0 = OP._g1(vk["C0"])
    p = [int(s) for s in pub]
    t = OP.Transcript(ci)
    t.add_pol(C0)
    for s in p:
        t.add_scalar(s)
    t.add_pol(pol["C1"])
    beta = t.challenge()
    t.reset(); t.add_scalar(beta)
    gamma = t.challenge()
    t.reset(); t.add_scalar(gamma); t.add_pol(pol["C2"])
    xi_seed = t.challenge()
    S0, S1, S2, S2p, xi = OF._roots(r, xi_seed, w3, w4, w8, wr)
    xiw = xi * plonk.fr_root(r, power) % r
    t.reset(); t.add_scalar(xi_seed)
    for k in OF.EVAL_NAMES:
        t.add_scalar(ev[k])
    alpha = t.challenge()
    t.reset(); t.add_scalar(alpha); t.add_pol(pol["W1"])
    y = t.challenge()
    n = 1 << power
    zh = (pow(xi, n, r) - 1) % r
    izh = pow(zh, -1, r)
    L = [None] + [pow(w, i, r) * zh * pow(n * (xi - pow(w, i, r)), -1, r) % r for i in range(max(1, len(p)))]
    pi = -sum(s * L[i + 1] for i, s in enumerate(p)) % r
    li = OF._li_si(S0, y, xi, r)
    r0 = sum(sum(ev[nm] * pow(S0[i], k, r) for k, nm in enumerate(("ql", "qr", "qo", "qm", "qc", "s1", "s2", "s3"))) * li[i]
             for i in range(8)) % r
    t0 = (ev["ql"] * ev["a"] + ev["qr"] * ev["b"] + ev["qm"] * ev["a"] * ev["b"] + ev["qo"] * ev["c"] + ev["qc"] + pi) * izh % r
    li = OF._li_si(S1, y, xi, r)
    r1 = sum((ev["a"] + h * ev["b"] + h * h * ev["c"] + h ** 3 * t0) * li[i] for i, h in enumerate(S1)) % r
    t1 = (ev["z"] - 1) * L[1] * izh % r
    bx = beta * xi % r
    t21 = (ev["a"] + bx + gamma) * (ev["b"] + bx * k1 + gamma) * (ev["c"] + bx * k2 + gamma) * ev["z"]
    t22 = (ev["a"] + beta * ev["s1"] + gamma) * (ev["b"] + beta * ev["s2"] + gamma) * (ev["c"] + beta * ev["s3"] + gamma) * ev["zw"]
    t2 = (t21 - t22) * izh % r
    li2 = OF._li_s2(S2, S2p, y, xi, xiw, r)
    r2 = (sum((ev["z"] + h * t1 + h * h * t2) * li2[i] for i, h in enumerate(S2))
          + sum((ev["zw"] + h * ev["t1w"] + h * h * ev["t2w"]) * li2[3 + i] for i, h in enumerate(S2p))) % r
    prod = lambda xs: __import__("math").prod((y - x) % r for x in xs) % r
    mH0, mH1, mH2 = prod(S0), prod(S1), prod(S2 + S2p)
    q1 = alpha * mH0 * pow(mH1, -1, r) % r
    q2 = alpha * alpha * mH0 * pow(mH2, -1, r) % r
    e = (r0 + r1 * q1 + r2 * q2) % r
    want = dict(beta=beta, gamma=gamma, xi_seed=xi_seed, alpha=alpha, y=y, xi=xi, xiw=xiw, zh=zh, l1=L[1], pi=pi, r0=r0, r1=r1,
                r2=r2, q1=q1, q2=q2, mulH0=mH0, s0=q1, s1=q2, s2=e, s3=mH0, s4=y,
                **{f"S0_{i}": x for i, x in enumerate(S0)}, **{f"S1_{i}": x for i, x in enumerate(S1)},
                **{f"S2_{i}": x for i, x in enumerate(S2)}, **{f"S2p_{i}": x for i, x in enumerate(S2p)})
    A1 = add(add(add(add(add(C0, mul(pol["C1"], q1)), mul(pol["C2"], q2)), neg(mul(ci.g1, e))), neg(mul(pol["W1"], mH0))), mul(pol["W2"], y))
    return want, [pol["W2"], neg(A1)]


def _golden(name):
    g = np.load(os.path.join(ROOT, "tests", "golden", name))
    return {k: bytes(g[k]) for k in g.files}


def _synth(proto, n_pub, cid=O.BN254, n_gates=13):
    ci = O.CURVES[cid]
    gates, adds, n_vars, npub, wit = OP.chain_gates(n_gates, r=ci.r, n_pub=n_pub)
    if proto == "plonk":
        zkey = OP.plonk_setup_synth(gates, adds, n_vars, npub, tau=0x5151 + n_pub, curve=cid)
    else:
        zkey = OF.fflonk_setup_synth(gates, adds, n_vars, npub, tau=0x5151 + n_pub)
    return zkey, OP.wtns_bytes(wit, ci.r)


def _plonk_cases():
    g = _golden("plonk_case.npz")
    yield "plonk_case", O.BN254, g["zkey"], g["wtns"]
    for n_pub in (1, 5):
        yield f"synth-pub{n_pub}", O.BN254, *_synth("plonk", n_pub)
    yield "synth-bls-pub5", O.BLS12_381, *_synth("plonk", 5, O.BLS12_381)
    # the first challenge absorbs 704 + 32 n bytes on BN254 and 1056 + 32 n on BLS12-381: whole Keccak blocks at 12 and 18
    yield "synth-pub12", O.BN254, *_synth("plonk", 12, n_gates=60)
    yield "synth-bls-pub18", O.BLS12_381, *_synth("plonk", 18, O.BLS12_381, n_gates=60)
    yield "synth-pub1000", O.BN254, *_synth("plonk", 1000, n_gates=3000)


def _off_subgroup_point(rng):
    """A point of y^2 = x^3 + 4 over the BLS12-381 base field outside the r-subgroup."""
    q = O.P_BLS_Q
    while True:
        x = rng.randrange(q)
        rhs = (x ** 3 + 4) % q
        y = pow(rhs, (q + 1) // 4, q)
        if y * y % q == rhs and PB.g1_mul((x, y), O.P_BLS_R) is not None:
            return (x, y)


def test_plonk_scalars_and_pairing_inputs(exe, tmp_path):
    recs, exp = [], []
    for label, cid, zkey, wtns in _plonk_cases():
        ci = O.CURVES[cid]
        vk = plonk.verification_key(zkey)
        proof, pub = OP.plonk_prove(zkey, wtns, BLINDERS)
        variants = [proof]
        if cid == O.BLS12_381:
            rng = random.Random(3)
            for keys in (("T2",), ("T2", "T3", "Wxiw"), ("T1", "A", "Z")):
                bad = dict(proof)
                for k in keys:
                    x, y = _off_subgroup_point(rng)
                    bad[k] = [str(x), str(y), "1"]
                variants.append(bad)
        for pr in variants:
            recs.append(_record(0, cid, vk, plonk.vk_bytes(vk), pub, plonk.proof_bytes(pr, ci.n8q, ci.q, ci.r)))
            exp.append((label, cid) + _plonk_expected(cid, vk, pub, pr))
    out = _run(exe, tmp_path, "verify", b"".join(recs))
    o = 0
    for label, cid, want, pts in exp:
        st, vals, got_pts, used = _parse(cid, PLONK_FIELDS, out[o:])
        o += used
        assert st == 0, label
        for k, v in want.items():
            assert vals[k] == v, (label, k)
        assert got_pts == pts, label
    assert o == len(out)


def test_fflonk_scalars_and_pairing_inputs(exe, tmp_path):
    g = _golden("fflonk_case.npz")
    cases = [("fflonk_case", g["zkey"], g["wtns"])] + [(f"synth-pub{n}", *_synth("fflonk", n)) for n in (1, 5)]
    # the first challenge absorbs C0, the publics and C1, 128 + 32 n bytes: whole Keccak blocks at 13
    cases += [(f"synth-pub{n}", *_synth("fflonk", n, n_gates=ng)) for n, ng in ((13, 60), (1000, 3000))]
    recs, exp = [], []
    ci = O.CURVES[O.BN254]
    for label, zkey, wtns in cases:
        vk = fflonk.verification_key(zkey)
        proof, pub = OF.fflonk_prove(zkey, wtns, BLINDERS[:9])
        recs.append(_record(1, O.BN254, vk, fflonk.vk_bytes(vk), pub, fflonk.proof_bytes(proof, ci.n8q, ci.q, ci.r)))
        exp.append((label,) + _fflonk_expected(vk, pub, proof))
    out = _run(exe, tmp_path, "verify", b"".join(recs))
    o = 0
    for label, want, pts in exp:
        st, vals, got_pts, used = _parse(O.BN254, FFLONK_FIELDS, out[o:])
        o += used
        assert st == 0, label
        for k, v in want.items():
            assert vals[k] == v, (label, k)
        assert got_pts == pts, label
    assert o == len(out)


def test_checks_in_reference_order(exe, tmp_path):
    """3 (a point off the curve) before 4 (an evaluation >= r as Montgomery bytes) before 2 (a signal >= r)."""
    ci = O.CURVES[O.BN254]
    g = _golden("plonk_case.npz")
    vk = plonk.verification_key(g["zkey"])
    proof, pub = OP.plonk_prove(g["zkey"], g["wtns"], BLINDERS)
    good = plonk.proof_bytes(proof, 32, ci.q, ci.r)
    off = good[:64] + (5).to_bytes(32, "little") + good[96:]
    big_ev = good[:9 * 64] + ci.r.to_bytes(32, "little") + good[9 * 64 + 32:]
    both = off[:9 * 64] + big_ev[9 * 64:]
    bad_pub = [str(ci.r)] + pub[1:]
    cases = [(pub, off, 3), (bad_pub, both, 3), (pub, big_ev, 4), (bad_pub, big_ev, 4), (bad_pub, good, 2)]
    out = _run(exe, tmp_path, "verify", b"".join(_record(0, O.BN254, vk, plonk.vk_bytes(vk), p, prf) for p, prf, _ in cases))
    o = 0
    for p, prf, want in cases:
        st, _vals, _pts, used = _parse(O.BN254, PLONK_FIELDS, out[o:])
        o += used
        assert st == want
