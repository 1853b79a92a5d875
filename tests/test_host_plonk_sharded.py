"""CPU: the range arithmetic of sb_plonk_prove_multi / sb_fflonk_prove_multi before any GPU time.  The host PLONK and fflonk
flows (tests/host/host_plonk.cpp, host_fflonk.cpp) run on a stand-in oracle (tests/host/host_plonk_sharded.cpp) whose G1
MSM splits the PTau set into 1..9 ranges with the library's sb_shard_range and sums one partial per range, as the device
commitments do; every proof must be oracle/plonk.py's or oracle/fflonk.py's, including shard counts above the number of
points some commitments have (their later ranges are empty)."""
import ctypes
import os
import subprocess

import pytest

from oracle import fflonk
from oracle import oracle as orc
from oracle import plonk

from .test_host_fflonk import proof_from_bytes as ff_proof_from_bytes
from .test_host_plonk import proof_from_bytes as pl_proof_from_bytes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHARDS = range(1, 10)
PL_BLINDERS = [0x3100 + 7919 * i for i in range(11)]
FF_BLINDERS = [0x6100 + 15485863 * i for i in range(9)]
PROVE_ARGS = [ctypes.c_char_p, ctypes.c_char_p, ctypes.c_uint64, ctypes.c_char_p, ctypes.c_uint64, ctypes.c_char_p, ctypes.c_char_p,
              ctypes.c_char_p, ctypes.c_int]


@pytest.fixture(scope="module")
def libs(tmp_path_factory):
    from snarkjs_b200 import _native as N
    d = tmp_path_factory.mktemp("hps")
    out = {}
    for name, src in (("shim", "host_plonk_sharded.cpp"), ("plonk", "host_plonk.cpp"), ("fflonk", "host_fflonk.cpp")):
        so = str(d / f"lib{name}.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", so, os.path.join(ROOT, "tests", "host", src), "-ldl"])
        out[name] = (ctypes.CDLL(so), so)
    shim = out["shim"][0]
    shim.hs_configure.restype = ctypes.c_int
    shim.hs_configure.argtypes = [ctypes.c_char_p, ctypes.c_uint64, ctypes.c_int, ctypes.c_void_p]
    shim.hs_stats.argtypes = [ctypes.POINTER(ctypes.c_uint64)]
    for proto in ("plonk", "fflonk"):
        fn = getattr(out[proto][0], f"hp_{proto}_prove")
        fn.restype, fn.argtypes = ctypes.c_int, PROVE_ARGS
    out["range"] = ctypes.cast(N.lib().sb_shard_range, ctypes.c_void_p).value
    return out


def sharded_prove(libs, proto, zkey, wtns, blinders, shards, ci):
    """(rc, err, proof bytes, (MSMs, parts multiplied, parts left empty)) with the commitments summed over `shards` ranges"""
    from snarkjs_b200 import fflonk as sf
    from snarkjs_b200 import plonk as sp
    shim, shim_so = libs["shim"]
    n = (sp.read_zkey_header_plonk if proto == "plonk" else sf.read_zkey_header_fflonk)(zkey)["domainSize"]
    points = n + 6 if proto == "plonk" else 9 * n + 18
    assert shim.hs_configure(orc.build().encode(), points, shards, libs["range"]) == 0
    _, wit = orc.read_wtns(wtns)
    out = ctypes.create_string_buffer(9 * 2 * ci.n8q + 6 * 32 if proto == "plonk" else 4 * 64 + 16 * 32)
    err = ctypes.create_string_buffer(256)
    bl = b"".join(ci.fr_to_mont(b) for b in blinders)
    rc = getattr(libs[proto][0], f"hp_{proto}_prove")(shim_so.encode(), zkey, len(zkey), wit, len(wit) // 32, bl, out, err, 256)
    st = (ctypes.c_uint64 * 3)()
    shim.hs_stats(st)
    return rc, err.value.decode(), out.raw, tuple(st)


def check_plonk(libs, zkey, wtns, ci=orc.CURVES[orc.BN254]):
    want, public = plonk.plonk_prove(zkey, wtns, PL_BLINDERS)
    empty = 0
    for shards in SHARDS:
        rc, err, raw, (msms, parts, skipped) = sharded_prove(libs, "plonk", zkey, wtns, PL_BLINDERS, shards, ci)
        assert rc == 0, err
        assert pl_proof_from_bytes(raw, ci) == want, shards
        assert msms == 9 and parts + skipped == 9 * shards
        empty += skipped
    return public, empty


def check_fflonk(libs, zkey, wtns):
    ci = orc.CURVES[orc.BN254]
    want, public = fflonk.fflonk_prove(zkey, wtns, FF_BLINDERS)
    empty = 0
    for shards in SHARDS:
        rc, err, raw, (msms, parts, skipped) = sharded_prove(libs, "fflonk", zkey, wtns, FF_BLINDERS, shards, ci)
        assert rc == 0, err
        assert ff_proof_from_bytes(raw) == want, shards
        assert msms == 4 and parts + skipped == 4 * shards
        empty += skipped
    return public, empty


def test_shard_ranges_cover_the_points(libs):
    """sb_shard_range splits P points into contiguous ranges that cover [0, P) once, empty ranges last."""
    from snarkjs_b200 import _native as N
    L = N.lib()
    for total in (0, 1, 5, 22, 27, 2 ** 14 + 6, 9 * 2 ** 10 + 18):
        for shards in range(1, 12):
            nxt = 0
            for i in range(shards):
                lo, cnt = ctypes.c_uint64(), ctypes.c_uint64()
                L.sb_shard_range(total, i, shards, ctypes.byref(lo), ctypes.byref(cnt))
                assert lo.value == nxt or cnt.value == 0
                nxt = lo.value + cnt.value
            assert nxt == total


def test_plonk_reference_fixture(libs, golden):
    g = golden("plonk_case.npz")
    _, empty = check_plonk(libs, bytes(g["zkey"]), bytes(g["wtns"]))
    assert empty > 0                           # with 9 ranges of n + 6 = 14 points, the n + 1 point commitments leave ranges empty


@pytest.mark.parametrize("n_gates,n_pub", [(13, 1), (29, 3), (120, 1)])
def test_plonk_synthetic(libs, n_gates, n_pub):
    gates, adds, n_vars, n_pub, wit = plonk.chain_gates(n_gates, n_pub=n_pub)
    zkey = plonk.plonk_setup_synth(gates, adds, n_vars, n_pub, tau=0x5A4D + n_gates)
    wtns = plonk.wtns_bytes(wit)
    public, _ = check_plonk(libs, zkey, wtns)
    rc, err, raw, _ = sharded_prove(libs, "plonk", zkey, wtns, PL_BLINDERS, 7, orc.CURVES[orc.BN254])
    assert plonk.plonk_verify(plonk.plonk_vk(zkey), public, pl_proof_from_bytes(raw))


def test_plonk_bls12381(libs):
    ci = orc.CURVES[orc.BLS12_381]
    gates, adds, n_vars, n_pub, wit = plonk.chain_gates(40, r=ci.r)
    zkey = plonk.plonk_setup_synth(gates, adds, n_vars, n_pub, tau=77713, curve=orc.BLS12_381)
    check_plonk(libs, zkey, plonk.wtns_bytes(wit, ci.r), ci)


def test_fflonk_reference_fixture(libs, golden):
    g = golden("fflonk_case.npz")
    check_fflonk(libs, bytes(g["zkey"]), bytes(g["wtns"]))


@pytest.mark.parametrize("n_gates,n_pub,with_additions", [(3, 1, False), (29, 3, True)])
def test_fflonk_synthetic(libs, n_gates, n_pub, with_additions):
    """3 gates: domain 4, so C1's 8n = 32 of the 9n + 18 = 54 points leave the last ranges of 9 empty"""
    gates, adds, n_vars, n_pub, wit = plonk.chain_gates(n_gates, n_pub=n_pub, with_additions=with_additions)
    zkey = fflonk.fflonk_setup_synth(gates, adds, n_vars, n_pub, tau=0xFF5A + n_gates, structured=True)
    public, empty = check_fflonk(libs, zkey, plonk.wtns_bytes(wit))
    assert fflonk.fflonk_verify(fflonk.fflonk_vk(zkey), public, ff_proof_from_bytes(sharded_prove(libs, "fflonk", zkey, plonk.wtns_bytes(wit), FF_BLINDERS, 9,
                                                                                                   orc.CURVES[orc.BN254])[2]))
    if n_gates == 3:
        assert empty > 0
