"""CPU: the six entries of a batch of one key on several devices are exported with the prototypes of include/snarkb200.h,
refuse null and repeated contexts before touching a device, and their Python wrappers fail with the library's no-device
error without a GPU."""
import ctypes
import os
import re

import pytest

from snarkjs_b200 import _native as N

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PROTOS = ("groth16", "plonk", "fflonk")
ENTRIES = tuple(f"sb_{p}_{e}" for p in PROTOS for e in ("load_replicas", "prove_batch_multi"))


@pytest.mark.parametrize("name", ENTRIES)
def test_signature_matches_header(name):
    hdr = open(os.path.join(ROOT, "include", "snarkb200.h")).read()
    m = re.search(r"int\s+%s\s*\(([^)]*)\)\s*;" % name, hdr)
    assert m, "prototype not found"
    params = [" ".join(p.split()) for p in m.group(1).split(",")]
    restype, argtypes = N._SIGNATURES[name]
    assert restype is ctypes.c_int
    assert len(argtypes) == len(params)
    scalar = {"int": ctypes.c_int, "uint64_t": ctypes.c_uint64, "uint32_t": ctypes.c_uint32}
    for p, t in zip(params, argtypes):
        if "* const*" in p:
            assert t is ctypes.POINTER(ctypes.c_void_p), p
        elif "uint64_t*" in p:
            assert t in (ctypes.POINTER(ctypes.c_uint64), ctypes.c_void_p), p
        elif "*" in p:
            assert t is ctypes.c_void_p, p
        else:
            assert t is scalar[p.split()[0]], p
    assert getattr(N.lib(), name) is not None


def prove_args(proto, ctxs, handles, n, buf):
    """sb_<proto>_prove_batch_multi arguments: one witness of one element, every buffer `buf`"""
    tail = (buf, buf, buf) if proto == "groth16" else (buf, buf, None)
    return (ctxs, handles, n, buf, 1, 1) + tail


@pytest.mark.parametrize("proto", PROTOS)
def test_rejects_null_and_repeated_contexts(proto):
    L = N.lib()
    load, prove = getattr(L, f"sb_{proto}_load_replicas"), getattr(L, f"sb_{proto}_prove_batch_multi")
    buf = ctypes.create_string_buffer(512)
    handles = (ctypes.c_uint64 * 4)(1, 2, 3, 4)
    none = (ctypes.c_void_p * 4)()
    fake = ctypes.c_void_p(ctypes.addressof(buf))      # never dereferenced: a repeated context is refused first
    twice = (ctypes.c_void_p * 2)(fake, fake)
    assert load(None, 1, buf, 512, handles) == -1
    assert load(none, 2, buf, 512, handles) == -1
    assert load(none, 0, buf, 512, handles) == -1
    assert load(none, 65, buf, 512, handles) == -1
    assert prove(*prove_args(proto, None, handles, 1, buf)) == -1
    assert prove(*prove_args(proto, none, handles, 3, buf)) == -1
    assert prove(*prove_args(proto, none, handles, 0, buf)) == -1
    assert prove(*prove_args(proto, none, handles, 65, buf)) == -1
    # the repeat is found before either context is touched; the message is the calling thread's
    assert load(twice, 2, buf, 512, handles) == -1
    assert L.sb_last_error(fake) == f"sb_{proto}_load_replicas: context 1 is context 0 again".encode()
    assert prove(*prove_args(proto, twice, handles, 2, buf)) == -1
    assert L.sb_last_error(fake) == f"sb_{proto}_prove_batch_multi: context 1 is context 0 again".encode()


def test_wrappers_raise_no_device_error():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    import snarkjs_b200
    from oracle import fflonk as offlonk
    from oracle import plonk as oplonk
    from snarkjs_b200 import synth
    gates, adds, n_vars, n_pub, _wit = oplonk.chain_gates(13)
    zkey = oplonk.plonk_setup_synth(gates, adds, n_vars, n_pub, tau=99)
    fzkey = offlonk.fflonk_setup_synth(gates, adds, n_vars, n_pub, tau=99)
    from oracle import oracle as O
    ci = O.CURVES[O.BN254]
    gzkey = synth.groth16_zkey_image(ci.q, ci.r, 32, 4, lambda grp, sd, k: bytes(k * 64 * grp))
    for M, key in ((snarkjs_b200.groth16, gzkey), (snarkjs_b200.plonk, zkey), (snarkjs_b200.fflonk, fzkey)):
        with pytest.raises(snarkjs_b200.SbError, match="no CUDA device"):
            M.ReplicatedProvingKey(key, [0, 0])
